#!/usr/bin/env python
"""Meter readouts as arrays (elem_b200_poll_readouts, elem_b200_process_offline_readouts) against the JSON event path, on cuda:0.  Prints
one JSON line; the card's name and power limit are read in the same run.

  (a) N SUBSYNTH32 voices, each under a `meter` (4096 and 131072 by default), mix only.  Offline legs: process_offline with JSON events,
      with readouts, and with neither.  Live legs: process() + JSON poll, process() + host-mode array poll, and enqueue_block +
      device-mode array poll into a [blocks][voices] device tensor with one synchronise at the end.
  (b) BASELINE config 5's 1250 random 64-node graphs (one voice group each), each with a `meter` between its root and its output: the
      host-mode array poll of all 1250 voices after each process() and the K5 launches it takes.
Time per block is the host clock around each call or loop (each ends with its results on the host, or after a synchronise).  The JSON
legs at the largest voice count are host-bound at several hundred ms per block, so they run `--json-blocks` blocks.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elementary_b200 import Runtime, el, graphs  # noqa: E402
from elementary_b200.runtime import FLAG_MIX  # noqa: E402

SR, BS = 48000.0, 512
METER = el.meter({"name": "v"}, graphs.subsynth32_graph())


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return out.strip().splitlines()[0]
    except Exception as exc:   # noqa: BLE001
        return f"unknown ({exc})"


def subsynth_meter(n_voices):
    rt = Runtime(SR, BS, n_voices, device=0)
    assert rt.apply_instructions(el.render(METER)) == 0
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(n_voices)])
    assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    return rt


def timed(fn, blocks):
    t0 = time.perf_counter()
    out = fn()
    return 1e3 * (time.perf_counter() - t0) / blocks, out


def legs_a(n_voices, blocks, json_blocks, warmup):
    import torch
    rt = subsynth_meter(n_voices)
    mid = METER.id()
    res = {"voices": n_voices, "blocks": blocks, "json_blocks": json_blocks}
    # warm-up of every leg's shapes
    rt.process_offline(num_samples=warmup * BS, on_event=lambda *a: None)
    rt.process_offline(num_samples=warmup * BS, readouts=[mid])
    rt.process_offline(num_samples=warmup * BS)
    for _ in range(warmup):
        rt.process(None, 1, BS)
        rt.poll_readouts(mid)
        rt.process(None, 1, BS)
        rt.process_queued_events()
    count = [0]

    def on_event(k, t, e):
        count[0] += 1
    res["offline_events_ms_per_block"], _ = timed(lambda: rt.process_offline(num_samples=json_blocks * BS, on_event=on_event), json_blocks)
    res["offline_events"] = count[0]
    res["offline_readouts_ms_per_block"], out = timed(lambda: rt.process_offline(num_samples=blocks * BS, readouts=[mid]), blocks)
    res["offline_readouts_fresh"] = int(out[2][mid]["fresh"].sum())
    res["offline_ms_per_block"], _ = timed(lambda: rt.process_offline(num_samples=blocks * BS), blocks)

    def json_loop():
        n = 0
        for _ in range(json_blocks):
            rt.process(None, 1, BS)
            n += len(rt.process_queued_events())
        return n
    res["loop_json_ms_per_block"], res["loop_json_events"] = timed(json_loop, json_blocks)

    def array_loop():
        n = 0
        for _ in range(blocks):
            rt.process(None, 1, BS)
            n += int(rt.poll_readouts(mid)["fresh"].sum())
        return n
    res["loop_array_ms_per_block"], res["loop_array_fresh"] = timed(array_loop, blocks)

    def plain_loop():
        for _ in range(blocks):
            rt.process(None, 1, BS)
    res["loop_no_poll_ms_per_block"], _ = timed(plain_loop, blocks)

    a = torch.empty((blocks, n_voices), device="cuda:0")
    b = torch.empty((blocks, n_voices), device="cuda:0")
    f = torch.zeros((blocks, n_voices), dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()

    def device_loop():
        for k in range(blocks):
            rt.enqueue_block(0, 1, BS, FLAG_MIX)
            rt.poll_readouts_device(mid, a[k].data_ptr(), b[k].data_ptr(), f[k].data_ptr())
        rt.synchronize()
    res["device_loop_ms_per_block"], _ = timed(device_loop, blocks)
    res["device_loop_fresh"] = int(f.sum().item())

    def device_plain():
        for _ in range(blocks):
            rt.enqueue_block(0, 1, BS, FLAG_MIX)
        rt.synchronize()
    res["device_no_poll_ms_per_block"], _ = timed(device_plain, blocks)
    rt.close()
    return res


def metered(batch, mid):
    """A random graph with a meter between its root and the root's child."""
    root = next(ins[1] for ins in batch if ins[0] == 0 and ins[2] == "root")
    out = [[0, mid, "meter"]]
    for ins in batch:
        if ins[0] == 2 and ins[1] == root:
            out += [[2, root, mid, 0], [2, mid, ins[2], ins[3]]]
        else:
            out.append(ins)
    return out


def legs_b(n_graphs, blocks, warmup):
    mid = 0x7ead0001
    rt = Runtime(SR, BS, n_graphs, device=0)
    for i in range(n_graphs):
        assert rt.apply_instructions(metered(graphs.random_graph(i, 64), mid), voices=(i, i + 1)) == 0, rt.last_error()
    for _ in range(warmup):
        rt.process(None, 1, BS)
        rt.poll_readouts(mid)

    def plain():
        for _ in range(blocks):
            rt.process(None, 1, BS)
    res = {"graphs": n_graphs, "blocks": blocks}
    res["loop_no_poll_ms_per_block"], _ = timed(plain, blocks)
    l0 = rt.kernel_launches
    rt.poll_readouts(mid)
    res["k5_launches_per_poll"] = rt.kernel_launches - l0

    def arrays():
        n = 0
        for _ in range(blocks):
            rt.process(None, 1, BS)
            n += int(rt.poll_readouts(mid)["fresh"].sum())
        return n
    res["loop_array_ms_per_block"], res["loop_array_fresh"] = timed(arrays, blocks)

    def js():
        n = 0
        for _ in range(blocks):
            rt.process(None, 1, BS)
            n += len(rt.process_queued_events())
        return n
    res["loop_json_ms_per_block"], res["loop_json_events"] = timed(js, blocks)
    rt.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, nargs="+", default=[4096, 131072])
    ap.add_argument("--blocks", type=int, default=1024)
    ap.add_argument("--json-blocks", type=int, nargs="+", default=[1024, 16], help="blocks of the JSON legs, per voice count")
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--graphs", type=int, default=1250)
    ap.add_argument("--graph-blocks", type=int, default=256)
    args = ap.parse_args()
    jb = args.json_blocks + [args.json_blocks[-1]] * max(0, len(args.voices) - len(args.json_blocks))
    out = {"gpu": gpu_info(), "block_size": BS,
           "a_subsynth32_meter": [legs_a(v, args.blocks, j, args.warmup) for v, j in zip(args.voices, jb)],
           "b_config5_meter": legs_b(args.graphs, args.graph_blocks, args.warmup)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
