#!/usr/bin/env python
"""Offline rendering with Runtime.process_offline against the block-by-block ways of doing the same job.  Prints one JSON line.

  (a) 4096 SUBSYNTH32 voices, mix only, 1 channel: process_offline vs an enqueue_block(FLAG_MIX) device-resident loop and a process() loop.
  (b) BASELINE config 4's shape: 1024 channels of per-voice input through one 16 384-tap IR, mix and per-voice outputs: process_offline vs
      a process_voices() loop (2 MiB of input per block go up).
  (c) BASELINE config 5's 1250 graphs as stems (graph i on channel i), mix only at nOut = 1250: process_offline vs render_offline's
      per-graph outputs.

Each leg is timed over --blocks blocks (default 1024) after --warmup blocks, with a host clock around a call that ends synchronised, and
checks its output bits against a block-by-block twin runtime with the same setup.  The card's name and power limit are read in the same
run.  Usage: python tools/offline_bench.py [--blocks N] [--warmup W] [--legs abc]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elementary_b200 import Runtime, graphs  # noqa: E402
from elementary_b200.runtime import FLAG_MIX  # noqa: E402

SR, BS = 48000.0, 512


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:        # the number is still reported; without the power limit it says so
        out["power_limit_w"] = f"unavailable: {e}"
    return out


def same_bits(a, b):
    return bool(np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32)))


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def leg_a(blocks, warmup):
    def make():
        rt = Runtime(SR, BS, 4096, device=0, specialize=2)
        assert rt.apply_instructions(graphs.subsynth32()) == 0, rt.last_error()
        ida, idb = graphs.subsynth32_param_ids()
        f0 = np.array([graphs.subsynth32_f0(v) for v in range(4096)], dtype=np.float64)
        assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
        return rt
    off, host, dev = make(), make(), make()
    n = blocks * BS
    off.process_offline(num_samples=warmup * BS, num_outputs=1)
    for _ in range(warmup):
        host.process(None, 1, BS)
        dev.enqueue_block(0, 1, BS, FLAG_MIX)
    dev.synchronize()
    t_off, (mix, _) = timed(lambda: off.process_offline(num_samples=n, num_outputs=1))
    ref = np.zeros((1, n), np.float32)

    def host_loop():
        for k in range(blocks):
            ref[:, k * BS:(k + 1) * BS] = host.process(None, 1, BS)
    t_host, _ = timed(host_loop)

    def dev_loop():
        for _ in range(blocks):
            dev.enqueue_block(0, 1, BS, FLAG_MIX)
        dev.synchronize()
    t_dev, _ = timed(dev_loop)
    return {"what": "4096 SUBSYNTH32 voices, mix only, 1 channel", "blocks": blocks,
            "process_offline_ms_per_block": t_off / blocks * 1e3, "process_loop_ms_per_block": t_host / blocks * 1e3,
            "enqueue_block_loop_ms_per_block": t_dev / blocks * 1e3, "bits_equal_process_loop": same_bits(mix, ref)}


def leg_b(blocks, warmup):
    channels = 1024
    ir = np.asarray(graphs.lcg_ir(16384), dtype=np.float32)

    def make():
        rt = Runtime(SR, BS, channels, device=0)
        assert rt.add_shared_resource("ir", ir)
        assert rt.apply_instructions(graphs.convolve_channel("ir")) == 0, rt.last_error()
        return rt
    off, twin = make(), make()
    rng = np.random.default_rng(1)
    w = (rng.random((channels, 1, warmup * BS), dtype=np.float32) - 0.5) * 0.5
    x = (rng.random((channels, 1, blocks * BS), dtype=np.float32) - 0.5) * 0.5
    off.process_offline(voice_inputs=w, want_voices=True)
    for k in range(warmup):
        twin.process_voices(w[:, :, k * BS:(k + 1) * BS], 1, BS)
    t_off, (mix, v) = timed(lambda: off.process_offline(voice_inputs=x, want_voices=True))
    rm = np.zeros_like(mix)
    rv = np.zeros_like(v)

    def loop():
        for k in range(blocks):
            s = slice(k * BS, (k + 1) * BS)
            rv[:, :, s], rm[:, s] = twin.process_voices(x[:, :, s], 1, BS)
    t_loop, _ = timed(loop)
    return {"what": "config 4 shape: 1024 channels of per-voice input, one 16384-tap IR, mix + per-voice outputs", "blocks": blocks,
            "process_offline_ms_per_block": t_off / blocks * 1e3, "process_voices_loop_ms_per_block": t_loop / blocks * 1e3,
            "h2d_mib_per_block": channels * BS * 4 / 2 ** 20, "bits_equal_process_voices_loop": same_bits(mix, rm) and same_bits(v, rv)}


def leg_c(blocks, warmup):
    n_graphs = 1250

    def make():
        rt = Runtime(SR, BS, n_graphs, device=0)
        for i in range(n_graphs):
            batch = graphs.random_graph(i, 64)
            for ins in batch:                    # graph i on channel i
                if ins[0] == 3 and ins[2] == "channel":
                    ins[3] = i
            assert rt.apply_instructions(batch, voices=(i, i + 1)) == 0, rt.last_error()
        return rt
    off, twin, per = make(), make(), make()
    off.process_offline(num_samples=warmup * BS, num_outputs=n_graphs)
    twin.process_offline(num_samples=warmup * BS, num_outputs=n_graphs)
    per.render_offline(warmup, 1)
    n = blocks * BS
    t_off, (mix, _) = timed(lambda: off.process_offline(num_samples=n, num_outputs=n_graphs))
    out = np.empty((n_graphs, 1, n), dtype=np.float32)
    t_per, _ = timed(lambda: per.render_offline(blocks, 1, out=out))
    check = min(blocks, 64)                      # the block-by-block twin over the first blocks of the timed window
    ref = np.zeros((n_graphs, check * BS), np.float32)
    for k in range(check):
        ref[:, k * BS:(k + 1) * BS] = twin.process(None, n_graphs, BS)
    return {"what": "config 5's 1250 graphs as stems (graph i on channel i), mix only at nOut = 1250", "blocks": blocks,
            "process_offline_ms_per_block": t_off / blocks * 1e3, "process_offline_msamples_per_s": n_graphs * n / t_off / 1e6,
            "render_offline_ms_per_block": t_per / blocks * 1e3, "render_offline_msamples_per_s": n_graphs * n / t_per / 1e6,
            "twin_blocks_checked": check, "bits_equal_process_loop": same_bits(mix[:, :check * BS], ref)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--legs", default="abc")
    a = ap.parse_args()
    res = {"gpu": card()}
    for leg in a.legs:
        res[leg] = {"a": leg_a, "b": leg_b, "c": leg_c}[leg](a.blocks, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
