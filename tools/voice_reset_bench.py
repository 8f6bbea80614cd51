#!/usr/bin/env python
"""Voice resets (Runtime.reset_voices, K6) under a voice allocator's load.  Prints one JSON line.

SUBSYNTH32 at 4096 and 131 072 voices in a device-resident enqueue_block(FLAG_MIX) loop; before every block a fresh random set of
0 %, 1 %, 10 % or 100 % of the voices is reset.  The arms alternate in rounds of --round blocks inside one run, and each block (reset +
render) is timed with CUDA events on the engine's stream after --warmup blocks of every arm, until every arm has --blocks blocks.
A second pass of its own, under torch.profiler, reads the reset kernel's own device time; its bytes per call are counted from the
reset plans (Runtime.reset_bytes_written) and set against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card's name and
power limit are read in the same run.  Usage: python tools/voice_reset_bench.py [--voices 4096,131072] [--blocks 200] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elementary_b200 import Runtime, graphs  # noqa: E402
from elementary_b200.runtime import FLAG_MIX  # noqa: E402

SR, BS = 48000.0, 512
RATES = (0.0, 0.01, 0.10, 1.0)
DATASHEET_BPS = 3.35e12


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:
        out["power_limit_w"] = f"unavailable: {e}"
    return out


def synth(nv, stream):
    rt = Runtime(SR, BS, nv, device=0, specialize=2)
    rt.set_stream(stream.cuda_stream)
    assert rt.apply_instructions(graphs.subsynth32()) == 0, rt.last_error()
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(nv)])
    assert rt.set_property_per_voice(ida, "value", f0) == 0
    assert rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    return rt


def block(rt, rng, rate):
    k = int(round(rate * rt.num_voices))
    if k:
        assert rt.reset_voices(rng.choice(rt.num_voices, size=k, replace=False).astype(np.int32)) == 0, rt.last_error()
    rt.enqueue_block(0, 1, BS, flags=FLAG_MIX)


def measure(nv, args, torch):
    stream = torch.cuda.Stream()
    rt = synth(nv, stream)
    rng = np.random.default_rng(nv)
    for rate in RATES:                                    # warm-up: every arm's shapes and buffers
        for _ in range(args.warmup):
            block(rt, rng, rate)
    rt.synchronize()
    times = {r: [] for r in RATES}
    launches = {}
    while min(len(t) for t in times.values()) < args.blocks:
        for rate in RATES:
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.round)]
            l0 = rt.kernel_launches
            for a, b in evs:
                a.record(stream)
                block(rt, rng, rate)
                b.record(stream)
            launches[rate] = (rt.kernel_launches - l0) / args.round
            stream.synchronize()
            times[rate] += [a.elapsed_time(b) for a, b in evs]
    out = {"voices": nv, "arms": {}}
    for rate in RATES:
        t = np.array(times[rate])
        out["arms"][f"{rate:g}"] = {"block_ms_median": float(np.median(t)), "block_ms_p10": float(np.percentile(t, 10)),
                                   "block_ms_p90": float(np.percentile(t, 90)), "blocks": int(t.size),
                                   "launches_per_block": launches[rate]}
    # the reset kernel's own time: a profiled pass of its own
    from torch.profiler import ProfilerActivity, profile
    for rate in RATES[1:]:
        b0, n = rt.reset_bytes_written, args.profile_blocks
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                block(rt, rng, rate)
            rt.synchronize()
        bytes_per_call = (rt.reset_bytes_written - b0) / n
        ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "reset_voices_kernel" in e.name]
        us = float(np.median([e.time_range.elapsed_us() for e in ks])) if ks else None
        arm = out["arms"][f"{rate:g}"]
        arm.update({"reset_kernel_us_median": us, "reset_kernel_calls_seen": len(ks), "reset_bytes_per_call": bytes_per_call})
        if us:
            arm["reset_bytes_per_s"] = bytes_per_call / (us * 1e-6)
            arm["reset_share_of_datasheet_hbm"] = arm["reset_bytes_per_s"] / DATASHEET_BPS
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", default="4096,131072")
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--round", type=int, default=20)
    ap.add_argument("--profile-blocks", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("voice_reset_bench: no CUDA device: nothing is measured")
    res = {"bench": "voice_reset", "card": card(), "datasheet_hbm_bytes_per_s": DATASHEET_BPS,
           "runs": [measure(int(v), args, torch) for v in args.voices.split(",")]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "voice_reset_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
