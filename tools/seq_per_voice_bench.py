#!/usr/bin/env python
"""Per-voice sequences on the GPU: ms per block and K1 time for sequenced voices whose patterns are one per voice group, one of 64 per
voice, or one per voice, against voice-group cuts.

Workloads per voice (48 kHz, 512-sample blocks, mix bus only, device-resident blocks through enqueue_block):
  * sampler:    sparseq (a 16-step trigger pattern, clocked by a per-voice pulse train) -> sample, which plays one of 64 one-second
                buffers (set_path_per_voice: one voice group);
  * oscillator: seq2 (an 8-step frequency pattern, hold, clocked the same way) -> cycle.
Arms:
  a  group:     one group-wide sequence, set by JSON `seq`, as before set_seq_per_voice existed;
  b  per64:     set_seq_per_voice, each voice one of 64 distinct sequences;
  c  distinct:  set_seq_per_voice, every voice its own sequence;
  d  cuts:      tile width 1, the voices cut into one group per distinct sequence (64) by JSON `seq` batches on voice sub-ranges —
                the way to give voices different patterns without set_seq_per_voice (only at 4096 voices: the tool's --cut-voices).
K1 time comes from per-kernel CUDA events in a second pass (engine option time_kernels), as tools/sample_bench.py takes it; every
arm runs the interpreter (specialize=0), so that the 64 groups of arm d do not each wait for their own NVRTC compile.
`set_ms` is the host time of the set_seq_per_voice call (arms b and c; d: the 64 JSON batches).  One JSON line per (workload, arm,
voices); the card's name and power limit are read in the same run.
Usage: python tools/seq_per_voice_bench.py [--voices 4096,131072] [--cut-voices 4096] [--blocks 100] [--warmup 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                                   # noqa: E402
from elementary_b200 import Runtime, el              # noqa: E402
from elementary_b200.runtime import FLAG_MIX         # noqa: E402

SR, BS, N_RES, N_SEQ = 48000.0, 512, 64, 64


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def pattern(workload, k):
    """The k-th distinct sequence of a workload (deterministic in k)."""
    rng = np.random.default_rng(1000 + k)
    if workload == "sampler":
        hits = rng.random(16) < 0.5
        hits[0] = True
        return [{"tickTime": 2 * i, "value": 1.0} for i in range(16) if hits[i]] + \
               [{"tickTime": 2 * i + 1, "value": 0.0} for i in range(16) if hits[i]]
    return [float(np.float32(110.0 * 2.0 ** (rng.integers(0, 24) / 12.0))) for _ in range(8)]


def graph(workload):
    clock = el.le(el.phasor(el.const(8.0, key="clk")), 0.5)
    if workload == "sampler":
        sq = el.sparseq({"key": "sq", "seq": pattern(workload, 0), "loop": [0, 32]}, clock)
        return sq, el.sample({"key": "smp", "path": "res0", "mode": "trigger"}, sq, el.const(1.0, key="rate"))
    sq = el.seq2({"key": "sq", "seq": pattern(workload, 0), "hold": True}, clock)
    return sq, el.mul(0.1, el.cycle(sq))


def build(workload, arm, n, device=0):
    rt = Runtime(SR, BS, n, device=device, specialize=0, **({"tile_width": 1} if arm == "cuts" else {}))
    rng = np.random.default_rng(1)
    names = [f"res{k}" for k in range(N_RES)]
    if workload == "sampler":
        for nm in names:
            assert rt.add_shared_resource(nm, rng.standard_normal(int(SR)).astype(np.float32))
    sq, root = graph(workload)
    assert rt.apply_instructions(el.render(root)) == 0, rt.last_error()
    v = np.arange(n)
    assert rt.set_property_per_voice(el.const(0, key="clk").id(), "value", 4.0 + (v % 13) * 0.37) == 0
    if workload == "sampler":
        assert rt.set_path_per_voice(root.id(), names, v % N_RES) == 0, rt.last_error()
    set_ms = None
    if arm in ("per64", "distinct"):
        k = N_SEQ if arm == "per64" else n
        seqs = [pattern(workload, i) for i in range(k)]
        index = (v * 7) % k if arm == "per64" else v
        t0 = time.perf_counter()
        assert rt.set_seq_per_voice(sq.id(), seqs, index) == 0, rt.last_error()
        set_ms = (time.perf_counter() - t0) * 1e3
    elif arm == "cuts":
        t0 = time.perf_counter()
        for i in range(N_SEQ):
            vb, ve = i * n // N_SEQ, (i + 1) * n // N_SEQ
            assert rt.apply_instructions([[3, sq.id(), "seq", pattern(workload, i)]], voices=(vb, ve)) == 0, rt.last_error()
        set_ms = (time.perf_counter() - t0) * 1e3
    return rt, set_ms


def run(workload, arm, n, blocks, warmup):
    rt, set_ms = build(workload, arm, n)
    for _ in range(warmup):
        rt.enqueue_block(0, 1, BS, FLAG_MIX)
    rt.synchronize()
    groups = rt.describe()["groups"]
    t0 = time.perf_counter()
    for _ in range(blocks):
        rt.enqueue_block(0, 1, BS, FLAG_MIX)
    rt.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / blocks
    rt.set_option("time_kernels", 1)        # kernel durations in a second pass: the event pairs stay out of the timed loop
    rt.take_kernel_time_ms()
    for _ in range(blocks):
        rt.enqueue_block(0, 1, BS, FLAG_MIX)
    k1_ms, k1_n = rt.take_kernel_time_ms()
    _, mix = rt.process_voices(None, 1, BS, want_voices=False)
    return {"workload": workload, "arm": arm, "voices": n, "groups": len(groups), "tile_width": groups[0]["tile_width"],
            "blocks": blocks, "ms_per_block": wall, "k1_ms_per_block": k1_ms / blocks, "k1_launches_per_block": k1_n / blocks,
            "set_ms": set_ms, "mix_peak": float(np.abs(mix).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", default="4096,131072")
    ap.add_argument("--cut-voices", default="4096")
    ap.add_argument("--blocks", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--workloads", default="sampler,oscillator")
    a = ap.parse_args()
    gpu = card()
    cut = {int(x) for x in a.cut_voices.split(",") if x}
    for workload in a.workloads.split(","):
        for n in (int(x) for x in a.voices.split(",")):
            for arm in ("group", "per64", "distinct", "cuts"):
                if arm == "cuts" and n not in cut:
                    continue
                r = run(workload, arm, n, a.blocks, a.warmup)
                r["gpu"] = gpu
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
