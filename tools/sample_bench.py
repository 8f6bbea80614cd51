#!/usr/bin/env python
"""Sampler voices on the GPU: ms per block, K1 time and the bytes the render program gathers, for `sample` next to the same
voice count with `table` in its place.

Workload per voice: a pulse train (le(phasor(f), 0.5), f per voice) triggers `sample` at a per-voice rate, straight into the root;
the voice plays one of 64 one-second resources (set_path_per_voice: one voice group).  The `table` arm reads one of the same
resources with a per-voice phasor.  48 kHz, 512-sample blocks, mix bus only, device-resident blocks (enqueue_block).
`gather_bytes_per_block` is counted from the program: every sample op may gather 2 readers x 2 floats per voice and sample, every
table op 2 floats; it is an upper bound (silent readers load nothing).  With --opprof the specialised kernel is compiled with the
per-opcode cycle counters (engine option spec_opprof, as tools/spec_opprof.py) and the SAMPLE / TABLE share of the sample loop is
printed.  One JSON line per (arm, voices); the card's name and power limit are read in the same run.
Usage: python tools/sample_bench.py [--voices 4096,131072] [--blocks 200] [--warmup 20] [--opprof]"""
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

SR, BS, N_RES = 48000.0, 512, 64
OP_TABLE, OP_SAMPLE, LOOP = 23, 43, 63


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build(arm, n, opprof, device=0):
    opts = dict(specialize=2, specialize_strict=1)
    if opprof:
        opts["spec_opprof"] = 1
    rt = Runtime(SR, BS, n, device=device, **opts)
    rng = np.random.default_rng(1)
    names = [f"res{k}" for k in range(N_RES)]
    for k, nm in enumerate(names):
        assert rt.add_shared_resource(nm, rng.standard_normal(int(SR)).astype(np.float32))
    if arm == "sample":
        node = el.sample({"key": "smp", "path": names[0], "mode": "trigger"},
                         el.le(el.phasor(el.const(2.0, key="tf")), 0.5), el.const(1.0, key="rate"))
        assert rt.apply_instructions(el.render(node)) == 0, rt.last_error()
        v = np.arange(n)
        assert rt.set_property_per_voice(el.const(0, key="tf").id(), "value", 1.0 + (v % 13) * 0.37) == 0
        assert rt.set_property_per_voice(el.const(0, key="rate").id(), "value", 0.5 + (v % 17) * 0.09) == 0
        assert rt.set_path_per_voice(node.id(), names, v % N_RES) == 0, rt.last_error()
    else:
        node = el.table({"key": "tab", "path": names[0]}, el.phasor(el.const(2.0, key="tf")))
        assert rt.apply_instructions(el.render(node)) == 0, rt.last_error()
        assert rt.set_property_per_voice(el.const(0, key="tf").id(), "value", 1.0 + (np.arange(n) % 13) * 0.37) == 0
    return rt


def gather_bytes(rt, n):
    words, pc, ops = rt.program_words(0), 0, []
    while pc < len(words):
        w0 = int(words[pc])
        if w0 & 0xFF == 0:
            break
        ops.append(w0 & 0xFF)
        pc += 8 + ((w0 >> 8) & 0xFF)
    return n * BS * (16 * ops.count(OP_SAMPLE) + 8 * ops.count(OP_TABLE))


def run(arm, n, blocks, warmup, opprof):
    rt = build(arm, n, opprof)
    for _ in range(warmup):
        rt.enqueue_block(0, 1, BS, FLAG_MIX)
    rt.synchronize()
    g = rt.describe()["groups"][0]
    assert g.get("spec_state") == 2, g
    if opprof:
        rt.debug_opprof(True)
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
    res = {"arm": arm, "voices": n, "tile_width": g["tile_width"], "spec_regs": g.get("spec_regs"), "blocks": blocks,
           "ms_per_block": wall, "k1_ms_per_block": k1_ms / blocks, "k1_launches": k1_n,
           "gather_bytes_per_block": gather_bytes(rt, n), "opprof": bool(opprof)}
    if opprof:
        p = rt.debug_opprof(True).astype(np.float64).reshape(64, 2)
        res["op_share_of_loop"] = {"SAMPLE": p[OP_SAMPLE, 0] / max(1.0, p[LOOP, 0]), "TABLE": p[OP_TABLE, 0] / max(1.0, p[LOOP, 0])}   # both passes
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", default="4096,131072")
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--opprof", action="store_true")
    a = ap.parse_args()
    gpu = card()
    for n in (int(x) for x in a.voices.split(",")):
        for arm in ("sample", "table"):
            r = run(arm, n, a.blocks, a.warmup, False)
            if a.opprof:
                r["op_share_of_loop"] = run(arm, n, max(10, a.blocks // 10), a.warmup, True)["op_share_of_loop"]
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
