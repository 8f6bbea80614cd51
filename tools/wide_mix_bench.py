"""Cost of the wide mix bus (nOut > 8, K2w) against the same graphs mixed into one channel (K2).  Prints one JSON line.

  (a) config 5's 1250 random graphs, one per voice: graph i on channel i (nOut = 1250, 1250 stems) vs all on channel 0 (nOut = 1)
  (b) 4096 SUBSYNTH32 voices in 16 voice groups of 256: group i on channel i (nOut = 16) vs all on channel 0 (nOut = 1)
  (c) one dense channel: 131072 SUBSYNTH32 voices at tile width 1 on channel 0, mixed with nOut = 9 (K2w) vs nOut = 1 (K2)

Per arm: ms per block of enqueue_block(mix) back to back (CUDA events around the timed loop), then a second pass with per-kernel event
pairs for the K1 and mix-reduction (K2 or K2w) device times.  K2w's bytes/s counts the rows it reads, sum_c |R_c| * numSamples * 4.

usage: python tools/wide_mix_bench.py [--steps 200] [--warmup 20]
"""
import argparse
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR, BS = 48000.0, 512


def aim(batch, channel):
    b = copy.deepcopy(batch)
    roots = next(ins for ins in b if ins[0] == 4)[1]
    for ins in b:
        if ins[0] == 3 and ins[2] == "channel" and ins[1] in roots:
            ins[3] = int(channel)
    return b


def workload(name, stems):
    import numpy as np
    from elementary_b200 import Runtime, graphs
    if name == "a":
        n = 1250
        rt = Runtime(SR, BS, n, device=0)
        for i in range(n):
            assert rt.apply_instructions(aim(graphs.random_graph(i, 64), i if stems else 0), voices=(i, i + 1)) == 0, rt.last_error()
        return rt, (n if stems else 1)
    if name == "c":
        rt = Runtime(SR, BS, 131072, device=0, tile_width=1)
        assert rt.apply_instructions(graphs.subsynth32()) == 0, rt.last_error()
        return rt, (9 if stems else 1)
    rt = Runtime(SR, BS, 4096, device=0)
    for i in range(16):
        assert rt.apply_instructions(aim(graphs.subsynth32(), i if stems else 0), voices=(256 * i, 256 * (i + 1))) == 0, rt.last_error()
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(4096)])
    assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    return rt, (16 if stems else 1)


def measure(rt, n_out, steps, warmup):
    import torch
    from elementary_b200.runtime import FLAG_MIX
    for _ in range(warmup):
        rt.enqueue_block(0, n_out, BS, FLAG_MIX)
    rt.synchronize()
    stream = torch.cuda.Stream()
    rt.set_stream(stream.cuda_stream)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for _ in range(steps):
        rt.enqueue_block(0, n_out, BS, FLAG_MIX)
    t1.record(stream)
    t1.synchronize()
    ms = t0.elapsed_time(t1) / steps
    rt.set_option("time_kernels", 1)
    rt.take_kernel_time_ms()
    for _ in range(steps):
        rt.enqueue_block(0, n_out, BS, FLAG_MIX)
    rt.take_kernel_time_ms()
    kinds = rt.last_kernel_times()
    rt.set_option("time_kernels", 0)
    groups = rt.describe()["groups"]
    if n_out > 8:
        rows = sum(((g["nv"] + g["tile_width"] - 1) // g["tile_width"]) * len([c for c in g.get("mix_channels", []) if c < n_out])
                   for g in groups if g["tile_width"])
    else:
        rows = sum((g["nv"] + g["tile_width"] - 1) // g["tile_width"] for g in groups if g["tile_width"]) * n_out
    mix_ms = kinds["K2"][0] / max(1, kinds["K2"][1])
    return {"n_out": n_out, "groups": len(groups), "ms_per_block": ms, "k1_ms": kinds["K1"][0] / steps,
            ("k2w_ms" if n_out > 8 else "k2_ms"): mix_ms, "partial_rows": rows,
            "mix_gbytes_per_s": rows * BS * 4 / (mix_ms * 1e-3) / 1e9 if mix_ms > 0 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    sys.path.insert(0, ROOT)
    from bench import gpu_description
    out = {"gpu": gpu_description(0), "block_size": BS}
    for name in ("a", "b", "c"):
        for stems in (True, False):
            rt, n_out = workload(name, stems)
            label = ("nout9" if stems else "nout1") if name == "c" else ("stems" if stems else "channel0")
            out[f"{name}_{label}"] = measure(rt, n_out, args.steps, args.warmup)
            del rt
            torch.cuda.synchronize()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
