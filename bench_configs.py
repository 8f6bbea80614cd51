#!/usr/bin/env python
"""Secondary measurements for the other BASELINE.json configs (not the driver's headline; bench.py is).

  config 1: the reference's own elembench (cli/Benchmark.cpp, unmodified) on the plumbing graph, against both engines
  config 3: additive synth, 64 el.cycle partials per voice (387 nodes)          — K1, many recurrences per voice
  config 4: el.convolve reverb, 16384-tap IR, one channel per voice             — K3 (partitioned FFT convolver)
  config 4v: the same with a different 16384-tap IR on every channel           — K3, per-channel-IR form (not in the default set)
  config 5: independent random 64-node graphs, one voice group each             — K1, one launch per graph

Each prints one JSON line: device-resident ms/block (CUDA events), Msamples/s, x real time, the kernel time measured
with events around the K1/K3 launches, the algorithmic-bytes roofline fraction and a CPU reference sample
(unmodified reference via oracle/_ref on all host threads).  Usage: python bench_configs.py [1] [3] [4] [4v] [5] [--quick]
"""
from __future__ import annotations

import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SR, BS = 48000.0, 512


def hbm_peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0      # H100 SXM data sheet


def timed_blocks(rt, n_in, flags, steps, warmup):
    import torch
    for _ in range(warmup):
        rt.enqueue_block(n_in, 1, BS, flags)
    rt.synchronize()
    rt.take_kernel_time_ms()
    l0 = rt.kernel_launches
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    total = 0.0
    for _ in range(steps):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rt.enqueue_block(n_in, 1, BS, flags)
        rt.synchronize()
        total += time.perf_counter() - t0
    k1_ms, k1_n = rt.take_kernel_time_ms()
    k3_ms, k3_n = rt.last_convolve_time_ms()
    return total / steps * 1e3, k1_ms / max(1, steps), k3_ms / max(1, steps), (rt.kernel_launches - l0) // steps


def cpu_ref(batch, voice_batches, voices, blocks, n_in=0, resource=None, inputs=None):
    from oracle import oracle as orc
    if not orc.ref_available():
        return None
    from bench import host_description
    cores = host_description()["threads_used"]
    secs, _, nb = orc.ref_bench(SR, BS, batch, voice_batches, voices, cores, n_in, 1, 3, blocks, resource=resource, inputs=inputs, min_seconds=3.0)
    return {"msamples_per_s": voices * BS * nb / secs / 1e6, "cores": cores, "sample": f"{voices} voices x {nb:.0f} blocks, {secs:.1f} s, pinned threads"}


def config1(quick):
    """BASELINE config 1: the reference's own benchmark program (cli/Benchmark.cpp + cli/BenchmarkMain.cpp, compiled unmodified by
    oracle/Makefile) on the plumbing graph — once against the reference runtime (host CPU), once against the source-compatible
    elem::Runtime of include/elem_b200_compat over libelem_b200.so (one voice on the GPU: pure plumbing / launch latency)."""
    import re, subprocess
    js = os.path.join(ROOT, "oracle", "config1_plumbing.js")
    out = {"config": "1: cli/Benchmark (elembench) on the saw->svf->mul plumbing graph, 44.1 kHz, 512-sample blocks, 10000 iterations, float then double"}
    for name, exe, env in (("reference", "elembench_ref", {}),
                           ("b200_1_voice", "elembench_b200", {"ELEM_B200_VOICES": "1", "ELEM_B200_SPECIALIZE": "2"}),
                           ("b200_4096_voices", "elembench_b200", {"ELEM_B200_VOICES": "4096", "ELEM_B200_SPECIALIZE": "2"})):
        path = os.path.join(ROOT, "oracle", "_ref", exe)
        if not os.path.exists(path):
            out[name] = {"unavailable": f"{path} missing (built only where /root/reference exists)"}
            continue
        p = subprocess.run([path, js], capture_output=True, text=True, env=dict(os.environ, **env), timeout=600)
        avg = [float(x) for x in re.findall(r"Average iteration time: ([0-9.eE+-]+)us", p.stdout)]
        if p.returncode != 0 or len(avg) < 2:
            out[name] = {"failed": p.returncode, "stderr": p.stderr[-500:], "stdout": p.stdout[-300:]}
            continue
        voices = int(env.get("ELEM_B200_VOICES", "1"))
        out[name] = {"float_us_per_block": avg[0], "double_us_per_block": avg[1], "voices": voices,
                     "msamples_per_s_float": voices * 512 / avg[0], "note": "the program's own report: mean of 10000 per-iteration times truncated to integer microseconds (Benchmark.cpp:99)"}
    return out


def config3(quick, steps=None):
    from elementary_b200 import Runtime, graphs
    from elementary_b200.runtime import FLAG_MIX
    voices = 8192                      # 65536 voices / 8 GPUs
    rt = Runtime(SR, BS, voices, device=0, time_kernels=1)
    assert rt.apply_instructions(graphs.additive64()) == 0, rt.last_error()
    f0 = np.array([graphs.additive64_f0(v) for v in range(voices)])
    from elementary_b200 import el
    for p in range(1, 65):
        assert rt.set_property_per_voice(el.const(0, key=f"f{p}").id(), "value", f0 * p) == 0
    ms, k1, k3, launches = timed_blocks(rt, 0, FLAG_MIX, steps or (10 if quick else 40), 5)
    algo = 1028 * voices               # SURVEY.md §8d: 512 B state R+W + 516 B params (mix-only)
    d = rt.describe()["groups"][0]
    cpu = cpu_ref(graphs.additive64(), [graphs.additive64_voice_props(v) for v in range(256)], 256, 20 if quick else 60)
    return {"config": "3: additive-64 (387-node voice), 8192 voices per GPU (65536 over 8)", "ms_per_block": ms, "k1_ms": k1,
            "msamples_per_s": voices * BS / ms / 1e3, "realtime_x": voices * BS / (ms * 1e-3) / (voices * SR),
            "roofline": {"bound": "hbm", "achieved_gbs": algo / (k1 * 1e-3) / 1e9, "peak_gbs": hbm_peak(), "frac": algo / (k1 * 1e-3) / 1e9 / hbm_peak()},
            "program": d, "launches_per_block": launches, "cpu_reference": cpu}


def config4(quick, steps=None):
    import torch
    from elementary_b200 import Runtime, graphs
    from elementary_b200.runtime import FLAG_MIX, FLAG_VOICE_IN
    channels = 1024
    ir = np.asarray(graphs.lcg_ir(16384), dtype=np.float32)
    rt = Runtime(SR, BS, channels, device=0, time_kernels=1)
    assert rt.add_shared_resource("ir", ir)
    assert rt.apply_instructions(graphs.convolve_channel("ir")) == 0, rt.last_error()
    x = torch.as_tensor(rt.voice_in_device(1), device="cuda")
    x.copy_((torch.rand(x.shape, device="cuda") - 0.5) * 0.5)      # device-resident noise, one channel per voice
    ms, k1, k3, launches = timed_blocks(rt, 1, FLAG_MIX | FLAG_VOICE_IN, steps or (10 if quick else 60), 40)   # warm-up fills the 32-block delay line
    S = 32
    algo = (2 * 512 * 4 + (S - 1) * 513 * 8 + 513 * 8 + 2 * 512 * 4) * channels     # convolve.h
    rng = np.random.RandomState(0)
    cpu = cpu_ref(graphs.convolve_channel("ir"), None, 256, 16 if quick else 64, n_in=1, resource=("ir", ir),
                  inputs=((rng.rand(1, BS) - 0.5) * 0.5).astype(np.float32))
    return {"config": "4: el.convolve 16384-tap IR, 1024 channels on one GPU", "ms_per_block": ms, "k1_ms": k1, "k3_ms": k3,
            "msamples_per_s": channels * BS / ms / 1e3, "realtime_x": BS / (ms * 1e-3) / SR,
            "roofline": {"bound": "hbm", "kernel": "convolve_chunk_kernel", "achieved_gbs": algo / (k3 * 1e-3) / 1e9, "peak_gbs": hbm_peak(),
                         "frac": algo / (k3 * 1e-3) / 1e9 / hbm_peak(), "algorithmic_bytes_per_channel_block": algo // channels},
            "launches_per_block": launches, "cpu_reference": cpu}


def config4v(quick, steps=None):
    """BASELINE config 4's per-channel-IR variant: 1024 channels, each with its own 16384-tap IR (Runtime.set_path_per_voice: one
    voice group, the per-channel form of K3), parity of 8 sampled channels against the reference over 40 blocks, and for contrast
    the same workload at 128 channels through per-voice JSON `path` batches (every voice its own group and K3 launch)."""
    import torch
    from bench import gpu_description
    from oracle import oracle as orc
    from elementary_b200 import Runtime, el, graphs
    from elementary_b200.runtime import FLAG_MIX, FLAG_VOICE_IN
    channels = 1024
    t0 = time.perf_counter()
    irs = [np.asarray(graphs.lcg_ir(16384, seed=c + 1), dtype=np.float32) for c in range(channels)]
    gen_s = time.perf_counter() - t0
    names = [f"ir{c}" for c in range(channels)]
    cv = el.convolve({"path": names[0], "key": "cv"}, el.in_(0))
    batch = el.render(cv)
    t0 = time.perf_counter()
    rt = Runtime(SR, BS, channels, device=0, time_kernels=1)
    for nm, ir in zip(names, irs):
        assert rt.add_shared_resource(nm, ir)
    assert rt.apply_instructions(batch) == 0, rt.last_error()
    assert rt.set_path_per_voice(cv.id(), names, np.arange(channels)) == 0, rt.last_error()
    rt.synchronize()
    setup_s = time.perf_counter() - t0
    desc = rt.describe()
    assert len(desc["groups"]) == 1 and desc["groups"][0]["convolvers"][0]["form"] == "per_channel"

    # parity first (host I/O, 40 blocks from silence), then a fresh runtime for the device-resident timing
    nb = 40
    sample = np.random.RandomState(1).choice(channels, size=8, replace=False)
    x = ((np.random.RandomState(2).rand(channels, 1, nb * BS) - 0.5) * 0.5).astype(np.float32)
    got, _ = rt.render_voices(nb, 1, x)
    parity = {"available": orc.ref_available(), "channels": [int(c) for c in sample], "blocks": nb}
    if orc.ref_available():
        worst = 0.0
        for c in sample:
            o = orc.RefRuntime(SR, BS)
            assert o.add_shared_resource(names[c], irs[c]) and o.apply(el.render(el.convolve({"path": names[c], "key": "cv"}, el.in_(0)))) == 0
            ref = o.render(nb, 1, BS, x[c])
            worst = max(worst, float(np.abs(got[c].astype(np.float64) - ref).max() / np.abs(ref).max()))
        parity.update({"worst_err_over_peak": worst, "ok": worst <= 1e-5})
    del rt

    rt = Runtime(SR, BS, channels, device=0, time_kernels=1)
    for nm, ir in zip(names, irs):
        rt.add_shared_resource(nm, ir)
    assert rt.apply_instructions(batch) == 0 and rt.set_path_per_voice(cv.id(), names, np.arange(channels)) == 0
    xd = torch.as_tensor(rt.voice_in_device(1), device="cuda")
    xd.copy_((torch.rand(xd.shape, device="cuda") - 0.5) * 0.5)
    ms, k1, k3, launches = timed_blocks(rt, 1, FLAG_MIX | FLAG_VOICE_IN, steps or (10 if quick else 60), 40)
    S = 32
    today = 2 * 512 * 4 + (S - 1) * 513 * 8 + 513 * 8 + 2 * 512 * 4          # config 4's formula
    algo = (today + S * 4096) * channels                                      # + every channel's own IR spectra (no unit shares an IR)
    del rt

    # contrast: per-voice JSON `path` batches cut the group into one group (one K3 launch) per voice
    n_json = 128
    t0 = time.perf_counter()
    rj = Runtime(SR, BS, n_json, device=0, time_kernels=1)
    for nm, ir in zip(names[:n_json], irs[:n_json]):
        rj.add_shared_resource(nm, ir)
    assert rj.apply_instructions(batch) == 0
    for v in range(1, n_json):
        assert rj.apply_instructions([[3, cv.id(), "path", names[v]]], voices=(v, v + 1)) == 0, rj.last_error()
    rj.synchronize()
    json_setup_s = time.perf_counter() - t0
    xj = torch.as_tensor(rj.voice_in_device(1), device="cuda")
    xj.copy_((torch.rand(xj.shape, device="cuda") - 0.5) * 0.5)
    jms, _, jk3, jl = timed_blocks(rj, 1, FLAG_MIX | FLAG_VOICE_IN, steps or (10 if quick else 30), 40)
    contrast = {"channels": n_json, "groups": len(rj.describe()["groups"]), "ms_per_block": jms, "k3_ms": jk3, "launches_per_block": jl,
                "setup_s": json_setup_s}
    del rj
    return {"config": "4v: el.convolve, 1024 channels each with its own 16384-tap IR (set_path_per_voice), one GPU",
            "ms_per_block": ms, "k1_ms": k1, "k3_ms": k3, "launches_per_block": launches,
            "setup_s": setup_s, "ir_generation_s": gen_s,
            "roofline": {"bound": "hbm", "kernel": "convolve_chunk_tm_kernel<per-channel>", "achieved_gbs": algo / (k3 * 1e-3) / 1e9,
                         "peak_gbs": hbm_peak(), "frac": algo / (k3 * 1e-3) / 1e9 / hbm_peak(), "algorithmic_bytes_per_channel_block": algo // channels},
            "gpu": gpu_description(0), "parity": parity, "json_per_voice_paths": contrast}


def config5(quick, steps=None):
    from elementary_b200 import Runtime, graphs
    from elementary_b200.runtime import FLAG_MIX
    n_graphs = 200 if quick else 1250   # 10000 graphs / 8 GPUs
    if "--graphs" in sys.argv:
        n_graphs = int(sys.argv[sys.argv.index("--graphs") + 1])
    extra = {}
    if "--stages" in sys.argv:
        extra["pipeline_stages"] = int(sys.argv[sys.argv.index("--stages") + 1])
    if "--niter" in sys.argv:
        extra["niter"] = int(sys.argv[sys.argv.index("--niter") + 1])
    if "--wpc" in sys.argv:
        extra["warps_per_cta"] = int(sys.argv[sys.argv.index("--wpc") + 1])
    rt = Runtime(SR, BS, n_graphs, device=0, time_kernels=1, **extra)
    batches = [graphs.random_graph(i, 64) for i in range(n_graphs)]     # the Python generator is not part of the engine's setup cost
    t0 = time.perf_counter()
    for i, batch in enumerate(batches):
        assert rt.apply_instructions(batch, voices=(i, i + 1)) == 0, rt.last_error()
    build_s = time.perf_counter() - t0
    ms, k1, k3, launches = timed_blocks(rt, 0, FLAG_MIX, steps or (10 if quick else 30), 5)
    # the offline path the config is about: per-graph output, blocks back to back, chunked D2H on a copy stream (host wall clock, D2H included)
    nb_off = 32 if quick else 128
    out = np.empty((n_graphs, 1, nb_off * BS), dtype=np.float32)
    rt.render_offline(8, 1, out=out[:, :, :8 * BS].copy())                      # warm-up (allocations, page faults of the driver)
    t0 = time.perf_counter()
    rt.render_offline(nb_off, 1, out=out)
    off_s = time.perf_counter() - t0
    offline = {"blocks": nb_off, "seconds": off_s, "ms_per_block": off_s / nb_off * 1e3, "msamples_per_s": n_graphs * BS * nb_off / off_s / 1e6,
               "realtime_x": (nb_off * BS / SR) / off_s, "note": "elem_b200_render_offline: per-graph outputs copied to host memory, wall clock"}
    # parity at this scale: a sample of the graphs against the reference over the offline output (blocks after the timed_blocks run are
    # not comparable from block 0, so a fresh small runtime renders the same graphs from the start)
    parity = None
    cpu = None
    from oracle import oracle as orc
    if orc.ref_available():
        chk = Runtime(SR, BS, 16, device=0)
        pick = [int(i * (n_graphs - 1) / 15) for i in range(16)]
        for j, gi in enumerate(pick):
            assert chk.apply_instructions(batches[gi], voices=(j, j + 1)) == 0
        got = chk.render_offline(12, 1)
        worst = 0.0
        for j, gi in enumerate(pick):
            o = orc.RefRuntime(SR, BS); assert o.apply(batches[gi]) == 0
            ref = o.render(12, 1)
            g = got[j, 0].reshape(12, BS).astype(np.float64); r = ref[0].reshape(12, BS).astype(np.float64)
            tol = 1e-5 * np.abs(r).max(axis=1, keepdims=True) + 1e-7
            worst = max(worst, float((np.abs(g - r) / tol).max()))
        parity = {"parity_checked": True, "graphs_checked": pick, "blocks": 12, "worst_err_over_tol": worst}
    if orc.ref_available():
        # CPU: time 64 of the graphs, one Runtime each, on all host threads (distinct graphs => one bench call per graph is
        # too slow to set up; use graph 0..63 sequentially on one thread each via the multi-instance harness per graph)
        cores = os.cpu_count() or 1
        tot = 0.0
        ng = 16
        for i in range(ng):
            secs, _ = orc.ref_bench(SR, BS, graphs.random_graph(i, 64), None, 1, 1, 0, 1, 3, 200)
            tot += secs
        cpu = {"msamples_per_s_per_core": ng * BS * 200 / tot / 1e6, "cores_used": 1, "sample": f"{ng} graphs x 200 blocks, one thread"}
    stages = sorted({g.get("pipeline_stages", 1) for g in rt.describe()["groups"]})
    return {"config": f"5: {n_graphs} independent random 64-node graphs on one GPU (10000 over 8), one voice group each", "pipeline_stages": stages,
            "ms_per_block": ms, "k1_ms_sum": k1, "msamples_per_s": n_graphs * BS / ms / 1e3, "realtime_x": BS / (ms * 1e-3) / SR,
            "launches_per_block": launches, "graph_setup_s": build_s, "offline": offline, "parity": parity, "cpu_reference": cpu}


def main():
    quick = "--quick" in sys.argv
    which = [a for i, a in enumerate(sys.argv[1:], 1) if a in ("1", "3", "4", "4v", "5") and sys.argv[i - 1] not in ("--stages", "--graphs", "--niter", "--wpc")] or ["1", "3", "4", "5"]
    for w in which:
        r = {"1": config1, "3": config3, "4": config4, "4v": config4v, "5": config5}[w](quick)
        print(json.dumps(r))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
