#!/usr/bin/env python
"""Offline rendering with every block's events (elem_b200_process_offline_events) against the same render without events and against
a process() + process_queued_events() loop, on cuda:0.  Prints one JSON line; the card's name and power limit are read in the same run.

  (a) 4096 SUBSYNTH32 voices, each under a `meter`, mix only: three legs — offline with events, offline without, the poll-per-block loop.
  (b) the `analysis` node family of tests/k1_families.py (meter, snapshot, scope, capture, fft) at 1024 voices: offline with and without
      events, and the loop.
Time per block is the host clock around each call (every call ends with its outputs and events on the host).  For the event legs it is
split into the time spent inside the user's callback (JSON parsing into dicts included) and the rest (render, log copies, formatting).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from elementary_b200 import Runtime, el, graphs  # noqa: E402

SR, BS = 48000.0, 512


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return out.strip().splitlines()[0]
    except Exception as exc:   # noqa: BLE001
        return f"unknown ({exc})"


def subsynth_meter(n_voices):
    rt = Runtime(SR, BS, n_voices, device=0)
    assert rt.apply_instructions(el.render(el.meter({"name": "v"}, graphs.subsynth32_graph()))) == 0
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(n_voices)])
    assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    return rt, None, 1


def analysis(n_voices):
    from k1_families import FAMILIES
    fam = FAMILIES["analysis"]
    rt = Runtime(SR, BS, n_voices, device=0)
    assert rt.apply_instructions(fam.batch) == 0
    fam.setup(rt)
    rng = np.random.RandomState(1)
    return rt, rng, fam.n_out


def legs(make, n_voices, blocks, warmup):
    rt, rng, n_out = make(n_voices)
    n_in = 2 if rng is not None else 0
    n = blocks * BS
    x = (rng.rand(n_in, n).astype(np.float32) * 2 - 1) if n_in else None
    xb = (rng.rand(n_in, BS).astype(np.float32) * 2 - 1) if n_in else None
    res = {}
    kw = dict(inputs=x, num_outputs=n_out, num_samples=n) if n_in else dict(num_outputs=n_out, num_samples=n)
    # warm-up of every leg's shapes
    rt.process_offline(**dict(kw, num_samples=warmup * BS, inputs=None if x is None else x[:, :warmup * BS]), on_event=lambda *a: None)
    rt.process_offline(**dict(kw, num_samples=warmup * BS, inputs=None if x is None else x[:, :warmup * BS]))
    for _ in range(warmup):
        rt.process(xb, n_out, BS)
        rt.process_queued_events()

    cb_s = [0.0]
    count = [0]

    def on_event(k, t, e):
        count[0] += 1

    # the host's share: the wrapper's callback (JSON text -> dict, then on_event), timed around each call from the library
    import elementary_b200.runtime as rtmod
    orig = rtmod.BLOCK_EVENT_CB

    def timed_cb_type(fn):
        def wrap(*a):
            t0 = time.perf_counter()
            fn(*a)
            cb_s[0] += time.perf_counter() - t0
        return orig(wrap)
    rtmod.BLOCK_EVENT_CB = timed_cb_type
    try:
        t0 = time.perf_counter()
        rt.process_offline(**kw, on_event=on_event)
        dt = time.perf_counter() - t0
    finally:
        rtmod.BLOCK_EVENT_CB = orig
    res["offline_events_ms_per_block"] = 1e3 * dt / blocks
    res["offline_events_callback_ms_per_block"] = 1e3 * cb_s[0] / blocks
    res["offline_events_render_ms_per_block"] = 1e3 * (dt - cb_s[0]) / blocks
    res["events"] = count[0]

    t0 = time.perf_counter()
    rt.process_offline(**kw)
    res["offline_ms_per_block"] = 1e3 * (time.perf_counter() - t0) / blocks

    cb_s[0] = 0.0
    polled = 0
    t0 = time.perf_counter()
    for k in range(blocks):
        rt.process(None if x is None else x[:, k * BS:(k + 1) * BS], n_out, BS)
        p0 = time.perf_counter()
        polled += len(rt.process_queued_events())
        cb_s[0] += time.perf_counter() - p0
    dt = time.perf_counter() - t0
    res["loop_ms_per_block"] = 1e3 * dt / blocks
    res["loop_poll_ms_per_block"] = 1e3 * cb_s[0] / blocks
    res["loop_events"] = polled
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--voices-a", type=int, default=4096)
    ap.add_argument("--voices-b", type=int, default=1024)
    ap.add_argument("--blocks-b", type=int, default=1024, help="blocks of (b), whose events (scope / capture windows, fft spectra) are host-bound")
    args = ap.parse_args()
    out = {"gpu": gpu_info(), "block_size": BS,
           "a_subsynth32_meter": dict(voices=args.voices_a, blocks=args.blocks, **legs(subsynth_meter, args.voices_a, args.blocks, args.warmup)),
           "b_analysis": dict(voices=args.voices_b, blocks=args.blocks_b, **legs(analysis, args.voices_b, args.blocks_b, args.warmup))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
