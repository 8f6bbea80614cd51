"""Canonical benchmark / parity graphs (SURVEY.md §8(d)), expressed with :mod:`elementary_b200.el`.

Every constant that varies per voice carries a ``key`` so that its node id is stable and a per-voice
``[3, id, "value", x]`` SET_PROPERTY batch can address it (this is how the reference's ``createRef`` /
keyed consts work: js/packages/core/index.ts:177-199).
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

from . import el


def _k(value: float, key: str) -> el.Node:
    return el.const(value, key=key)


# --- config 1: plumbing graph of cli/Benchmark (saw -> svf -> mul, two roots) ---------------------------------
def plumbing() -> List[list]:
    saw = el.sub(el.mul(_k(2, "two"), el.phasor(_k(110, "f"))), _k(1, "one"))
    flt = el.svf({"mode": "lowpass"}, _k(800, "fc"), _k(1, "q"), saw)
    out = el.mul(_k(0.5, "g"), flt)
    return el.render(out, out)


# --- config 2: SUBSYNTH32 -------------------------------------------------------------------------------------
def subsynth32_f0(voice: int) -> float:
    return 55.0 * (1 + voice % 40)


def subsynth32_graph(f0: float = 110.0) -> el.Node:
    two, one = _k(2, "two"), _k(1, "one")
    saw1 = el.sub(el.mul(two, el.phasor(_k(f0, "f0a"))), one)
    saw2 = el.sub(el.mul(two, el.phasor(_k(f0 * 1.007, "f0b"))), one)
    mix = el.mul(_k(0.5, "mixg"), el.add(saw1, saw2))
    lfo = el.sin(el.mul(_k(2.0 * math.pi, "twopi"), el.phasor(_k(0.5, "lforate"))))
    fc = el.add(_k(1200, "fcbase"), el.mul(_k(800, "fcdepth"), lfo))
    flt = el.svf({"mode": "lowpass"}, fc, _k(1.5, "q"), mix)
    sat = el.tanh(el.mul(_k(2, "drive"), flt))
    dly = el.delay({"size": 4800}, _k(3001.5, "dlen"), _k(0.35, "dfb"), sat)
    return el.add(sat, dly)


def subsynth32(f0: float = 110.0) -> List[list]:
    """32-node subtractive voice (31 + root), one output channel."""
    return el.render(subsynth32_graph(f0))


def subsynth32_voice_props(voice: int) -> List[list]:
    """Per-voice SET_PROPERTY batch: f0 = 55*(1 + v mod 40) Hz, second saw detuned by 1.007."""
    f0 = subsynth32_f0(voice)
    return [[3, _k(0, "f0a").id(), "value", f0], [3, _k(0, "f0b").id(), "value", f0 * 1.007]]


def subsynth32_param_ids() -> Tuple[int, int]:
    return _k(0, "f0a").id(), _k(0, "f0b").id()


# --- config 3: additive-64 ------------------------------------------------------------------------------------
def additive64_f0(voice: int) -> float:
    return 55.0 * 2.0 ** ((voice % 48) / 12.0)


def additive64_graph(f0: float = 110.0, partials: int = 64) -> el.Node:
    twopi = _k(2.0 * math.pi, "twopi")
    terms = []
    for p in range(1, partials + 1):
        osc = el.sin(el.mul(twopi, el.phasor(_k(f0 * p, f"f{p}"))))
        terms.append(el.mul(_k(1.0 / p, f"a{p}"), osc))
    return el.add(*terms)


def additive64(f0: float = 110.0, partials: int = 64) -> List[list]:
    return el.render(additive64_graph(f0, partials))


def additive64_voice_props(voice: int, partials: int = 64) -> List[list]:
    f0 = additive64_f0(voice)
    return [[3, _k(0, f"f{p}").id(), "value", f0 * p] for p in range(1, partials + 1)]


# --- config 4: convolution reverb channel -----------------------------------------------------------------------
def convolve_channel(path: str = "ir") -> List[list]:
    return el.render(el.convolve({"path": path}, el.in_(0)))


def lcg_ir(taps: int = 16384, seed: int = 1) -> "list[float]":
    """16384-tap decaying-noise IR: s = s*1664525 + 1013904223 (s0 = seed), x = ((s>>8)/2^24 - 0.5)*0.01*exp(-6 n/N).

    The generator states come from a prefix scan of the affine maps s -> a*s + c (log2(taps) numpy steps, arithmetic mod 2^64,
    which is exact mod 2^32), so a thousand IRs take milliseconds each; the values are those of the plain sequential loop."""
    import numpy as np
    if taps <= 0:
        return []
    mask = np.uint64(0xFFFFFFFF)
    A = np.full(taps, 1664525, dtype=np.uint64)          # after round k, entry i maps s0 to s_{min(i+1, 2k)}
    C = np.full(taps, 1013904223, dtype=np.uint64)
    k = 1
    while k < taps:
        ak, ck = A[k - 1], C[k - 1]
        A[k:], C[k:] = (A[:-k] * ak) & mask, (C[:-k] * ak + ck) & mask
        k *= 2
    s = (A * np.uint64(seed & 0xFFFFFFFF) + C) & mask
    x = ((s >> np.uint64(8)).astype(np.float64) / float(1 << 24) - 0.5) * 0.01
    env = np.array([math.exp(-6.0 * n / taps) for n in range(taps)])   # math.exp: the same bits as the loop it replaces
    return (x * env).tolist()


# --- config 5: random 64-node graphs ----------------------------------------------------------------------------
class _Lcg:
    def __init__(self, seed: int):
        self.s = (seed * 2654435761 + 12345) & 0xFFFFFFFF

    def next(self) -> int:
        self.s = (self.s * 1664525 + 1013904223) & 0xFFFFFFFF
        return self.s >> 8

    def uniform(self, lo: float, hi: float) -> float:
        return lo + (hi - lo) * (self.next() / float(1 << 24))

    def pick(self, seq):
        return seq[self.next() % len(seq)]


def random_graph(seed: int, nodes: int = 64) -> List[list]:
    """Deterministic random DAG over the star-marked builtin set (SURVEY.md §8d config 5).

    Children are always chosen among earlier nodes so the graph is a DAG by construction; filters get stable
    coefficients; ``rand`` always gets an explicit seed (Noise.h:42 would otherwise call std::rand()).
    """
    r = _Lcg(seed)
    pool: List[el.Node] = []
    uid = [0]

    def kconst(v: float) -> el.Node:
        uid[0] += 1
        return el.const(v, key=f"g{seed}c{uid[0]}")

    # a few signal sources first
    pool.append(el.phasor(kconst(r.uniform(20.0, 2000.0))))
    pool.append(el.sin(el.mul(kconst(2.0 * math.pi), el.phasor(kconst(r.uniform(0.1, 20.0))))))
    uid[0] += 1
    pool.append(el.sub(el.mul(kconst(2.0), el.rand(seed=(seed * 7919 + uid[0]) & 0x7FFFFFFF, key=f"g{seed}r{uid[0]}")), kconst(1.0)))

    def reachable(n: el.Node, seen: set) -> None:
        if n.id() in seen:
            return
        seen.add(n.id())
        for c in n.children:
            reachable(c, seen)

    def output_graph() -> el.Node:
        return el.tanh(el.mul(kconst(0.25), el.add(*pool[-4:])))

    ops = ["sin", "tanh", "add", "sub", "mul", "min", "max", "pole", "svf", "biquad", "z", "sdelay", "delay",
           "phasor", "rand", "abs", "mm1p"]
    while True:
        seen: set = set()
        saved = uid[0]
        reachable(output_graph(), seen)
        uid[0] = saved                      # the probe must not consume const keys
        if len(seen) + 1 >= nodes:          # + the root
            break
        op = r.pick(ops)
        a = r.pick(pool)
        b = r.pick(pool)
        if op == "sin":
            n = el.sin(el.mul(kconst(r.uniform(0.5, 3.0)), a))
        elif op == "tanh":
            n = el.tanh(el.mul(kconst(r.uniform(0.5, 4.0)), a))
        elif op == "abs":
            n = el.abs_(a)
        elif op in ("add", "sub", "mul", "min", "max"):
            n = getattr(el, op if op not in ("min", "max") else op + "_")(a, b)
        elif op == "pole":
            n = el.pole(kconst(r.uniform(-0.95, 0.95)), a)
        elif op == "svf":
            mode = r.pick(["lowpass", "bandpass", "highpass", "notch", "allpass"])
            n = el.svf({"mode": mode}, kconst(r.uniform(100.0, 8000.0)), kconst(r.uniform(0.5, 4.0)), a)
        elif op == "mm1p":
            mode = r.pick(["lowpass", "highpass", "allpass"])
            n = el.mm1p({"mode": mode}, el.prewarp(kconst(r.uniform(100.0, 8000.0))), a)
        elif op == "biquad":
            # stable low-pass-ish biquad: poles inside the unit circle
            rad, th = r.uniform(0.3, 0.95), r.uniform(0.05, 2.5)
            a1, a2 = -2.0 * rad * math.cos(th), rad * rad
            n = el.biquad(kconst(0.25), kconst(0.5), kconst(0.25), kconst(a1), kconst(a2), a)
        elif op == "z":
            n = el.z(a)
        elif op == "sdelay":
            n = el.sdelay({"size": int(r.uniform(1, 2000))}, a)
        elif op == "delay":
            size = int(r.uniform(64, 4000))
            n = el.delay({"size": size}, kconst(r.uniform(1.0, size - 1.0)), kconst(r.uniform(0.0, 0.5)), a)
        elif op == "phasor":
            n = el.phasor(kconst(r.uniform(20.0, 4000.0)))
        else:  # rand
            uid[0] += 1
            n = el.rand(seed=(seed * 104729 + uid[0]) & 0x7FFFFFFF, key=f"g{seed}r{uid[0]}")
        pool.append(n)

    return el.render(output_graph())
