"""The `sample` node scenarios, shared by tests/test_sample_cpu.py (SampleModel against the compiled reference),
tests/test_sample_gpu.py (the GPU against SampleModel, every voice bit for bit) and tests/golden/make_reference_sample.py.

A scenario is a graph (one `sample` node keyed "smp" under root 0), shared resources, per-voice paths and offsets, per-voice host
inputs (trigger in channel 0, rate in channel 1) and events between process() calls.  On the GPU the per-voice props go through
set_path_per_voice / set_property_per_voice, so one voice group holds every voice; each reference instance gets the same props as
[3, id, key, value] batches.  Every run starts with WARM samples of zero inputs, after which root 0 multiplies by exactly 1: output 0
is then the sample node's own output, which SampleModel (a numpy restatement of Sample.h, one lane per voice) computes.

Out of the reference's domain (a read index past the buffer after its one wrap, DESIGN.md section 4) the engine and the model give
0 from that reader where the reference reads out of bounds.  For those scenarios the reference is only ever run up to the sample
before the first such read (`Scenario.ref_prefix`)."""
import ctypes
import hashlib
import math

import numpy as np

from elementary_b200 import el
from k1_families import CALLS, FADE_END, N_VOICES, SR, BS   # noqa: F401  (re-exported for the test modules)
from oracle import oracle as orc

LENGTHS = (1, 2, 7, 13, 1000, 3001)        # 1, 2, non-multiples of 4, longer than a block
UNUSED = "never_played"
N_OUT = 2                                   # output 0: the sample node's root; output 1: a root that live edits and cuts add
WARM = FADE_END                             # zero-input samples before every scenario: the root fade-in is over


def resource(n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32)


def sample_node(mode, rate):
    props = {"key": "smp", "mode": mode}
    if rate == "nochild":
        return el.create_node("sample", props, [])
    trig = el.in_(0)
    if rate == "input":
        return el.sample(props, trig, el.in_(1))
    if rate == "const":
        return el.sample(props, trig, el.const(0.75, key="rate"))
    return el.sample(props, trig)


class Scenario:
    """events: {call index: [event, ...]} applied before that process() call; an event is one of
    ("path", index[v]), ("reset",), ("reset_voices", voices), ("edit", batch), ("cut", first voice, batch), ("prune",)."""

    def __init__(self, name, mode="trigger", rate="input", n_voices=N_VOICES, calls=CALLS, lengths=LENGTHS, offsets="inside",
                 path_at_start=True, events=None, ood=False, seed=0):
        self.name, self.mode, self.rate, self.n_voices, self.calls = name, mode, rate, n_voices, tuple(calls)
        self.offsets, self.path_at_start, self.ood, self.seed = offsets, path_at_start, ood, seed
        self.n_in = {"input": 2, "const": 1, "none": 1, "nochild": 0}[rate]
        self.names = [f"len{n}" for n in lengths]
        self.resources = {nm: resource(n, 1000 + i) for i, (nm, n) in enumerate(zip(self.names, lengths))}
        self.lengths = dict(zip(self.names, lengths))
        self.renderer = el.Renderer()
        self.batch = self.renderer.render(sample_node(mode, rate))
        self.sid = sample_node(mode, rate).id()     # keyed: the same id whatever the props
        rng = np.random.default_rng(7 + seed)
        self.index = rng.integers(0, len(self.names), n_voices) if n_voices > 64 else np.arange(n_voices) % len(self.names)
        self.start, self.stop = np.zeros(n_voices, np.int64), np.zeros(n_voices, np.int64)
        for v in range(n_voices):
            n = self.lengths[self.names[self.index[v]]]
            if offsets == "inside" and v % 3 and n > 0:
                self.start[v] = rng.integers(0, n)
                self.stop[v] = rng.integers(0, n // 2 + 1)
            elif offsets == "stop_past_end":            # size_t wrap of len - stop: the reader runs past the buffer
                self.stop[v] = n + 1 + v % 5
            elif offsets == "start_past_2len":          # loop: the first read is already past the buffer after one wrap
                self.start[v] = 2 * n + v % 3
        self.events = {k: [ev(self) if callable(ev) else ev for ev in evs] for k, evs in (events or {}).items()}

    # ---- inputs ----
    def inputs(self, total):
        """[voice, n_in, total] float32: piecewise-constant triggers (rises that do not start at 0, retriggers closer than the
        10 ms fade, gates), and per voice a constant, fractional, > 1, zero, negative or moving rate."""
        if self.n_in == 0:
            return None
        out = np.zeros((self.n_voices, self.n_in, total), np.float32)
        for v in range(self.n_voices):
            rng = np.random.default_rng((self.seed, v))
            t = int(rng.integers(0, 40))
            level = 0.0
            while t < total:
                seg = int(rng.integers(20, 700))
                level = float(rng.choice([0.0, 0.0, 1.0, 1.0, 0.5, 2.0])) if level != 0.0 or rng.random() < 0.9 else 0.0
                out[v, 0, t:t + seg] = level
                t += seg
            if self.n_in > 1:
                kind = v % 6
                if kind == 5:
                    out[v, 1] = (0.5 + 1.2 * np.sin(np.arange(total) * (0.003 + 0.001 * v))).astype(np.float32)
                else:
                    out[v, 1] = (1.0, 0.37, 2.5, 0.0, -0.8)[kind]
        return out

    def first_rise(self, inputs, v):
        x = inputs[v, 0].astype(np.float64)
        d = np.flatnonzero(np.diff(np.concatenate([[0.0], x])) > 0)
        return int(d[0]) if d.size else None

    def ref_prefix(self, inputs, v):
        """Samples of voice v the reference may render before its first read outside the buffer (None: all of them)."""
        if not self.ood:
            return None
        name = self.names[self.index[v]]
        n = self.lengths[name]
        t0 = self.first_rise(inputs, v)
        if t0 is None:
            return None
        if n == 0:                                # an empty buffer in loop mode: the first tick
            return t0
        if self.offsets == "stop_past_end":       # rate 1 from 0: the right index leaves the buffer at pos = 2 len - 1
            return t0 + 2 * n - 1
        if self.offsets == "start_past_2len":     # the first tick
            return t0
        return None

    # ---- the compiled reference: one instance per voice ----
    def voice_props(self, v, with_path=True):
        b = [[3, self.sid, "path", self.names[self.index[v]]]] if with_path else []
        return b + [[3, self.sid, "startOffset", int(self.start[v])], [3, self.sid, "stopOffset", int(self.stop[v])]]

    def zeros_in(self, n):
        return np.zeros((self.n_in, n), np.float32) if self.n_in else None

    def instance(self, v):
        """A reference instance of voice v after the warm-up: WARM samples of zero inputs, which settle the root fade-in (the
        root then multiplies by exactly 1) and leave the sample node as created (no edge, silent readers)."""
        o = orc.RefRuntime(SR, BS)
        for name, data in self.resources.items():
            assert o.add_shared_resource(name, data)
        assert o.apply(self.batch) == 0
        assert o.apply(self.voice_props(v, self.path_at_start)) == 0
        for _ in range(WARM // BS):
            o.process(self.zeros_in(BS), N_OUT, BS)
        return o

    def reference(self, voices=None, inputs=None):
        """[len(voices), 1, total]: output 0 of one compiled-reference instance per voice, with the scenario's calls and events,
        each voice stopped before its first read outside the buffer (ref_prefix) and padded with NaN."""
        total = sum(self.calls)
        inputs = self.inputs(total) if inputs is None else inputs
        voices = range(self.n_voices) if voices is None else voices
        outs = []
        for v in voices:
            o = self.instance(v)
            limit = self.ref_prefix(inputs, v)
            res = np.full((1, total), np.nan, np.float32)
            s = 0
            for k, n in enumerate(self.calls):
                for ev in self.events.get(k, []):
                    o = self.apply_ref(o, v, ev)
                m = n if limit is None else min(n, limit - s)
                if m <= 0:
                    break
                res[:, s:s + m] = o.process(None if inputs is None else inputs[v, :, s:s + m], N_OUT, m)[:1]
                s += n
            outs.append(res)
        return np.stack(outs), inputs

    def apply_ref(self, o, v, ev):
        kind = ev[0]
        if kind == "path":
            assert o.apply([[3, self.sid, "path", self.names[ev[1][v]]]]) == 0
        elif kind == "reset":
            lib = o.lib                                     # Runtime::reset() of the reference driver
            lib.elem_ref_reset.argtypes = [ctypes.c_void_p]
            lib.elem_ref_reset(o.h)
        elif kind == "reset_voices":
            if v in ev[1]:
                return self.instance(v)
        elif kind == "edit":
            assert o.apply(ev[1]) == 0
        elif kind == "cut":
            if v >= ev[1]:
                assert o.apply(ev[2]) == 0
        return o

    # ---- the model: every voice at once ----
    def model(self, inputs=None):
        """[voice, 1, total]: SampleModel over the scenario's calls and events (no truncation: the model defines what the engine
        does outside the reference's domain)."""
        total = sum(self.calls)
        inputs = self.inputs(total) if inputs is None else inputs
        m = SampleModel(self)
        out = np.zeros((self.n_voices, 1, total), np.float32)
        s = 0
        for k, n in enumerate(self.calls):
            for ev in self.events.get(k, []):
                if ev[0] == "path":
                    m.set_paths(ev[1])
                elif ev[0] == "reset":
                    m.tg[:] = 0.0
                elif ev[0] == "reset_voices":
                    m.reset_voices(ev[1])
            out[:, 0, s:s + n] = m.process(None if inputs is None else inputs[:, :, s:s + n], n)
            s += n
        return out, inputs

    # ---- the GPU side: one runtime, every voice in one group ----
    def setup_gpu(self, rt):
        for name, data in self.resources.items():
            assert rt.add_shared_resource(name, data)
        assert rt.add_shared_resource(UNUSED, np.ones(5, np.float32))
        assert rt.apply_instructions(self.batch) == 0, rt.last_error()
        if self.path_at_start:
            assert rt.set_path_per_voice(self.sid, self.names, self.index) == 0, rt.last_error()
        assert rt.set_property_per_voice(self.sid, "startOffset", self.start.astype(np.float64)) == 0, rt.last_error()
        assert rt.set_property_per_voice(self.sid, "stopOffset", self.stop.astype(np.float64)) == 0, rt.last_error()

    def apply_gpu(self, rt, ev):
        kind = ev[0]
        if kind == "path":
            assert rt.set_path_per_voice(self.sid, self.names, ev[1]) == 0, rt.last_error()
        elif kind == "reset":
            rt.reset()
        elif kind == "reset_voices":
            assert rt.reset_voices(ev[1]) == 0, rt.last_error()
        elif kind == "edit":
            assert rt.apply_instructions(ev[1]) == 0, rt.last_error()
        elif kind == "cut":
            assert rt.apply_instructions(ev[2], (ev[1], self.n_voices)) == 0, rt.last_error()
        elif kind == "prune":
            rt.prune_shared_resources()
            keys = set(rt.get_shared_resource_map_keys())
            assert UNUSED not in keys, keys
            assert set(self.names[i] for i in set(self.index.tolist())) <= keys, keys

    def run_gpu(self, rt, inputs):
        """(per-voice output 0 [voice, 1, total], mix bus channel 0 [1, total]) after the warm-up."""
        for _ in range(WARM // BS):
            rt.process_voices(None if inputs is None else np.zeros((self.n_voices, self.n_in, BS), np.float32), N_OUT, BS)
        vs, ms, s = [], [], 0
        for k, n in enumerate(self.calls):
            for ev in self.events.get(k, []):
                self.apply_gpu(rt, ev)
            v, m = rt.process_voices(None if inputs is None else inputs[:, :, s:s + n], N_OUT, n)
            vs.append(v[:, :1])
            ms.append(m[:1])
            s += n
        return np.concatenate(vs, axis=2), np.concatenate(ms, axis=1)


class SampleModel:
    """Sample.h restated over numpy arrays, one lane per voice, in the reference's float32 / float64 operations and order: the
    edge detector (helpers/Change.h), noteOn / noteOff, and per sample the two VariablePitchLerpReader ticks.  A reader whose read
    index is still past the buffer after its one wrap, or whose position is NaN or not below 2^64, gives 0 for that sample and
    advances as usual (DESIGN.md section 4)."""

    def __init__(self, sc):
        nv = sc.n_voices
        self.sc = sc
        self.alpha = np.float32(1.0 - math.exp(-1.0 / (0.01 * float(np.float32(SR)))))
        parts = [sc.resources[n] for n in sc.names]
        self.flat = np.concatenate(parts + [np.zeros(1, np.float32)])
        self.base_of = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        self.has = np.zeros(nv, bool)
        self.base = np.zeros(nv, np.int64)
        self.len = np.zeros(nv, np.uint64)
        self.start, self.stop = sc.start.astype(np.uint64), sc.stop.astype(np.uint64)
        self.last = np.zeros(nv, np.float32)
        self.cur = np.zeros(nv, np.uint64)
        self.tg, self.g, self.pos = np.zeros((2, nv), np.float32), np.zeros((2, nv), np.float32), np.zeros((2, nv), np.float64)
        if sc.path_at_start:
            self.set_paths(sc.index)

    def set_paths(self, index):          # a new buffer brings two fresh readers; currentReader and lastIn stay
        index = np.asarray(index)
        self.has[:] = True
        self.base = self.base_of[index]
        self.len = np.array([len(self.sc.resources[self.sc.names[i]]) for i in index], np.uint64)
        self.tg[:], self.g[:], self.pos[:] = 0.0, 0.0, 0.0

    def reset_voices(self, voices):
        v = np.asarray(voices)
        self.last[v], self.cur[v] = 0.0, 0
        self.tg[:, v], self.g[:, v], self.pos[:, v] = 0.0, 0.0, 0.0

    def _tick(self, r, rate, act, end, restart, loop):
        p, g, tg = self.pos[r], self.g[r], self.tg[r]
        live = act & ~(p < 0.0) & ~((g == 0.0) & (tg == 0.0))
        past = live & (p >= end)
        if loop:
            p = np.where(past, restart, p)
        else:
            live = live & ~past
        valid = live & (p < 18446744073709551616.0)
        pc = np.where(valid, p, 0.0)
        rl = pc.astype(np.uint64)
        rr = rl + np.uint64(1)
        frac = (pc - rl.astype(np.float64)).astype(np.float32)
        rl = np.where(rl >= self.len, rl - self.len, rl)
        rr = np.where(rr >= self.len, rr - self.len, rr)
        inb = valid & (rl < self.len) & (rr < self.len)
        left = self.flat[np.where(inb, self.base + rl.astype(np.int64), 0)]
        right = self.flat[np.where(inb, self.base + rr.astype(np.int64), 0)]
        y = np.where(inb, g * (left + frac * (right - left)), np.float32(0.0)).astype(np.float32)
        d = tg - g
        ng = np.where(np.abs(d) <= np.finfo(np.float32).eps, tg, g + self.alpha * d).astype(np.float32)
        ng = np.where(ng < 0.0, np.float32(0.0), np.where(np.float32(1.0) < ng, np.float32(1.0), ng))
        self.pos[r] = np.where(live, p + rate.astype(np.float64), self.pos[r])
        self.g[r] = np.where(live, ng, g)
        return y

    def process(self, inputs, n):
        nv = self.sc.n_voices
        if self.sc.rate == "nochild":
            return np.zeros((nv, n), np.float32)
        out = np.zeros((nv, n), np.float32)
        end = (self.len - self.stop).astype(np.float64)        # size_t: wraps when stopOffset > length
        restart = self.start.astype(np.float64)
        on = self.start.astype(np.float32).astype(np.float64)  # noteOn stores the offset through float
        loop, gated = self.sc.mode == "loop", self.sc.mode != "trigger"
        cols = np.arange(nv)
        for t in range(n):
            x = inputs[:, 0, t]
            rate = inputs[:, 1, t] if self.sc.rate == "input" else np.full(nv, 0.75 if self.sc.rate == "const" else 1.0, np.float32)
            act = self.has
            d = x - self.last
            rise, fall = act & (d > 0.0), act & (d < 0.0)
            self.last = np.where(act, x, self.last)
            c = (self.cur & np.uint64(1)).astype(np.int64)
            self.tg[c[rise], cols[rise]] = 0.0
            self.cur[rise] += np.uint64(1)
            c = (self.cur & np.uint64(1)).astype(np.int64)
            self.tg[c[rise], cols[rise]] = 1.0
            self.pos[c[rise], cols[rise]] = on[rise]
            if gated:
                self.tg[c[fall], cols[fall]] = 0.0
            y0 = self._tick(0, rate, act, end, restart, loop)
            y1 = self._tick(1, rate, act, end, restart, loop)
            out[:, t] = np.where(act, y0 + y1, np.float32(0.0))
        return out


def _edit(sc):       # a second root over the same sample node (output 1): the node, its state and root 0 stay
    smp = sample_node(sc.mode, sc.rate)
    return ("edit", sc.renderer.render(smp, el.mul(smp, el.const(0.5, key="g"))))


def _cut(sc):        # voices 32.. get a graph of their own (a voice-group cut on a tile boundary of every geometry) that keeps the node
    smp = sample_node(sc.mode, sc.rate)
    r = el.Renderer()
    r.render(smp)
    return ("cut", 32, r.render(smp, el.add(smp, el.const(0.25, key="dc"))))


def _path2(sc):
    return ("path", (np.arange(sc.n_voices) + 3) % len(sc.names))


def _path1(sc):
    return ("path", sc.index)


def scenarios():
    return [
        Scenario("trigger"),
        Scenario("gate", mode="gate", seed=1),
        Scenario("loop", mode="loop", seed=2),
        Scenario("one_child", rate="none", seed=3),
        Scenario("const_rate", mode="loop", rate="const", seed=4),
        Scenario("no_child", rate="nochild"),
        Scenario("path_change", offsets="zero", events={6: [_path2]}, seed=5),   # offsets of one buffer may lie outside the next
        Scenario("path_late", mode="gate", path_at_start=False, events={4: [_path1]}, seed=6),
        Scenario("live_edit", mode="loop", events={5: [_edit]}, seed=7),
        Scenario("cut", events={5: [_cut]}, seed=8),
        Scenario("reset_voices", mode="loop", events={7: [("reset_voices", [0, 3, 17, 31, 44])]}, seed=9),
        Scenario("reset", mode="loop", events={6: [("reset",)]}, seed=10),
        Scenario("prune", events={2: [("prune",)]}, seed=11),
        Scenario("ood_stop_past_end", rate="none", offsets="stop_past_end", ood=True, seed=12),
        Scenario("ood_start_past_2len", mode="loop", rate="none", offsets="start_past_2len", ood=True, seed=13),
        Scenario("ood_empty", mode="loop", rate="none", lengths=(0, 1, 5), ood=True, seed=14),
    ]


def many_voices():
    """4096 voices choosing among 64 one-shot resources inside one voice group, per-voice offsets."""
    return Scenario("per_voice_4096", n_voices=4096, lengths=tuple(100 + 37 * k for k in range(64)), calls=(512, 333, 7, 512, 100),
                    seed=20)


def one_voice_graph(v, names, sampler=True):
    """A graph per voice that the warp pipeline would cut if it held no `sample`, in exact IEEE arithmetic (no transcendental
    function, whose device and host results may differ by an ulp): the trigger and the rate come from phasors, not from host inputs."""
    trig = el.le(el.phasor(el.const(3.0 + 0.7 * v, key="tf")), 0.3)
    rate = el.add(0.6, el.mul(0.9, el.phasor(el.const(0.5 + 0.1 * v, key="rf"))))
    smp = el.sample({"key": "smp", "path": names[v % len(names)], "mode": ("trigger", "gate", "loop")[v % 3],
                     "startOffset": v % 5, "stopOffset": v % 3}, trig, rate) if sampler else el.mul(trig, rate)
    saw = el.mul(el.sub(el.phasor(el.const(110.0 + v, key="of")), 0.5), 0.1)
    return el.add(el.mul(smp, 0.5), saw, el.mul(el.min_(el.mul(smp, 1.5), 0.3), 0.2), el.mul(el.max_(el.mul(saw, 3.0), -0.02), 0.05))


def digest(a):
    """sha256 of a float32 array's bytes: the stored form of a reference output (tests/golden/reference_sample.npz)."""
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a, dtype=np.float32)).tobytes()).hexdigest()
