"""The voice axis of the engine: live cuts of a voice group, the warp pipeline on every eligible opcode, re-wiring after a cut, and the
mix bus against its float32 model (tests/mix_model.py) at every scale.

C1  A cut is invisible.  A structural batch sent to part of a running group cuts it (graph_host.cpp, Engine::splitGroupsAt): the moved
    voices take their rows (double states as doubles), delay / sdelay rings, tap buffers, scope / capture / fft rings and capture relays
    along, and the new group gets a freshly compiled program, after which the runtime launches differently (render_groups_kernel,
    render_groups_pipe_kernel at L = 1, a launch per group without batching).  Every family of tests/k1_families.py, in every K1 tile
    geometry, through six cut plans: every voice's outputs must be the SAME BITS as the uncut run, the family contract against the
    reference must hold, the events of the analysis family must equal the uncut run's (global voice ids included), and the mix bus
    must equal the model of the current layout after every call, in both runtimes.
C2  The warp pipeline (one-voice groups, program cut into W stages) on each family whose ops are all pipeline-eligible: bit-identical
    to pipeline_stages = 0, and against the reference.
C3  Re-wiring after a cut: the moved voices get the family graph plus one more root, at the same sample time as per-voice reference
    instances.
C4  The mix bus at scale: layouts from 1 to 8192 voices (K2 group counts 1 to 16, an empty and a short last K2 group), many groups of
    different widths, a range with no graph, a faded-out group, fewer roots than outputs and a fused convolve -> root group; every mix
    bit for bit equal to the model, through process_voices and through process() (host delivery).

ELEM_B200_CUTS_FULL=1 runs the specialised arms of C1 in every geometry and plan (by default a rotating subset).
"""
import os

import numpy as np
import pytest

from elementary_b200 import Runtime, el, graphs
from events_common import canon
from helpers import oracle_cls
from k1_families import (BS, BUILDS, CALLS, FADE_END, FAMILIES, GEOMETRIES, N_VOICES, SR, assert_exact, check_family, make_runtime,
                         reference)
from mix_model import assert_mix, k2_groups, mix_model

FULL = os.environ.get("ELEM_B200_CUTS_FULL") == "1"
CUT_ID = 0x7E000000                      # ids of the unconnected nodes whose creation cuts a group (a fresh one per cut)


# ---- C1: cut plans ------------------------------------------------------------------------------------------------------

PLANS = ("first_tile", "off_32", "two_in_one_batch", "nested", "mid_fade", "pending")


def cut_plan(plan, L):
    """[(call index, (vb, ve), queue a recompiled program first)] for 45 voices at tile width L, or None where the geometry has no
    room for the plan (cuts must fall on tile boundaries)."""
    def m(v):                            # the multiple of L at or below v, at least L
        return L * max(1, v // L)
    if plan == "first_tile":
        return [(6, (L, N_VOICES), False)]
    if plan == "off_32":                 # the new group starts off a 32-voice row boundary: its Vpad and row columns differ
        v = m(24)
        return None if v % 32 == 0 else [(5, (v, N_VOICES), False)]
    if plan == "two_in_one_batch":       # vb and ve both inside the group: three groups
        a, b = m(8), L * (40 // L)
        return None if not a < b < N_VOICES else [(4, (a, b), False)]
    if plan == "nested":                 # cut the new group three calls later, then the old one below the first cut
        c0, c1, c2 = m(8), m(16), L * (32 // L)
        return None if not 0 < c0 < c1 < c2 < N_VOICES else [(3, (c1, N_VOICES), False), (6, (c2, N_VOICES), False),
                                                              (9, (c0, c1), False)]
    if plan == "mid_fade":               # before FADE_END: the roots are still fading in, the new group takes the ramp along
        assert sum(CALLS[:1]) < FADE_END
        return [(1, (m(20), N_VOICES), False)]
    if plan == "pending":                # [[4, roots], [5]] to all voices queues a program; the cut comes before the next process()
        return [(5, (m(12), N_VOICES), True)]
    raise ValueError(plan)


def expected_layout(steps, upto):
    bounds = {0, N_VOICES}
    for call, (vb, ve), _ in steps:
        if call <= upto:
            bounds |= {vb, ve}
    b = sorted(bounds)
    return [(b[i], b[i + 1] - b[i]) for i in range(len(b) - 1)]


def events_by_voice(rt):
    out = {}
    for e in rt.process_queued_events():
        out.setdefault(e["event"]["voice"], []).append(e)
    return {v: canon(es) for v, es in out.items()}


def run_plan(fam, L, niter, build, steps, inputs, **extra):
    """One runtime through CALLS with the cuts of `steps`; after every call: the mix bus against the model, the layout against the
    plan.  Returns (voices [V, nOut, sum(CALLS)], events per call or None)."""
    rt = make_runtime(fam, L, niter, build, **extra)
    roots = fam.batch[-2]
    assert roots[0] == 4
    by_call = {}
    for i, (call, rng, pending) in enumerate(steps):
        by_call.setdefault(call, []).append((CUT_ID + 16 * call + i, rng, pending))
    vs, evs, s = [], [], 0
    for c, n in enumerate(CALLS):
        for node_id, rng, pending in by_call.get(c, ()):
            if pending:
                assert rt.apply_instructions([roots, [5]]) == 0, rt.last_error()
            assert rt.apply_instructions([[0, node_id, "sin"]], voices=rng) == 0, rt.last_error()
        v, mix = rt.process_voices(None if inputs is None else inputs[:, :, s:s + n], fam.n_out, n)
        groups = rt.describe()["groups"]
        assert [(g["v0"], g["nv"]) for g in groups] == expected_layout(steps, c), groups
        assert all(g["tile_width"] == L for g in groups), groups
        assert_mix(mix, mix_model(v, groups), f"{fam.name} L={L} niter={niter} {build} call {c}")
        vs.append(v)
        if fam.name == "analysis":
            evs.append(events_by_voice(rt))
        s += n
    if build != "interp" and not extra.get("batch_groups", 1):
        assert all(g.get("spec_state") == 2 for g in rt.describe()["groups"]), rt.describe()["groups"]
    return np.concatenate(vs, axis=2), (evs if fam.name == "analysis" else None)


_UNCUT = {}


def uncut(fam, L, niter, build, inputs):
    key = (fam.name, L, niter, build)
    if key not in _UNCUT:
        _UNCUT[key] = run_plan(fam, L, niter, build, [], inputs)
    return _UNCUT[key]


def _c1_params():
    """Every family x geometry x plan in the interpreter.  The specialised arms (one NVRTC compile per group and program) run, for
    each family and batch_groups setting, one plan in one geometry, rotated over the families; ELEM_B200_CUTS_FULL=1: all of them."""
    out = []
    for i, f in enumerate(FAMILIES):
        for gi, (L, niter) in enumerate(GEOMETRIES):
            plans = [p for p in PLANS if cut_plan(p, L)]
            for plan in plans:
                out.append(pytest.param(f, L, niter, plan, "interp", 1, id=f"{f}-L{L}n{niter}-{plan}-interp"))
                for bg in (0, 1):
                    if FULL or (gi == (2 * i + bg) % len(GEOMETRIES) and plan == plans[(i + bg) % len(plans)]):
                        out.append(pytest.param(f, L, niter, plan, "spec", bg, id=f"{f}-L{L}n{niter}-{plan}-spec-bg{bg}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("family,tile_width,niter,plan,build,batch_groups", _c1_params())
def test_cut_is_invisible(family, tile_width, niter, plan, build, batch_groups):
    fam = FAMILIES[family]
    ref, inputs = reference(fam)
    steps = cut_plan(plan, tile_width)
    what = f"{family} L={tile_width} niter={niter} {plan} {build} batch_groups={batch_groups}"
    got, evs = run_plan(fam, tile_width, niter, build, steps, inputs, batch_groups=batch_groups)
    # batch_groups = 1 runs the cut groups through the interpreter's many-groups kernel: the same bits as the uncut interpreter run
    # wherever the interpreter and the specialised kernel agree bit for bit (the exact families, tests/test_kernel_matrix_gpu.py)
    base_build = "interp" if (build == "interp" or batch_groups == 1) else build
    if build == "interp" or batch_groups == 0 or fam.contract == "exact":
        want, want_evs = uncut(fam, tile_width, niter, base_build, inputs)
        assert_exact(got, want, what + " against the uncut run")
        if evs is not None:
            for c, (a, b) in enumerate(zip(evs, want_evs)):
                assert a == b, f"{what}: events after call {c} differ from the uncut run"
            assert any(evs), what
    check_family(fam, got, None, ref, inputs, what)


# ---- C2: the warp pipeline on every eligible opcode ------------------------------------------------------------------------

# The host pipelines a one-voice program only if every op is eligible (graph_host.cpp, the warp pipeline section) and the program
# has one root, no tap promotion, no event or ring node and no registered node type.  Host-input reads are not eligible either:
# the variants below feed the families' input channels from in-graph noise (rand) instead.
PIPE_INELIGIBLE = {
    "integer": "el.once (OP_ONCE)",
    "oscillators": "metro (an event node), time (OP_TIME), seq / seq2 / sparseq / sparseq2",
    "delay": "tap_in / tap_out (tap promotion)",
    "analysis": "meter, snapshot (event nodes), scope, fft (ring nodes), capture",
}
MATH_RANGES = [(-10.0, 20.0), (-5.0, 10.0), (0.001, 100.0), (0.5, 3.5), (1.5, 2.0)]      # (offset, span) per math input channel


def _substitute(node, fam, memo):
    if not isinstance(node, el.Node):
        return node
    if node.id() not in memo:
        if node.type == "in" and not node.children:
            c = int(node.props["channel"])
            r = el.rand(seed=101 + c)
            lo, span = MATH_RANGES[c] if fam.contract == "math" else (-1.0, 2.0)
            memo[node.id()] = el.add(lo, el.mul(span, r))
        else:
            memo[node.id()] = el.Node(node.type, node.props, [_substitute(c, fam, memo) for c in node.children])
    return memo[node.id()]


def single_root_variant(fam):
    memo = {}
    return el.add(*[_substitute(r, fam, memo) for r in fam.roots])


PIPE_FAMILIES = [f for f in FAMILIES if f not in PIPE_INELIGIBLE]
PIPE_VOICES = 4


def _pipe_reference(fam, batch):
    outs = []
    for v in range(PIPE_VOICES):
        o = oracle_cls()(SR, BS)
        for name, data in fam.resources.items():
            assert o.add_shared_resource(name, data)
        assert o.apply(batch) == 0
        vb = fam.voice_batch(v)
        if vb:
            assert o.apply(vb) == 0
        outs.append(np.concatenate([o.process(None, 1, n) for n in CALLS], axis=1))
    return np.stack(outs)


def _pipe_run(fam, batch, stages, niter):
    rt = Runtime(SR, BS, PIPE_VOICES, device=0, specialize=0, pipeline_stages=stages, **({"niter": niter} if niter else {}))
    for name, data in fam.resources.items():
        assert rt.add_shared_resource(name, data)
    for v in range(PIPE_VOICES):
        assert rt.apply_instructions(batch, voices=(v, v + 1)) == 0, rt.last_error()
        vb = fam.voice_batch(v)
        if vb:
            assert rt.apply_instructions(vb, voices=(v, v + 1)) == 0, rt.last_error()
    vs = []
    for n in CALLS:
        v, mix = rt.process_voices(None, 1, n)
        assert_mix(mix, mix_model(v, rt.describe()["groups"]), f"{fam.name} pipelined W={stages}")
        vs.append(v)
    return np.concatenate(vs, axis=2), rt.describe()["groups"]


@pytest.mark.gpu
@pytest.mark.parametrize("stages,niter", [(2, 0), (3, 0), (4, 0), (3, 4)])
@pytest.mark.parametrize("family", PIPE_FAMILIES)
def test_pipeline_on_every_eligible_family(family, stages, niter):
    fam = FAMILIES[family]
    batch = el.render(single_root_variant(fam))
    got, groups = _pipe_run(fam, batch, stages, niter)
    base, base_groups = _pipe_run(fam, batch, 0, niter)
    units = groups[0]["ops"] - 1                     # the op list without its leading segment header
    cut = all(g["pipeline_stages"] == stages for g in groups)
    assert all(g["tile_width"] == 1 for g in groups) and all(g["pipeline_stages"] == 1 for g in base_groups)
    if units >= 2 * stages:
        assert cut, groups
    what = f"{family} single root W={stages} niter={niter}"
    assert_exact(got, base, what + " against pipeline_stages=0")
    ref = _pipe_reference(fam, batch)
    if fam.contract == "exact":
        assert_exact(got, ref, what + " against the reference")
    else:
        g, r = got.astype(np.float64), ref.astype(np.float64)
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(g), fin) and np.array_equal(g[~fin], r[~fin], equal_nan=True), what
        peak = np.zeros_like(r)
        for s in range(0, r.shape[-1], BS):
            w = np.where(fin[..., s:s + BS], np.abs(r[..., s:s + BS]), 0.0)
            peak[..., s:s + BS] = w.max(axis=-1, keepdims=True)
        err = np.abs(g - r)[fin]
        assert (err <= 1e-5 * peak[fin] + 1e-7).all(), f"{what}: worst err / (1e-5 peak) {float((err / (1e-5 * peak[fin] + 1e-7)).max()):.3g}"
    print(f"PIPELINE {what}: ops={groups[0]['ops']} pipelined={cut}")


# ---- C3: re-wiring after a cut ----------------------------------------------------------------------------------------------

def _c3_params():
    return [pytest.param(f, *GEOMETRIES[(i + 3 * j) % len(GEOMETRIES)], id=f"{f}-L{GEOMETRIES[(i + 3 * j) % len(GEOMETRIES)][0]}"
                         f"n{GEOMETRIES[(i + 3 * j) % len(GEOMETRIES)][1]}") for i, f in enumerate(FAMILIES) for j in range(3)]


@pytest.mark.gpu
@pytest.mark.parametrize("family,tile_width,niter", _c3_params())
def test_rewire_after_a_cut(family, tile_width, niter):
    fam = FAMILIES[family]
    L = tile_width
    cut, at = L * max(1, 16 // L), 6
    extra = el.mul(0.5, el.phasor(el.const(0.0, key="mx_rw")))        # phasor: exact, with a per-voice frequency
    rg = el.Renderer()
    rg.render(*fam.roots)
    update = rg.render(*fam.roots, extra) + [[3, el.const(0, key="mx_rw").id(), "value", 0.0]]
    n_out = min(fam.n_out + 1, 8)                                      # (an eighth root has no ninth output channel to go to)
    freqs = [300.0 + 37.0 * v for v in range(N_VOICES)]
    _, inputs = reference(fam)
    total = sum(CALLS)
    # per-voice reference instances: the same batches at the same sample time
    refs = []
    for v in range(N_VOICES):
        o = oracle_cls()(SR, BS)
        for name, data in fam.resources.items():
            assert o.add_shared_resource(name, data)
        assert o.apply(fam.batch) == 0
        vb = fam.voice_batch(v)
        if vb:
            assert o.apply(vb) == 0
        parts, s = [], 0
        for c, n in enumerate(CALLS):
            if c == at and v >= cut:
                assert o.apply(update) == 0 and o.apply([[3, el.const(0, key="mx_rw").id(), "value", freqs[v]]]) == 0
            parts.append(o.process(None if inputs is None else inputs[v, :, s:s + n], n_out, n))
            s += n
        refs.append(np.concatenate(parts, axis=1))
    ref = np.stack(refs)
    rt = make_runtime(fam, L, niter, "interp")
    vs, s = [], 0
    for c, n in enumerate(CALLS):
        if c == at:
            assert rt.apply_instructions(update, voices=(cut, N_VOICES)) == 0, rt.last_error()
            assert rt.set_property_per_voice(el.const(0, key="mx_rw").id(), "value", freqs[cut:], cut) == 0, rt.last_error()
            assert [(g["v0"], g["nv"]) for g in rt.describe()["groups"]] == [(0, cut), (cut, N_VOICES - cut)]
        v, mix = rt.process_voices(None if inputs is None else inputs[:, :, s:s + n], n_out, n)
        assert_mix(mix, mix_model(v, rt.describe()["groups"]), f"{family} rewire call {c}")
        vs.append(v)
        s += n
    got = np.concatenate(vs, axis=2)
    assert got.shape[-1] == total
    what = f"{family} L={L} niter={niter} re-wired at voice {cut}"
    k = min(fam.n_out, n_out)
    check_family(fam, got[:, :k], None, ref[:, :k], inputs, what)
    if n_out > fam.n_out:
        assert_exact(got[:, fam.n_out:], ref[:, fam.n_out:], what + " extra root")
        assert np.abs(got[cut:, fam.n_out, FADE_END + sum(CALLS[:at]):]).max() > 0.1, what


# ---- C4: the mix bus at scale ---------------------------------------------------------------------------------------------

def _gain_graph(n_roots):
    """Per-voice gains +-2^k (k in [-20, 20]) on a per-voice phasor mantissa in [1, 2), plus a second per-voice gain switched in by
    a per-voice pulse train, so that the largest terms move between voices from sample to sample."""
    sig = el.add(el.mul(el.const(1.0, key="mb_g"), el.add(1.0, el.phasor(el.const(100.0, key="mb_f")))),
                 el.mul(el.const(1.0, key="mb_h"), el.train(el.const(50.0, key="mb_r"))))
    return [sig, el.mul(-0.375, sig)][:n_roots]


def _gain_props(rt, v0, n, salt=0):
    v = np.arange(v0, v0 + n)
    g = np.where(v % 3 == 0, -1.0, 1.0) * np.exp2((7 * v + salt) % 41 - 20)
    h = np.where(v % 5 == 0, -1.0, 1.0) * np.exp2((11 * v + 3 + salt) % 41 - 20)
    for key, vals in (("mb_g", g), ("mb_h", h), ("mb_f", 31.0 + 13.0 * (v % 97)), ("mb_r", 40.0 + 7.0 * (v % 61))):
        assert rt.set_property_per_voice(el.const(0, key=key).id(), "value", vals, v0) == 0, rt.last_error()


def _ir():
    return (np.asarray(graphs.lcg_ir(700), dtype=np.float32) * 0.5).astype(np.float32)


def _setup_layout(rt, name):
    """Puts the layout `name` on rt; returns the voice ranges whose roots are faded out after the first call."""
    V = rt.num_voices
    if name in SINGLE:
        assert rt.apply_instructions(el.render(*_gain_graph(2))) == 0, rt.last_error()
        _gain_props(rt, 0, V)
        return []
    if name == "12 groups":
        v0 = 0
        for i, (n, L) in enumerate(TWELVE):
            rt.set_option("tile_width", L)                      # a group's tile width is fixed when it is first compiled
            assert rt.apply_instructions(el.render(*_gain_graph(1 + i % 2)), voices=(v0, v0 + n)) == 0, rt.last_error()
            _gain_props(rt, v0, n, salt=i)
            v0 += n
        return []
    if name == "gaps, fade-out, conv":
        # [0, 40) graph at L = 4, [40, 70) no graph, [70, 102) graph whose roots fade out, [102, 107) convolve -> root at L = 1,
        # [107, 140) graph at L = 2
        assert rt.add_shared_resource("mb_ir", _ir())
        for (a, b), L, batch in (((0, 40), 4, el.render(*_gain_graph(2))), ((70, 102), 8, el.render(*_gain_graph(2))),
                                 ((102, 107), 1, el.render(el.convolve({"path": "mb_ir"}, _gain_graph(1)[0]))),
                                 ((107, 140), 2, el.render(*_gain_graph(1)))):
            rt.set_option("tile_width", L)
            assert rt.apply_instructions(batch, voices=(a, b)) == 0, rt.last_error()
            _gain_props(rt, a, b - a, salt=a)
        return [(70, 102)]
    raise ValueError(name)


SINGLE = {"1 voice": (1, 0), "31 voices": (31, 0), "33 voices": (33, 0), "45 voices": (45, 0), "4096 voices L=2": (4096, 2),
          "4097 tiles L=1": (4097, 1), "5000 voices L=1": (5000, 1), "8192 voices L=1": (8192, 1)}
TWELVE = [(40, 4), (3, 1), (64, 32), (20, 2), (48, 8), (1, 1), (32, 16), (9, 4), (17, 2), (70, 32), (24, 8), (6, 1)]
LAYOUTS = {**{k: v[0] for k, v in SINGLE.items()}, "12 groups": sum(n for n, _ in TWELVE), "gaps, fade-out, conv": 140}


def _c4_params():
    out = []
    for i, name in enumerate(LAYOUTS):
        for j, n_out in enumerate((1, 2, 8)):
            if LAYOUTS[name] > 1000 and n_out == 8:
                continue
            bs = (441, 512, 1024)[(i + j) % 3]
            out.append(pytest.param(name, n_out, bs, id=f"{name.replace(' ', '_').replace(',', '')}-out{n_out}-bs{bs}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("layout,n_out,bs", _c4_params())
def test_mix_bus_equals_the_model(layout, n_out, bs):
    V = LAYOUTS[layout]
    L = SINGLE.get(layout, (0, 0))[1]
    opts = {"tile_width": L} if L else {}
    a = Runtime(SR, bs, V, device=0, **opts)                     # process_voices: per-voice outputs + mix
    b = Runtime(SR, bs, V, device=0, **opts)                     # process(): the mix through host delivery
    faded = _setup_layout(a, layout)
    _setup_layout(b, layout)
    calls = (bs, 7, bs - 7, 1, bs, bs, 100, bs, bs)
    groups = None
    for c, n in enumerate(calls):
        if c == 1:
            for vb, ve in faded:                                 # an empty root set: the group's roots fade out
                for rt in (a, b):
                    assert rt.apply_instructions([[4, []], [5]], voices=(vb, ve)) == 0, rt.last_error()
        v, mix = a.process_voices(None, n_out, n)
        host = b.process(None, n_out, n)
        groups = a.describe()["groups"]
        assert groups == b.describe()["groups"]
        want = mix_model(v, groups)
        what = f"{layout} nOut={n_out} bs={bs} call {c} ({n} samples)"
        assert_mix(mix, want, what)
        assert_mix(host, want, what + " process()")
        if c == len(calls) - 1:
            for vb, ve in faded:
                assert not v[vb:ve].any(), f"{what}: the faded-out group still sounds"
            assert np.abs(mix).max() > 0, what
    n_tiles = sum((g["nv"] + g["tile_width"] - 1) // g["tile_width"] for g in groups if g["tile_width"])
    widths = [g["tile_width"] for g in groups]
    if layout in SINGLE and SINGLE[layout][1]:
        assert widths == [L], groups
    if layout == "12 groups":
        assert widths == [w for _, w in TWELVE], groups
    if layout == "gaps, fade-out, conv":
        assert [(g["v0"], g["nv"], g["tile_width"]) for g in groups] == [(0, 40, 4), (40, 30, 0), (70, 32, 8), (102, 5, 1),
                                                                          (107, 33, 2)], groups
    print(f"MIXBUS {layout} nOut={n_out} bs={bs}: tiles={n_tiles} G={k2_groups(n_tiles)} widths={sorted(set(widths))}")


def test_c1_case_count():
    """The size of the cut matrix (CPU): every family in every geometry and every plan the geometry has room for."""
    n = sum(1 for p in _c1_params() if p.values[4] == "interp")
    assert n == len(FAMILIES) * sum(sum(1 for p in PLANS if cut_plan(p, L)) for L, _ in GEOMETRIES)
    assert all(cut_plan(p, L) for p in PLANS for L in (1, 2, 4, 8))
    print(f"C1 interpreter cases: {n}; specialised: {sum(1 for p in _c1_params() if p.values[4] == 'spec')}")
