"""The mix bus past 8 output channels (nOut in (8, 4096]): compact partial rows per voice group and K2w (DESIGN.md sections 3-5).

W1  Reference parity: the K1 matrix families (tests/k1_families.py) with their roots re-aimed at channels 0..15, two roots on one
    channel, one at -1 and one past nOut, rendered with nOut in {9, 12, 16, 64} and against per-voice reference instances given the
    same nOut; the family contracts hold for every per-voice output.  Roots aimed past nOut do not run and keep their state frozen
    until a later call's nOut reaches them, as in the reference.
W2  The mix bus equals its float32 model (tests/wide_mix_model.py) bit for bit after every call, through process_voices, process()
    (host delivery) and enqueue_block + mix_device: one group, 12 groups of mixed widths and channel sets, 1250 one-voice stems
    (batched and pipelined), a fused convolve -> root group, a range without a graph, a group fading out, ragged call lengths,
    block sizes 441 and 1024.
W3  nOut alternating 2 <-> 16: per-voice outputs are the bits of a constant-nOut run; each mix is its own path's model.
W4  The steady-state fast path gives the bits of the slow path.
ELEM_B200_SPECIALIZE=1 runs all of it on the specialised kernels.
"""
import copy

import numpy as np
import pytest

from elementary_b200 import Runtime, el
from elementary_b200.runtime import FLAG_MIX, FLAG_VOICE_OUT
from helpers import oracle_cls
from k1_families import (CALLS, FADE_END, FAMILIES, SR, assert_exact, check_family, family_inputs, make_runtime)
from mix_model import assert_mix
from wide_mix_model import engine_mix_model, wide_k2, wide_mix_model

PARITY_FAMILIES = [f for f in FAMILIES if FAMILIES[f].contract != "math"]   # the math contract names its roots by position
RAGGED = (512, 7, 100, 1, 333)


def aim_roots(batch, channels):
    """The batch with root i re-aimed at channels[i] (the channel props of the roots are rewritten in place)."""
    b = copy.deepcopy(batch)
    roots = next(ins for ins in b if ins[0] == 4)[1]
    where = {ins[1]: ins for ins in b if ins[0] == 3 and ins[2] == "channel" and ins[1] in roots}
    for rid, c in zip(roots, channels):
        where[rid][3] = int(c)
    return b


def parity_channels(n_roots, n_out, distinct=False):
    """Channels among 0..15 (mod nOut), 11 twice: every root of a family runs.  distinct: one root per channel, for the filter
    contract, whose ulp bound is per root output (two roots summed into one channel can cancel).  (A family's roots share nodes, and a node belongs to
    the segment of the first root that reaches it: a root that does not run leaves its nodes unrendered for the later roots that
    read them.  Roots at -1 and past nOut are tested on graphs whose roots share no rendered node, test_roots_outside_nout_*.)"""
    if distinct:
        return [(11 + 5 * i) % n_out for i in range(n_roots)]          # 5 is prime to 9, 12, 16 and 64
    return [c % n_out for c in (11, 0, 11, 3, 15, 5, 9, 12)][:n_roots]


def _roots(rt, voices, pairs, renderer=None):
    """One root per (channel, graph) on the voices [vb, ve)."""
    batch = (renderer or el.Renderer()).render(*[g for _, g in pairs])
    assert rt.apply_instructions(aim_roots(batch, [c for c, _ in pairs]), voices=voices) == 0, rt.last_error()


# ---- W1: reference parity -----------------------------------------------------------------------------------------------

def _parity_run(fam, n_outs, calls, L):
    """GPU per-voice outputs and the reference's, both [V, max nOut, sum(calls)], call k rendered with nOut = n_outs[k]."""
    width = max(n_outs)
    batch = aim_roots(fam.batch, parity_channels(len(next(i for i in fam.batch if i[0] == 4)[1]), min(n_outs), fam.contract == "filter"))
    f2 = copy.copy(fam)
    f2.batch = batch
    rt = make_runtime(f2, L, 0, "interp" if not _spec() else "spec")
    V = rt.num_voices
    inputs = family_inputs(fam, V, sum(calls))
    got = np.zeros((V, width, sum(calls)), np.float32)
    ref = np.zeros_like(got)
    s = 0
    for n, n_out in zip(calls, n_outs):
        v, mix = rt.process_voices(None if inputs is None else inputs[:, :, s:s + n], n_out, n)
        assert_mix(mix, engine_mix_model(v, rt.describe()["groups"], n_out), f"{fam.name} nOut={n_out}")
        got[:, :n_out, s:s + n] = v
        s += n
    for vi in range(V):
        o = oracle_cls()(SR, rt.block_size)
        for name, data in fam.resources.items():
            assert o.add_shared_resource(name, data)
        assert o.apply(batch) == 0
        vb = fam.voice_batch(vi)
        if vb:
            assert o.apply(vb) == 0
        s = 0
        for n, n_out in zip(calls, n_outs):
            ref[vi, :n_out, s:s + n] = o.process(None if inputs is None else inputs[vi, :, s:s + n], n_out, n)
            s += n
    return got, ref, inputs


def _spec():
    import os
    return os.environ.get("ELEM_B200_SPECIALIZE") == "1"


@pytest.mark.gpu
@pytest.mark.parametrize("family", PARITY_FAMILIES)
@pytest.mark.parametrize("n_out", [9, 12, 16, 64])
def test_reference_parity(family, n_out):
    fam = FAMILIES[family]
    got, ref, inputs = _parity_run(fam, [n_out] * len(CALLS), CALLS, 4)
    check_family(fam, got, None, ref, inputs, f"{family} nOut={n_out}")


def _disjoint(i):
    """_gain(i) with every constant its own node: in the reference a `const` is a node that renders in the segment of the first root
    reaching it, so roots that do not run must share none with the roots that do."""
    k = lambda name, v: el.const(v, key=f"wd{name}_{i}")
    return el.add(el.mul(el.const(1.0, key=f"wg0_{i}"), el.add(k("one", 1.0), el.phasor(el.const(100.0, key=f"wf0_{i}")))),
                  el.mul(el.const(1.0, key=f"wh0_{i}"), el.le(el.phasor(el.const(50.0, key=f"wr0_{i}")), k("half", 0.5))))


def _outside_run(n_outs, calls, L):
    """Five independent per-voice graphs (no node shared between roots) on channels 11, 0, -1, 11 and 13, per-voice constants; GPU
    and per-voice reference instances, call k with nOut = n_outs[k].  Returns (gpu, ref) [V, max nOut, sum(calls)]."""
    V, width = 45, max(n_outs)
    pairs = [(11, _disjoint(0)), (0, _disjoint(1)), (-1, _disjoint(2)), (11, el.mul(el.const(-0.375, key="wdneg"), _disjoint(3))),
             (13, _disjoint(4))]
    batch = aim_roots(el.Renderer().render(*[g for _, g in pairs]), [c for c, _ in pairs])
    rt = Runtime(SR, 512, V, device=0, tile_width=L)
    assert rt.apply_instructions(batch) == 0, rt.last_error()
    props = {}
    for i in range(5):
        props.update(_gain_props(rt, 0, V, i))
    got = np.zeros((V, width, sum(calls)), np.float32)
    ref = np.zeros_like(got)
    s = 0
    for n, n_out in zip(calls, n_outs):
        v, mix = rt.process_voices(None, n_out, n)
        assert_mix(mix, engine_mix_model(v, rt.describe()["groups"], n_out), f"outside nOut={n_out}")
        got[:, :n_out, s:s + n] = v
        s += n
    for vi in range(V):
        o = oracle_cls()(SR, 512)
        assert o.apply(batch) == 0
        assert o.apply([[3, nid, "value", float(vals[vi])] for nid, vals in props.items()]) == 0
        s = 0
        for n, n_out in zip(calls, n_outs):
            ref[vi, :n_out, s:s + n] = o.process(None, n_out, n)
            s += n
    return got, ref


@pytest.mark.gpu
@pytest.mark.parametrize("n_out", [9, 12, 16, 64])
def test_roots_outside_nout_against_the_reference(n_out):
    got, ref = _outside_run([n_out] * 6, (512, 512, 7, 100, 1, 333), 4)
    assert_exact(got, ref, f"roots at -1 and past nOut, nOut={n_out}")
    assert not got[:, 1:min(11, n_out)].any() and got[:, 0].any() and (n_out <= 11 or got[:, 11].any())


@pytest.mark.gpu
def test_roots_past_nout_stay_frozen_until_nout_grows():
    """The root on channel 13 does not run at nOut = 9 or 12 (its phasor and train keep their state) and starts where it stopped
    when a call's nOut reaches it, as in the reference."""
    got, ref = _outside_run([9, 12, 9, 16, 12, 16], (512, 512, 100, 512, 333, 512), 2)
    assert_exact(got, ref, "nOut 9 -> 16")
    assert got[:, 13].any()


# ---- W2: the mix bus against the model --------------------------------------------------------------------------------

def _gain(i, salt=0):
    """A per-voice signal with gains +-2^k: the largest terms move between voices from sample to sample."""
    return el.add(el.mul(el.const(1.0, key=f"wg{salt}_{i}"), el.add(1.0, el.phasor(el.const(100.0, key=f"wf{salt}_{i}")))),
                  el.mul(el.const(1.0, key=f"wh{salt}_{i}"), el.train(el.const(50.0, key=f"wr{salt}_{i}"))))


def _gain_props(rt, v0, n, i, salt=0):
    v = np.arange(v0, v0 + n)
    g = np.where(v % 3 == 0, -1.0, 1.0) * np.exp2((7 * v + salt) % 41 - 20)
    h = np.where(v % 5 == 0, -1.0, 1.0) * np.exp2((11 * v + 3 + salt) % 41 - 20)
    for key, vals in ((f"wg{salt}_{i}", g), (f"wh{salt}_{i}", h), (f"wf{salt}_{i}", 31.0 + 13.0 * (v % 97)),
                      (f"wr{salt}_{i}", 40.0 + 7.0 * (v % 61))):
        assert rt.set_property_per_voice(el.const(0, key=key).id(), "value", vals, v0) == 0, rt.last_error()
    return {el.const(0, key=key).id(): vals for key, vals in ((f"wg{salt}_{i}", g), (f"wh{salt}_{i}", h),
                                                              (f"wf{salt}_{i}", 31.0 + 13.0 * (v % 97)), (f"wr{salt}_{i}", 40.0 + 7.0 * (v % 61)))}


TWELVE = [(40, 4), (3, 1), (64, 32), (20, 2), (48, 8), (1, 1), (32, 16), (9, 4), (17, 2), (70, 32), (24, 8), (6, 1)]


def _setup(rt, layout, n_out):
    """Puts `layout` on rt; returns the voice ranges whose roots fade out after the first call."""
    V = rt.num_voices
    if layout == "one group":
        _roots(rt, (0, V), [(11, _gain(0)), (0, _gain(1)), (11, el.mul(-0.375, _gain(0))), (-1, _gain(2)), (n_out + 4, _gain(3))])
        for i in range(4):
            _gain_props(rt, 0, V, i)
        return []
    if layout in ("12 groups", "12 groups in range"):
        v0 = 0
        for i, (n, L) in enumerate(TWELVE):
            rt.set_option("tile_width", L)
            chans = [(i * 5 + 3) % n_out, i % n_out, n_out + i if layout == "12 groups" else (i * 3 + 1) % n_out][:1 + i % 3]
            _roots(rt, (v0, v0 + n), [(c, _gain(k, salt=i)) for k, c in enumerate(chans)])
            for k in range(len(chans)):
                _gain_props(rt, v0, n, k, salt=i)
            v0 += n
        return []
    if layout == "stems":
        for i in range(V):
            _roots(rt, (i, i + 1), [(i, _gain(0, salt=i % 7))])
            _gain_props(rt, i, 1, 0, salt=i % 7)
        return []
    if layout == "gaps, fade-out, conv":
        # [0, 40) L = 4 on 3 and 9, [40, 70) no graph, [70, 102) L = 8 fading out, [102, 107) convolve -> root on 11 at L = 1,
        # [107, 140) L = 2 on 9
        ir = np.asarray([(((i * 1103515245 + 12345) >> 8) % 2001 - 1000) / 1000.0 * np.exp(-i / 150.0) for i in range(700)],
                        np.float32) * 0.5
        assert rt.add_shared_resource("wm_ir", ir)
        for (a, b), L, pairs, salt in (((0, 40), 4, [(3, _gain(0, 1)), (9, _gain(1, 1))], 1),
                                       ((70, 102), 8, [(12, _gain(0, 2)), (3, _gain(1, 2))], 2),
                                       ((102, 107), 1, [(11, el.convolve({"path": "wm_ir"}, _gain(0, 3)))], 3),
                                       ((107, 140), 2, [(9, _gain(0, 4))], 4)):
            rt.set_option("tile_width", L)
            _roots(rt, (a, b), pairs)
            for k in range(len(pairs)):
                _gain_props(rt, a, b - a, k, salt=salt)
        return [(70, 102)]
    if layout == "long lists":
        for (a, b), L, chans, salt in LONG:
            rt.set_option("tile_width", L)
            _roots(rt, (a, b), [(c, _gain(k, salt)) for k, c in enumerate(chans)])
            for k in range(len(chans)):
                _gain_props(rt, a, b - a, k, salt=salt)
        return []
    raise ValueError(layout)


# K2w's long row lists: channel 3 has 4097 + 200 rows (G = 16 tile groups of 288 rows, the last one empty: the scratch / ticket finish
# and the CTA-per-segment kernel), channel 7 has 4097 (G = 16, last empty), channel 5 has 200 (G = 1, four-accumulator rounds), a
# few small groups on other channels; 12 is past nOut at nOut = 9.
LONG = [((0, 4097), 1, (3, 7), 11), ((4097, 4297), 1, (5, 3), 12), ((4297, 4330), 4, (0, 8), 13), ((4330, 4340), 2, (1, 12), 14)]
LAYOUTS = {"one group": 45, "12 groups": sum(n for n, _ in TWELVE), "stems": 1250, "gaps, fade-out, conv": 140, "long lists": 4340}


def _device_mix(rt, n_out, n, voices):
    import torch
    rt.synchronize()
    mix = torch.as_tensor(rt.mix_device(n_out), device="cuda").cpu().numpy()[:, :n]
    v = torch.as_tensor(rt.voice_out_device(n_out), device="cuda").cpu().numpy()[:, :, :n] if voices else None
    return mix, v


def _stem_outputs(rt, n_out, n):
    """(mix [n_out, n], the diagonal v[i, i] [V, n]) of an enqueue_block; asserts every off-diagonal per-voice channel is zero."""
    import torch
    rt.synchronize()
    mix = torch.as_tensor(rt.mix_device(n_out), device="cuda").cpu().numpy()[:, :n]
    dv = torch.as_tensor(rt.voice_out_device(n_out), device="cuda")[:, :, :n].clone()
    idx = torch.arange(rt.num_voices, device="cuda")
    diag = dv[idx, idx].clone()
    dv[idx, idx] = 0.0
    assert not bool(dv.any()), "a stem wrote outside its own channel"
    return mix, diag.cpu().numpy()


def _w2_params():
    out = []
    for name in LAYOUTS:
        for n_out, bs in (((9, 512), (16, 441)) if name == "long lists" else ((16, 512), (64, 441), (16, 1024))):
            if name == "stems":
                n_out = 1250
            out.append(pytest.param(name, n_out, bs, id=f"{name.replace(' ', '_').replace(',', '')}-out{n_out}-bs{bs}"))
    out.append(pytest.param("stems", 1250, 512, {"pipeline_stages": 0}, id="stems-out1250-bs512-unpipelined"))
    return [p if len(p.values) == 4 else pytest.param(*p.values, {}, id=p.id) for p in out]


@pytest.mark.gpu
@pytest.mark.parametrize("layout,n_out,bs,opts", _w2_params())
def test_mix_bus_equals_the_model(layout, n_out, bs, opts):
    V = LAYOUTS[layout]
    a, b, c = (Runtime(SR, bs, V, device=0, **opts) for _ in range(3))
    faded = _setup(a, layout, n_out)
    _setup(b, layout, n_out)
    _setup(c, layout, n_out)
    calls = (bs,) + tuple(min(n, bs) for n in RAGGED) + (bs, bs)
    if layout == "stems":
        calls = (bs, 7, 333, bs, bs)
    for k, n in enumerate(calls):
        if k == 1:
            for vb, ve in faded:
                for rt in (a, b, c):
                    assert rt.apply_instructions([[4, []], [5]], voices=(vb, ve)) == 0, rt.last_error()
        what = f"{layout} nOut={n_out} bs={bs} call {k} ({n} samples)"
        host = b.process(None, n_out, n)
        c.enqueue_block(0, n_out, n, flags=FLAG_MIX | FLAG_VOICE_OUT)
        if layout == "stems":
            # [1250][1250][n] per-voice outputs stay on the device: stem i is voice i on channel i, every other channel is zero
            _, mix = a.process_voices(None, n_out, n, want_voices=False)
            dmix, v = _stem_outputs(c, n_out, n)
            groups = a.describe()["groups"]
            want = wide_k2(v, [[i] for i in range(V)], n)
        else:
            v, mix = a.process_voices(None, n_out, n)
            dmix, dv = _device_mix(c, n_out, n, True)
            assert np.array_equal(dv.view(np.uint32), v.view(np.uint32)), what + ": per-voice outputs of enqueue_block"
            groups = a.describe()["groups"]
            want = wide_mix_model(v, groups, n_out)
        assert_mix(mix, want, what + " process_voices")
        assert_mix(host, want, what + " process()")
        assert_mix(dmix, want, what + " enqueue_block")
        if k == len(calls) - 1:
            for vb, ve in faded:
                assert not v[vb:ve].any(), f"{what}: the faded-out group still sounds"
            assert np.abs(mix).max() > 0, what
    if layout == "stems":
        assert all(g["mix_channels"] == [i] for i, g in enumerate(groups)), groups[:3]
    if layout == "gaps, fade-out, conv":
        assert [g["mix_channels"] for g in groups if "mix_channels" in g] == [[3, 9], [3, 12], [11], [9]], groups
    if layout == "long lists":
        from wide_mix_model import wide_rows
        assert [(g["v0"], g["nv"], g["tile_width"]) for g in groups] == [(a, b - a, L) for (a, b), L, _, _ in LONG], groups
        _, R = wide_rows(v, groups, n_out)
        assert [len(R[c]) for c in (3, 7, 5, 0, 8, 1)] == [4297, 4097, 200, 9, 9, 5]


# ---- W3 / W4 -----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_alternating_nout_matches_a_constant_run():
    V = LAYOUTS["12 groups"]
    alt, const = Runtime(SR, 512, V, device=0), Runtime(SR, 512, V, device=0)
    for rt in (alt, const):
        v0 = 0
        for i, (n, L) in enumerate(TWELVE):                              # roots on channels 0 and 1 only: every root runs at nOut = 2
            rt.set_option("tile_width", L)
            _roots(rt, (v0, v0 + n), [(ch, _gain(k, salt=i)) for k, ch in enumerate([i % 2, 1 - i % 2][:1 + i % 2])])
            for k in range(1 + i % 2):
                _gain_props(rt, v0, n, k, salt=i)
            v0 += n
    for k, n in enumerate((512, 7, 100, 512, 1, 333, 512, 512)):
        n_out = (2, 16)[k % 2]
        v, mix = alt.process_voices(None, n_out, n)
        w, _ = const.process_voices(None, 16, n)
        groups = alt.describe()["groups"]
        assert np.array_equal(v[:, :2].view(np.uint32), w[:, :2].view(np.uint32)), f"call {k} nOut={n_out}"
        assert not w[:, 2:].any()
        assert_mix(mix, engine_mix_model(v, groups, n_out), f"alternating call {k} nOut={n_out}")
        if n_out == 2:
            from mix_model import mix_model
            assert_mix(mix, mix_model(v, groups), f"alternating call {k}: the dense model")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["stems", "12 groups in range"])
def test_steady_fast_path_gives_the_slow_path_bits(layout):
    """Runtime `slow` has its steady state invalidated before every block (any option does that); `fast` relaunches its cached work
    once its fades have settled (describe()["steady"]: the next block of the same shape takes the fast path).  Each phase keeps one
    call shape — per-voice outputs + mix (scatter and K2w relaunched), then process() (K2w with host delivery) — so the fast path
    really runs in both.  (Every root aims inside [0, nOut): a root that does not run never finishes its fade-in, and a fading root
    keeps an engine off the fast path.)"""
    V = LAYOUTS["12 groups" if layout == "12 groups in range" else layout]
    n_out = 1250 if layout == "stems" else 16
    fast, slow = Runtime(SR, 512, V, device=0), Runtime(SR, 512, V, device=0)
    for rt in (fast, slow):
        _setup(rt, layout, n_out)
    voices = layout != "stems"               # 1250 x 1250 per-voice channels: the mix alone
    fast_blocks = 0
    for phase in ("process_voices", "process"):
        for k in range(6):                   # the 20 ms fades settle within two blocks
            if k >= 3:
                assert fast.describe()["steady"], f"{layout} {phase} block {k}: the fast path is not armed"
            fast_blocks += fast.describe()["steady"]
            slow.set_option("time_kernels", 0)
            assert not slow.describe()["steady"]
            what = f"{layout} {phase} block {k}"
            if phase == "process":
                assert_mix(fast.process(None, n_out, 512), slow.process(None, n_out, 512), what)
                continue
            vf, mf = fast.process_voices(None, n_out, 512, want_voices=voices)
            vs, ms = slow.process_voices(None, n_out, 512, want_voices=voices)
            assert_mix(mf, ms, what)
            if voices:
                assert np.array_equal(vf.view(np.uint32), vs.view(np.uint32)), f"{what}: per-voice outputs"
                assert_mix(mf, wide_mix_model(vf, fast.describe()["groups"], n_out), f"{what}: model")
    assert fast_blocks >= 6 and fast.kernel_launches == slow.kernel_launches
    assert FADE_END < 8 * 512
