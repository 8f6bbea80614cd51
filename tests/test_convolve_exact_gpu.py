"""GPU: K3 (`convolve_chunk_tm_kernel`, both forms) against the exact float64 convolution of tests/conv_exact.py, every channel of
every run, under the normwise contract `max over block |gpu - exact| <= C * E_b` — plus the properties that hold bit for bit:

* layout invariance: a channel's output does not depend on the channel count, its place in its pair or unit, its partner's input
  or IR, or the kernel form;
* exact silence: once a channel's input has been zero for (S + 1) * 512 samples (through the end of the current partition) its
  output is 0.0;
* exact scaling: an input scaled by 2^+-32 gives the output scaled by exactly that factor.

Every run starts with `lead` silent samples (at least 1024, a whole number of blocks) so that the root's 20 ms fade-in has reached
its target: after that the root multiplies by exactly 1.0 and the per-voice output is K3's output.  The lead is part of the compared
stream (its output must be exactly 0.0), and the partition grid starts with the runtime's first sample.

The default run covers every IR kind and length, every layout edge and BASELINE config 4's geometry (1024 channels, one 16384-tap
IR, 40 blocks, more channel pairs than CTAs) and rotates the block sizes, call patterns and forms over the IR lengths;
ELEM_B200_CONV_FULL=1 runs the whole cross product.  The worst |err| / E_b per form is printed at the end of the module."""
import os

import numpy as np
import pytest

import conv_exact as ce
from elementary_b200 import Runtime, el

pytestmark = pytest.mark.gpu
SR = 48000.0
FULL = os.environ.get("ELEM_B200_CONV_FULL") == "1"
RAGGED = (512, 7, 100, 1, 511, 333, 512)
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nK3 worst |err| / E_b: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())) + f" (contract: C = {ce.C:g})")


def grid():
    """Persistent K3 CTAs: two per SM."""
    import torch
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count


def lead_for(bs):
    return -(-1024 // bs) * bs


def engine(nv, resources, path, bs=512, **opts):
    rt = Runtime(SR, bs, nv, device=0, **opts)
    for k, v in resources.items():
        assert rt.add_shared_resource(k, v)
    cv = el.convolve({"path": path, "key": "cv"}, el.in_(0))
    assert rt.apply_instructions(el.render(cv)) == 0, rt.last_error()
    return rt, cv.id()


def form(rt):
    return [c for g in rt.describe()["groups"] for c in g.get("convolvers", [])][0]["form"]


def stream(rt, x, calls=None, t0=0, t1=None, want_mix=False):
    """Feed x[:, t0:t1] through process_voices in call lengths `calls` (cycled; default: the block size)."""
    t1 = x.shape[-1] if t1 is None else t1
    calls = calls or (rt.block_size,)
    outs, mixes, t, k = [], [], t0, 0
    while t < t1:
        m = min(calls[k % len(calls)], t1 - t)
        v, mx = rt.process_voices(x[:, None, t:t + m], 1, m, want_mix=want_mix)
        outs.append(v[:, 0])
        mixes.append(mx[0] if want_mix else None)
        t, k = t + m, k + 1
    return np.concatenate(outs, axis=1), (np.concatenate(mixes) if want_mix else None)


def check(out, x, h, label, start=None, want=None, E=None):
    """Every row of `out` against exact(x, h) under C * bound(x, h)."""
    want = ce.exact(x, h, start) if want is None else want
    E = ce.bound(x, h, start) if E is None else E
    r = ce.ratio(out, want, E)
    WORST[label] = max(WORST.get(label, 0.0), float(r.max()))
    bad = np.nonzero(r > ce.C)[0]
    assert bad.size == 0, f"{label}: {bad.size} channels over the contract, worst {r.max():.3g} x E_b (channel {int(r.argmax())}), C = {ce.C}"


def check_silence(out, x, hs):
    """Exact silence: out[c, m] == 0.0 wherever x[c] is zero from m - (S_c + 1) * 512 + 1 to the end of m's partition."""
    n = x.shape[-1]
    nz = np.concatenate([np.zeros((x.shape[0], 1), np.int64), np.cumsum(x != 0, axis=1)], axis=1)
    m = np.arange(n)
    end = np.minimum((m // ce.P + 1) * ce.P, n)
    for c in range(x.shape[0]):
        S = ce.partitions(hs if isinstance(hs, np.ndarray) else hs[c])
        lo = np.maximum(m - (S + 1) * ce.P + 1, 0)
        quiet = nz[c, end] - nz[c, lo] == 0
        assert not out[c, quiet].any(), f"channel {c}: {int((out[c, quiet] != 0).sum())} nonzero samples after silence"


def since(out, start):
    """out with the samples before each row's start index cleared (they belong to an earlier IR)."""
    st = np.broadcast_to(np.asarray(start), (out.shape[0],))
    return np.where(np.arange(out.shape[1])[None, :] >= st[:, None], out, 0.0)


def inputs(kinds, n, lead, seed0=0):
    return np.stack([ce.make_input(k, n, seed=seed0 + s, lead=lead) for k, s in kinds])


# ---- 1. IR kinds x lengths (plus trailing runs below 1e-6), rotated block sizes / call patterns / forms -------------------------
PATTERNS = ["bs512", "bs64", "bs441", "bs1024", "ragged"]
KINDS7 = [(k, 1) for k in ce.INPUT_KINDS]


def _length_params():
    out = []
    for i, (kind, (taps, tail)) in enumerate((k, lt) for lt in ce.LENGTHS for k in ce.IR_KINDS):
        pats = PATTERNS if FULL else ["bs512", PATTERNS[1 + i % 4]]
        forms = ("shared", "per_channel") if FULL else (("shared", "per_channel")[i % 2],)
        for pat in pats:
            for f in forms:
                out.append(pytest.param(kind, taps, tail, pat, f, id=f"{kind}-{taps}+{tail}-{pat}-{f}"))
    return out


@pytest.mark.parametrize("kind,taps,tail,pattern,frm", _length_params())
def test_ir_kinds_and_lengths(kind, taps, tail, pattern, frm):
    """Seven channels, one per input kind (odd: the last unit holds one channel); per-channel form: three more channels on a
    longer IR, a one-partition IR and a zero IR."""
    h = ce.make_ir(kind, taps, seed=taps + 7, tail=tail)
    assert ce.partitions(h) == -(-taps // ce.P)
    bs = int(pattern[2:]) if pattern.startswith("bs") else 512
    calls = RAGGED if pattern == "ragged" else None
    lead = lead_for(bs)
    S = ce.partitions(h)
    n = lead + 3 * ce.P * len(ce.IMPULSE_OFFSETS) + (S + 2) * ce.P
    x = inputs(KINDS7, n, lead)
    res = {"h": h}
    hs = [h] * 7
    if frm == "per_channel":
        others = {"o_long": ce.make_ir("lcg", 5000, seed=3), "o_one": ce.make_ir("flat", 300, seed=4), "o_zero": np.zeros(64, np.float32)}
        res |= others
        hs += list(others.values())
        x = np.concatenate([x, inputs([("noise", 5), ("tone", 1), ("noise", 6)], n, lead)])
    rt, cid = engine(x.shape[0], res, "h", bs=bs)
    if frm == "per_channel":
        assert rt.set_path_per_voice(cid, list(res), [0] * 7 + [1, 2, 3]) == 0, rt.last_error()
    assert form(rt) == frm
    out, _ = stream(rt, x, calls)
    check(out, x, hs, frm)
    check_silence(out, x, hs)


# ---- 2. BASELINE config 4's geometry: 1024 channels, one 16384-tap IR, 40 blocks ------------------------------------------------
def test_config4_geometry_every_channel_and_layout_invariance():
    """1024 channels = 512 pairs on 2 * SMs persistent CTAs (two pairs per CTA on an H100), every channel against `exact`; then
    the same 1024 signals one channel further on with a silent channel 0 (every channel changes place in its pair, its unit and
    its CTA; the balanced grid changes) must give the same bits."""
    nv, nb = 1024, 40
    assert nv // 2 > grid()
    h = ce.make_ir("lcg", 16384)
    lead = 1024
    n = nb * 512
    kinds = [(ce.INPUT_KINDS[c % 7] if c % 3 == 0 else "noise", c) for c in range(nv)]
    x = inputs(kinds, n, lead)
    rt, _ = engine(nv, {"ir": h}, "ir")
    out, _ = stream(rt, x)
    check(out, x, h, "shared")
    check_silence(out, x, h)
    x2 = np.concatenate([np.zeros((1, n), np.float32), x])
    rt2, _ = engine(nv + 1, {"ir": h}, "ir")
    out2, _ = stream(rt2, x2)
    assert not out2[0].any()
    assert np.array_equal(out2[1:], out)


# ---- 3. layouts: unit counts around the persistent grid, odd and even channel counts, both forms ---------------------------------
POOL = [("noise", 1), ("noise", 2), ("noise", 3), ("impulses", 0), ("impulses", 1), ("dc", 0), ("alternating", 0), ("quarter", 0),
        ("tone", 0), ("burst", 0), ("silence", 0)]
LAYOUT_IRS = {"a": ("lcg", 2049), "t": ("taps", 300), "z": None, "l": ("lcg", 8193), "b": ("flat", 700)}
_refs = {}


def _layout_ir(name):
    spec = LAYOUT_IRS[name]
    return np.zeros(64, np.float32) if spec is None else ce.make_ir(spec[0], spec[1], seed=11)


def _layout_n():
    return 1024 + 3 * ce.P * len(ce.IMPULSE_OFFSETS) + (ce.partitions(_layout_ir("l")) + 2) * ce.P


def layout_ref(name):
    """One shared-form run of the whole signal pool on IR `name` (plus a one-channel run of two signals): the bits every channel
    of the layouts must reproduce, and the pool's exact outputs and bounds."""
    if name not in _refs:
        h, n = _layout_ir(name), _layout_n()
        x = inputs(POOL, n, 1024)
        rt, _ = engine(len(POOL), {"ir": h}, "ir")
        out, _ = stream(rt, x)
        want, E = ce.exact(x, h), ce.bound(x, h)
        check(out, x, h, "shared", want=want, E=E)
        check_silence(out, x, h)
        for k in (0, 4):
            solo, _ = engine(1, {"ir": h}, "ir")
            assert np.array_equal(stream(solo, x[k:k + 1])[0][0], out[k])
        _refs[name] = (x, out, want, E)
    return _refs[name]


def _layout_params():
    out = []
    for i, u in enumerate(["1", "2", "g-1", "g", "g+1", "2g", "2g+1", "3g+1"]):
        for odd in (False, True):
            forms = ("shared", "per_channel") if FULL or u in ("2", "g+1", "3g+1") or (i + odd) % 2 else ("shared",)
            for f in forms:
                out.append(pytest.param(u, odd, f, id=f"units={u}-{'odd' if odd else 'even'}-{f}"))
    return out


@pytest.mark.parametrize("units,odd,frm", _layout_params())
def test_layouts(units, odd, frm):
    """Channel c carries pool signal (5 c + units) mod 11 (silent partners included).  Per-channel form: IRs of S = 5, 1, 0, 17
    and 2 assigned in runs of odd length, so that pairs mix IRs of different S and units of S <= 1 (which the producer skips) lie
    between long ones.  Every channel must equal the shared-form pool run bit for bit, and so lie within the contract."""
    g = grid()
    u = {"1": 1, "2": 2, "g-1": g - 1, "g": g, "g+1": g + 1, "2g": 2 * g, "2g+1": 2 * g + 1, "3g+1": 3 * g + 1}[units]
    nv = 2 * u - (1 if odd else 0)
    if nv == 0:
        pytest.skip("no channel")
    sig = (5 * np.arange(nv) + u) % len(POOL)
    names = list(LAYOUT_IRS)
    if frm == "shared":
        irn = np.zeros(nv, np.int64)
    else:
        run = np.array([3, 5, 1, 7, 3])                         # odd run lengths: a then t, z, l, b, repeated
        irn = np.repeat(np.tile(np.arange(len(names)), nv // run.sum() + 1), np.tile(run, nv // run.sum() + 1))[:nv]
        if nv >= 2:
            irn[:2] = [1, 0]                                    # channel 0 on a one-partition IR, first in the unit order
    res = {nm: _layout_ir(nm) for nm in names}
    x0 = layout_ref("a")[0]
    x = x0[sig]
    rt, cid = engine(nv, res, "a")
    if frm == "per_channel":
        assert rt.set_path_per_voice(cid, names, irn) == 0, rt.last_error()
        assert form(rt) == ("per_channel" if len(set(irn.tolist())) > 1 else "shared")
    out, _ = stream(rt, x)
    for k, nm in enumerate(names):
        rows = np.nonzero(irn == k)[0]
        if rows.size == 0:
            continue
        _, ref, want, E = layout_ref(nm)
        check(out[rows], x[rows], _layout_ir(nm), frm, want=want[sig[rows]], E=E[sig[rows]])
        assert np.array_equal(out[rows], ref[sig[rows]]), f"IR {nm}: channels differ from the pool run"


# ---- 4. exact scaling ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frm", ["shared", "per_channel"])
def test_input_scaled_by_a_power_of_two_scales_the_output_exactly(frm):
    h = ce.make_ir("flat", 3000, seed=5)
    res = {"a": h, "b": ce.make_ir("lcg", 1200, seed=6)}
    n = 1024 + 12 * ce.P
    x = inputs([(k, s) for k, s in POOL], n, 1024)
    outs = {}
    for e in (0, 32, -32):
        rt, cid = engine(len(POOL), res, "a")
        if frm == "per_channel":
            assert rt.set_path_per_voice(cid, ["a", "b"], [k % 2 for k in range(len(POOL))]) == 0
        outs[e], _ = stream(rt, x * np.float32(2.0 ** e), RAGGED)
    assert np.abs(outs[0]).max() > 0
    for e in (32, -32):
        assert np.array_equal(outs[e], outs[0] * np.float32(2.0 ** e)), e


# ---- 5. reassignment mid-stream, ring growth, back to the shared form ---------------------------------------------------------
def test_reassignment_mid_stream_then_back_to_the_shared_form():
    """More units than CTAs, ragged calls.  t1 (mid-partition): channels [s, s + k) get IRs b (S = 2) and long (S = 18, the ring
    grows: relayout); t2: set_path_per_voice puts every channel on c (S = 3): the shared form with a ring of R = 18 > S; t3: a
    whole-group JSON `path` a: a fresh convolver.  Reassigned channels match `exact` from their restart, the others keep the bits
    of a run without the reassignment, and all of them fall exactly silent (S + 1) partitions after their input does."""
    g = grid()
    nv = 2 * g + 5
    res = {"a": ce.make_ir("lcg", 2049, seed=21), "b": ce.make_ir("flat", 700, seed=22), "long": ce.make_ir("lcg", 9000, seed=23),
           "c": ce.make_ir("taps", 1500, seed=24)}
    lead = 1024
    seg = 40 * ce.P
    n = 3 * seg + 30 * ce.P
    x = inputs([POOL[c % len(POOL)] for c in range(nv)], n, lead, seed0=0)
    for t in (seg - 2 * ce.P, 2 * seg - 21 * ce.P, 3 * seg - 4 * ce.P, n - 19 * ce.P):
        x[:, t:t + 19 * ce.P // 2] = 0.0                           # silences longer than (S + 1) partitions before each change
    x[:, n - 19 * ce.P:] = 0.0
    rt, cid = engine(nv, res, "a")
    plain, _ = engine(nv, res, "a")
    s, k = 37, 2 * g - 40
    sub = np.arange(s, s + k)
    idx = np.arange(k) % 3 == 0                                    # 1 of 3 on "long", the rest on "b"
    parts, pparts, t = [], [], 0
    t1 = seg + 333                                                 # not a partition boundary: fill > 0
    t2, t3 = 2 * seg + 100, 3 * seg + 7
    for stop, act in ((t1, None), (t2, "assign"), (t3, "shared"), (n, "json")):
        if act == "assign":
            assert rt.set_path_per_voice(cid, ["b", "long"], idx.astype(np.int32), voice_begin=s) == 0, rt.last_error()
            conv = [c for gr in rt.describe()["groups"] for c in gr["convolvers"]][0]
            assert conv["form"] == "per_channel" and conv["partitions"] == 18
        elif act == "shared":
            assert rt.set_path_per_voice(cid, ["c"], [0] * nv) == 0
            conv = [c for gr in rt.describe()["groups"] for c in gr["convolvers"]][0]
            assert conv["form"] == "shared" and conv["partitions"] == 18
        elif act == "json":
            assert rt.apply_instructions([[3, cid, "path", "a"], [5]]) == 0, rt.last_error()
            assert form(rt) == "shared"
        parts.append(stream(rt, x, RAGGED, t0=t, t1=stop)[0])
        if stop <= t2:
            pparts.append(stream(plain, x, RAGGED, t0=t, t1=stop)[0])
        t = stop
    out = np.concatenate(parts, axis=1)
    base = np.concatenate(pparts, axis=1)
    keep = np.setdiff1d(np.arange(nv), sub)
    assert np.array_equal(out[keep, :t2], base[keep])
    check(out[:, :t1], x[:, :t1], res["a"], "shared")
    # t1..t2: the reassigned channels from their restart, the others still on a
    hs = [res["a"]] * nv
    for j, c in enumerate(sub):
        hs[c] = res["long"] if idx[j] else res["b"]
    start = np.where(np.isin(np.arange(nv), sub), t1, 0)
    check(since(out[:, :t2], start), x[:, :t2], hs, "per_channel", start=start)
    check_silence(since(out[:, :t2], start), x[:, :t2] * (np.arange(t2)[None, :] >= start[:, None]), hs)
    # t2..t3: every channel restarted on c (shared form, R > S)
    check(since(out[:, :t3], t2), x[:, :t3], res["c"], "shared", start=t2)
    xs = x[:, :t3] * (np.arange(t3) >= t2)
    check_silence(since(out[:, :t3], t2), xs, res["c"])
    # t3..: a fresh convolver, its partition grid starting at t3
    check(out[:, t3:], x[:, t3:], res["a"], "shared")
    check_silence(out[:, t3:], x[:, t3:], res["a"])


# ---- 6. stage boundaries -----------------------------------------------------------------------------------------------------
def _spread(E, h):
    """Bound per block on |conv(d, h)| given |d| <= E per 512-sample block (Cauchy-Schwarz over the partitions of h)."""
    from scipy import signal as ssig
    hb = ce._block_norms(ce.trim(h).astype(np.float64)[None, :])
    t = np.sqrt(ce.P) * np.atleast_2d(E)
    t[:, 1:] += t[:, :-1].copy()
    return np.maximum(ssig.fftconvolve(t, hb, axes=-1)[:, :t.shape[-1]], 0.0).reshape(np.shape(E))


def within(got, want, tol, label):
    """Per block |got - want| <= tol (tol 0: exactly 0.0)."""
    r = ce.ratio(got, want, tol)
    assert r.max() <= 1.0, f"{label}: worst {r.max():.3g} x tolerance (channel {int(r.argmax())})"


def _blockmax(a):
    return ce.block_error(a, np.zeros_like(a))


@pytest.mark.parametrize("frm", ["shared", "per_channel"])
def test_dry_wet_and_series_against_a_float64_composition(frm):
    """wet/dry: 0.75 conv(2 x) + 0.25 (2 x) through K1 stages; series: conv_b(0.5 conv_a(x)).  Tolerance: C E_b of each
    convolver on its (exact) input, the first convolver's bound carried through the second, and one float rounding per K1 op."""
    nv = 9
    lead = 1024
    n = lead + 24 * ce.P
    x = inputs(POOL[:nv], n, lead)
    irs = {"a": ce.make_ir("lcg", 3000, seed=31), "b": ce.make_ir("flat", 1500, seed=32), "c": ce.make_ir("taps", 600, seed=33)}
    names = list(irs)
    ia = [0] * nv if frm == "shared" else [k % 3 for k in range(nv)]
    ib = [1] * nv if frm == "shared" else [(k + 1) % 3 for k in range(nv)]
    ha = [irs[names[i]] for i in ia]
    hb = [irs[names[i]] for i in ib]
    # dry / wet
    xin = el.mul(2.0, el.in_(0))
    wet = el.convolve({"path": "a", "key": "w"}, xin)
    rt = Runtime(SR, 512, nv, device=0)
    for k, v in irs.items():
        assert rt.add_shared_resource(k, v)
    assert rt.apply_instructions(el.render(el.add(el.mul(0.75, wet), el.mul(0.25, xin)))) == 0, rt.last_error()
    if frm == "per_channel":
        assert rt.set_path_per_voice(wet.id(), names, ia) == 0
    out, _ = stream(rt, x, RAGGED)
    x2 = (2.0 * x).astype(np.float32)
    w = ce.exact(x2, ha)
    want = 0.75 * w + 0.25 * x2.astype(np.float64)
    tol = 0.75 * ce.C * ce.bound(x2, ha) + 3 * ce.U * _blockmax(np.abs(0.75 * w) + np.abs(0.25 * x2))
    within(out, want, tol, "dry/wet")
    # two convolvers in series
    a = el.convolve({"path": "a", "key": "s1"}, el.in_(0))
    b = el.convolve({"path": "b", "key": "s2"}, el.mul(0.5, a))
    rt = Runtime(SR, 512, nv, device=0)
    for k, v in irs.items():
        assert rt.add_shared_resource(k, v)
    assert rt.apply_instructions(el.render(b)) == 0, rt.last_error()
    if frm == "per_channel":
        assert rt.set_path_per_voice(a.id(), names, ia) == 0 and rt.set_path_per_voice(b.id(), names, ib) == 0
    out, _ = stream(rt, x, RAGGED)
    y1 = ce.exact(x, ha)
    y2 = np.stack([ce.exact((0.5 * y1[c]), hb[c]) for c in range(nv)])
    E1 = ce.C * ce.bound(x, ha)
    # the second convolver's own error, the first one's carried through it, and the float32 rounding of its input
    E2 = np.stack([ce.C * ce.bound((0.5 * y1[c]).astype(np.float32), hb[c]) + _spread(0.5 * E1[c] + ce.U * _blockmax(0.5 * y1[c:c + 1])[0], hb[c])
                   for c in range(nv)])
    within(out, y2, 1.01 * E2, "series")                            # 1 %: the second bound is evaluated on the float32-rounded input


@pytest.mark.parametrize("frm", ["shared", "per_channel"])
def test_root_epilogue_voices_and_mix_bus(frm):
    """`convolve -> root` (the fused epilogue), more units than CTAs: every per-voice output against `exact`, and the mix bus against
    the float64 sum of the exact outputs with the bounds summed (plus the float summation of nv terms)."""
    nv = 2 * grid() + 3
    lead = 1024
    n = lead + 12 * ce.P
    x = inputs([(k, s + c) for c, (k, s) in enumerate(POOL[c % len(POOL)] for c in range(nv))], n, lead)
    res = {"a": ce.make_ir("lcg", 2500, seed=41), "b": ce.make_ir("flat", 800, seed=42)}
    rt, cid = engine(nv, res, "a")
    hs = [res["a"]] * nv
    if frm == "per_channel":
        idx = [(c // 3) % 2 for c in range(nv)]
        assert rt.set_path_per_voice(cid, ["a", "b"], idx) == 0
        hs = [res["ab"[i]] for i in idx]
    out, mix = stream(rt, x, RAGGED, want_mix=True)
    want = ce.exact(x, hs)
    E = ce.bound(x, hs)
    check(out, x, hs, frm, want=want, E=E)
    tol = ce.C * E.sum(axis=0) + nv * ce.U * _blockmax(np.abs(want).sum(axis=0))
    within(mix[None], want.sum(axis=0)[None], tol[None], "mix")
