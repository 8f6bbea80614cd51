"""Runtime.process_offline (elem_b200_process_offline): whole signals rendered in one call, with inputs, the mix bus and per-voice
outputs, through the offline chunk loop.

Every test compares BIT FOR BIT against a twin runtime with the same setup stepped block by block: process() for the mix,
process_voices() for per-voice outputs (and the mix with per-voice inputs), on zero-padded full blocks, truncated to the call's length.

O1  Every K1 matrix family (tests/k1_families.py), fed per-voice and shared inputs, in a rotating subset of geometries, interpreted and
    specialised (ELEM_B200_MATRIX_FULL=1: every geometry), plus the family contract against the reference.
O2  numSamples 1, bs - 1, bs, bs + 1, 37 bs + 100 with chunkBlocks 1, 2, 3 and the default; 700 then 300 samples continue at the block
    boundary.
O3  The mix equals its model (tests/mix_model.py, tests/wide_mix_model.py) at nOut 1, 2, 8, 9 and 16, including a group that fades out
    between calls (its channel is +0.0 in later chunks: no stale slot contents), and 1250 one-voice stems, pipelined and not.
O4  convolve fed by a shared input, by per-voice inputs with per-channel IRs, and in the fused convolve -> root form.
O5  Many batched voice groups past the root fade-in: the steady-state fast path runs with inputs.
O6  time / metro with userData NULL and set, the engine clock after the call, and the events polled after the call.
O7  The reference's jest replays (tests/jest_common.py) that read no events, one process_offline call per OfflineRenderer.process.
"""
import os

import numpy as np
import pytest

import jest_common
from elementary_b200 import Runtime, el
from jest_common import compare, replay_all
from k1_families import BS, CALLS, FAMILIES, GEOMETRIES, SR, check_family, make_runtime, reference
from mix_model import assert_mix
from wide_mix_model import engine_mix_model

FULL = os.environ.get("ELEM_B200_MATRIX_FULL") == "1"


def bits(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_same(got, want, what):
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    if not np.array_equal(bits(got), bits(want)):
        bad = np.argwhere(bits(got) != bits(want))
        raise AssertionError(f"{what}: {len(bad)} samples differ, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} != {want[tuple(bad[0])]!r}")


def _pad(x, n_blocks, bs):
    if x is None:
        return None
    out = np.zeros(x.shape[:-1] + (n_blocks * bs,), np.float32)
    out[..., :x.shape[-1]] = x
    return out


def twin(rt, n, n_out, inputs=None, voice_inputs=None, voices=True, mix="voices", sample_time=None):
    """Block by block on zero-padded full blocks: (mix [n_out, n] | None, voices [V, n_out, n] | None).  mix = "process": the mix of
    process() (shared inputs); "voices": the mix of process_voices() (inputs broadcast to every voice when shared)."""
    bs = rt.block_size
    nb = -(-n // bs)
    x, xv = _pad(inputs, nb, bs), _pad(voice_inputs, nb, bs)
    ms, vs = [], []
    for k in range(nb):
        sl = slice(k * bs, (k + 1) * bs)
        t = None if sample_time is None else sample_time + k * bs
        if mix == "process":
            ms.append(rt.process(None if x is None else x[:, sl], n_out, bs, sample_time=t))
            continue
        assert t is None
        vin = xv[:, :, sl] if xv is not None else (None if x is None else np.broadcast_to(x[:, sl], (rt.num_voices,) + x[:, sl].shape))
        v, m = rt.process_voices(vin, n_out, bs, want_voices=voices, want_mix=mix is not None)
        ms.append(m)
        vs.append(v)
    m = np.concatenate(ms, axis=1)[:, :n] if mix is not None else None
    v = np.concatenate(vs, axis=2)[:, :, :n] if voices and vs else None
    return m, v


# ---- O1: every K1 family ------------------------------------------------------------------------------------------------------

def _family_params():
    out = []
    for i, name in enumerate(FAMILIES):
        geoms = GEOMETRIES if FULL else [GEOMETRIES[(i + 4 * j) % len(GEOMETRIES)] for j in range(2)]
        for j, (L, niter) in enumerate(geoms):
            build = "interp" if j % 2 == 0 else "spec"
            out.append(pytest.param(name, L, niter, build, id=f"{name}-L{L}-n{niter}-{build}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("family,tile_width,niter,build", _family_params())
def test_family_offline(family, tile_width, niter, build):
    fam = FAMILIES[family]
    n = sum(CALLS)                             # the matrix's input length (the same designed inputs); the last block is zero-padded
    calls = (BS,) * (n // BS) + (n % BS,)      # the reference renders the full blocks, then the rest
    ref, inputs = reference(fam, calls=calls)
    inputs = None if inputs is None else inputs[:, :, :n]
    what = f"{family} L={tile_width} niter={niter} {build}"
    # per-voice inputs: mix and per-voice outputs against process_voices, and the family contract against the reference
    a, b = (make_runtime(fam, tile_width, niter, build) for _ in range(2))
    mix, v = a.process_offline(voice_inputs=inputs, num_samples=n, num_outputs=fam.n_out, want_voices=True, chunk_blocks=2)
    tm, tv = twin(b, n, fam.n_out, voice_inputs=inputs)
    assert_same(v, tv, what + " voices")
    assert_same(mix, tm, what + " mix")
    check_family(fam, v, mix, ref[:, :, :n], inputs, what)
    # shared inputs (voice 0's, broadcast): the mix against process(), per-voice outputs against process_voices
    shared = None if inputs is None else np.ascontiguousarray(inputs[0])
    c, d, e = (make_runtime(fam, tile_width, niter, build) for _ in range(3))
    mix, v = c.process_offline(shared, num_samples=n, num_outputs=fam.n_out, want_voices=True, chunk_blocks=3)
    tm, _ = twin(d, n, fam.n_out, inputs=shared, mix="process")
    _, tv = twin(e, n, fam.n_out, inputs=shared, mix=None)
    assert_same(mix, tm, what + " shared-input mix")
    assert_same(v, tv, what + " shared-input voices")


# ---- O2: lengths and chunk sizes --------------------------------------------------------------------------------------------

def _filter_rt(V=21, L=4, bs=BS):
    rt = Runtime(SR, bs, V, device=0, tile_width=L)
    x = el.add(el.in_(0), el.mul(0.25, el.in_(1)))
    g = el.svf({"mode": "lowpass"}, el.const(800.0, key="fc"), el.const(1.5, key="q"), el.add(x, el.z(x)))
    assert rt.apply_instructions(el.render(g, el.delay({"size": 3000}, el.const(700.0, key="dl"), 0.5, x))) == 0, rt.last_error()
    assert rt.set_property_per_voice(el.const(0, key="fc").id(), "value", 300.0 + 40.0 * np.arange(V)) == 0
    assert rt.set_property_per_voice(el.const(0, key="dl").id(), "value", 100.0 + 3.0 * np.arange(V)) == 0
    return rt


def _noise(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, BS - 1, BS, BS + 1, 37 * BS + 100])
@pytest.mark.parametrize("chunk", [1, 2, 3, 0])
@pytest.mark.parametrize("per_voice", [False, True], ids=["shared", "per-voice"])
def test_lengths_and_chunks(n, chunk, per_voice):
    a, b, c = _filter_rt(), _filter_rt(), _filter_rt()
    what = f"n={n} chunk={chunk} per_voice={per_voice}"
    if per_voice:
        x = _noise((a.num_voices, 2, n), n)
        mix, v = a.process_offline(voice_inputs=x, num_outputs=2, want_voices=True, chunk_blocks=chunk)
        tm, tv = twin(b, n, 2, voice_inputs=x)
        assert_same(mix, tm, what + " mix")
    else:
        x = _noise((2, n), n)
        mix, v = a.process_offline(x, num_outputs=2, want_voices=True, chunk_blocks=chunk)
        tm, _ = twin(b, n, 2, inputs=x, mix="process")
        _, tv = twin(c, n, 2, inputs=x, mix=None)
        assert_same(mix, tm, what + " mix")
    assert_same(v, tv, what + " voices")
    assert a.current_time() == b.current_time() == -(-n // BS) * BS


@pytest.mark.gpu
def test_consecutive_calls_continue_at_the_block_boundary():
    a, b = _filter_rt(), _filter_rt()
    x = _noise((2, 1000), 7)
    m1, _ = a.process_offline(x[:, :700], num_outputs=2, chunk_blocks=1)
    m2, _ = a.process_offline(x[:, 700:], num_outputs=2, chunk_blocks=1)
    t1, _ = twin(b, 700, 2, inputs=x[:, :700], mix="process")
    t2, _ = twin(b, 300, 2, inputs=x[:, 700:], mix="process")
    assert_same(m1, t1, "first call")
    assert_same(m2, t2, "second call")
    assert a.current_time() == b.current_time() == 3 * BS       # two blocks for 700 samples, one for 300


# ---- O3: the mix bus and its model --------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("layout,n_out", [("one group", 1), ("one group", 2), ("one group", 8), ("one group", 9), ("one group", 16),
                                          ("gaps, fade-out, conv", 8), ("gaps, fade-out, conv", 16)])
def test_mix_equals_the_model(layout, n_out):
    from test_wide_mix_gpu import LAYOUTS, _setup
    V = LAYOUTS[layout]
    a, b = Runtime(SR, BS, V, device=0), Runtime(SR, BS, V, device=0)
    faded = _setup(a, layout, n_out)
    _setup(b, layout, n_out)
    n1, n2 = 5 * BS + 3, 9 * BS
    for k, n in enumerate((n1, n2)):
        if k == 1:
            for vb, ve in faded:           # the group fades out during the second call: its slots held sound in the first
                for rt in (a, b):
                    assert rt.apply_instructions([[4, []], [5]], voices=(vb, ve)) == 0, rt.last_error()
        mix, v = a.process_offline(num_samples=n, num_outputs=n_out, want_voices=n_out <= 8, chunk_blocks=2)
        want_m, want_v = twin(b, n, n_out, voices=True)
        what = f"{layout} nOut={n_out} call {k}"
        if v is not None:
            assert_same(v, want_v, what + " voices")
        assert_same(mix, want_m, what + " mix (process_voices)")
        groups = b.describe()["groups"]
        nb = -(-n // BS)
        for blk in range(nb):                                           # the model block by block (each block is one K2 / K2w)
            s = slice(blk * BS, min(n, (blk + 1) * BS))
            assert_mix(mix[:, s], engine_mix_model(want_v[:, :, s], groups, n_out), f"{what} block {blk}")
        if k == 1 and faded:
            (vb, ve), = faded
            assert not want_v[vb:ve, :, -2 * BS:].any()
            quiet = [c for c in range(n_out) if not want_v[:vb, c].any() and not want_v[ve:, c].any()]
            assert quiet and not mix[quiet, -2 * BS:].any(), (quiet, "a faded channel kept stale chunk contents")


@pytest.mark.gpu
@pytest.mark.parametrize("opts", [{}, {"pipeline_stages": 0}], ids=["pipelined", "unpipelined"])
def test_1250_stems(opts):
    from test_wide_mix_gpu import LAYOUTS, _setup
    V = LAYOUTS["stems"]
    a, b = Runtime(SR, BS, V, device=0, **opts), Runtime(SR, BS, V, device=0, **opts)
    _setup(a, "stems", 1250)
    _setup(b, "stems", 1250)
    n = 6 * BS + 11
    for k in range(2):                                                  # the second call runs on the steady fast path
        mix, _ = a.process_offline(num_samples=n, num_outputs=1250, chunk_blocks=4)
        want, _ = twin(b, n, 1250, mix="process")
        assert_same(mix, want, f"stems call {k}")
        assert np.abs(mix).max() > 0
    assert all(g["mix_channels"] == [i] for i, g in enumerate(a.describe()["groups"]))


# ---- O4: convolve -----------------------------------------------------------------------------------------------------------

def _irs():
    r = np.random.default_rng(3)
    return {f"ir{i}": (r.standard_normal(1500 + 700 * i) * np.exp(-np.arange(1500 + 700 * i) / 400.0)).astype(np.float32)
            for i in range(3)}


def _conv_rt(V, form):
    rt = Runtime(SR, BS, V, device=0)
    for name, data in _irs().items():
        assert rt.add_shared_resource(name, data)
    cv = el.convolve({"path": "ir0", "key": "cv"}, el.in_(0))
    g = cv if form == "fused" else el.add(el.mul(0.5, cv), el.in_(0))
    assert rt.apply_instructions(el.render(g)) == 0, rt.last_error()
    if form == "per-voice IRs":
        assert rt.set_path_per_voice(cv.id(), ["ir0", "ir1", "ir2"], [v % 3 for v in range(V)]) == 0, rt.last_error()
    return rt


@pytest.mark.gpu
@pytest.mark.parametrize("form,per_voice", [("plain", False), ("per-voice IRs", True), ("fused", False), ("fused", True)])
def test_convolve(form, per_voice):
    V, n = 12, 11 * BS + 200
    a, b, c = (_conv_rt(V, form) for _ in range(3))
    if per_voice:
        x = _noise((V, 1, n), 11)
        mix, v = a.process_offline(voice_inputs=x, want_voices=True, chunk_blocks=3)
        tm, tv = twin(b, n, 1, voice_inputs=x)
    else:
        x = _noise((1, n), 12)
        mix, v = a.process_offline(x, want_voices=True, chunk_blocks=3)
        tm, _ = twin(b, n, 1, inputs=x, mix="process")
        _, tv = twin(c, n, 1, inputs=x, mix=None)
    assert_same(v, tv, f"{form} voices")
    assert_same(mix, tm, f"{form} mix")
    assert np.abs(v).max() > 0


# ---- O5: the steady-state fast path with inputs --------------------------------------------------------------------------

def _batched_rt(n_groups=40):
    rt = Runtime(SR, BS, 3 * n_groups, device=0)
    for i in range(n_groups):
        rt.set_option("tile_width", (1, 2, 4)[i % 3])
        g = el.add(el.mul(el.in_(i % 2), 0.5 + 0.01 * i), el.pole(el.const(0.9, key=f"p{i}"), el.in_(0)))
        r = el.Renderer().render(g)
        assert rt.apply_instructions(r, voices=(3 * i, 3 * i + 3)) == 0, rt.last_error()
    return rt


@pytest.mark.gpu
@pytest.mark.parametrize("per_voice", [False, True], ids=["shared", "per-voice"])
def test_steady_fast_path_with_inputs(per_voice):
    a, b = _batched_rt(), _batched_rt()
    n = 8 * BS
    for k in range(3):                                                  # calls 2 and 3 run past the root fade-in
        if per_voice:
            x = _noise((a.num_voices, 2, n), 20 + k)
            mix, v = a.process_offline(voice_inputs=x, want_voices=True, chunk_blocks=(1, 3, 0)[k])
            tm, tv = twin(b, n, 1, voice_inputs=x)
        else:
            x = _noise((2, n), 20 + k)
            mix, v = a.process_offline(x, want_voices=True, chunk_blocks=(1, 3, 0)[k])
            tm, tv = twin(b, n, 1, inputs=x)
        assert_same(v, tv, f"call {k} voices")
        assert_same(mix, tm, f"call {k} mix")


# ---- O6: sample clock and events --------------------------------------------------------------------------------------------

def _clock_rt():
    rt = Runtime(SR, BS, 3, device=0)
    g = [el.time(), el.mul(el.metro({"interval": 30}), 1.0), el.meter({"name": "m"}, el.in_(0))]
    assert rt.apply_instructions(el.render(*g)) == 0, rt.last_error()
    return rt


@pytest.mark.gpu
@pytest.mark.parametrize("t0", [None, 123_456_789_000])
def test_time_metro_clock_and_events(t0):
    a, b = _clock_rt(), _clock_rt()
    for rt in (a, b):
        rt.set_current_time(1000)
    n = 4 * BS + 300
    x = _noise((1, n), 5)
    mix, _ = a.process_offline(x, num_outputs=3, sample_time=t0, chunk_blocks=2)
    tm, _ = twin(b, n, 3, inputs=x, mix="process", sample_time=t0)
    assert_same(mix, tm, f"t0={t0}")
    assert a.current_time() == b.current_time() == (1000 if t0 is None else t0) + 5 * BS
    ea, eb = a.process_queued_events(), b.process_queued_events()
    assert ea == eb and any(e["type"] == "meter" for e in ea) and any(e["type"] == "metro" for e in ea), (ea[:4], eb[:4])


# ---- O7: the reference's jest replays ---------------------------------------------------------------------------------------

class _OfflineEngine:
    def __init__(self, sr, bs):
        self.rt = Runtime(sr, bs, 2, device=0)

    def apply(self, batch):
        return self.rt.apply_instructions(batch)

    def process_queued_events(self):
        return [e for e in self.rt.process_queued_events() if e["event"]["voice"] == 0]

    def set_current_time(self, t):
        self.rt.set_current_time(t)


class _OfflineRenderer(jest_common.OfflineRenderer):
    """OfflineRenderer.process as one process_offline call (no events are polled inside it)."""

    def process(self, inps, n):
        x = None
        if self.n_in:
            x = np.zeros((self.n_in, n), dtype=np.float32)
            for c, buf in enumerate(inps):
                seg = np.asarray(buf, dtype=np.float32)[:n]
                x[c, :len(seg)] = seg
        mix, v = self.engine.rt.process_offline(voice_inputs=None if x is None else np.stack([x, x]), num_samples=n,
                                                num_outputs=self.n_out, want_mix=False, want_voices=True)
        self.events.extend(self.engine.process_queued_events())
        return v[0]


@pytest.mark.gpu
def test_jest_replays(monkeypatch):
    import json
    snap = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jest_snapshots.json")))["snapshots"]
    monkeypatch.setattr(jest_common, "OfflineRenderer", _OfflineRenderer)
    produced = replay_all(lambda sr, bs: _OfflineEngine(sr, bs))
    produced = {k: v for k, v in produced.items() if not k.startswith("events")}     # events are polled per block by those tests
    assert len(produced) >= 10
    bad = compare(produced, snap)
    assert not bad, "\n".join(bad)
