"""GPU: voice resets (Runtime.reset_voices, elem_b200_reset_voices, K6 in reset_kernel.cu).

R1  Every family of tests/k1_families.py, interpreted and specialised, over the K1 tile geometries (_r1_params).  Every root sits behind
    an `el.z` with fadeInMs 0.  Runtime A resets a scattered set (the first voice, the last, a whole tile and lanes of another tile, passed unsorted
    with repeats) before a call that starts off a block boundary, once before FADE_END and once after it.  Voices outside the set are
    the same bits as an un-reset twin (a second copy of the voices in the same runtime); voices in the set are, from each reset on, the same bits as a fresh runtime B started at that
    sample time with the same per-voice values and inputs and cut into the same calls (the z makes sample 0 after the reset
    comparable despite B's one-sample root fade).  The mix bus equals its model after every call.  In the analysis family the queues
    are not polled before a reset, so a reset drops real pending readouts: after it, meter / snapshot / capture events of the reset
    voices are B's, and every event of the other voices is the twin's.
R2  Convolver: a reset is bit for bit set_path_per_voice with each voice's current IR, in the shared-IR and per-channel-IR forms and
    behind the fused convolve -> root epilogue.
R3  Props replay: rand restarts from the seed last set for the voice, once is re-armed iff it was ever armed, across a later group cut.
R4  Launch paths: one-voice groups (warp pipeline on and off), a reset with a COMMIT pending, process_offline after a reset, a reset
    while the specialised kernel is still compiling.
R5  One launch per non-empty call, none for an empty one.

ELEM_B200_CUTS_FULL=1 runs R1 in every family x geometry x build (by default a rotating subset).
"""
import copy
import os
import time

import numpy as np
import pytest

from elementary_b200 import Runtime, el, graphs
from events_common import canon
from k1_families import CALLS, FADE_END, FAMILIES, GEOMETRIES, N_VOICES, SR, BS, make_runtime
from mix_model import assert_mix, mix_model

pytestmark = pytest.mark.gpu
FULL = os.environ.get("ELEM_B200_CUTS_FULL") == "1"
STARTS = np.cumsum((0,) + CALLS)
RESET_CALLS = (2, 8)                      # before call 2 (sample 519, in the fade-in) and call 8 (sample 1145): off block boundaries
assert STARTS[RESET_CALLS[0]] < FADE_END < STARTS[RESET_CALLS[1]] and all(STARTS[c] % BS for c in RESET_CALLS)
EVENT_TYPES = ("meter", "snapshot", "capture")


def z_family(fam):
    f = copy.copy(fam)
    f.batch = el.Renderer(0.0).render(*[el.z(r) for r in fam.roots])
    return f


def reset_set(L, n=N_VOICES):
    """The first and last voice, a whole tile, and one or two lanes of the next tile (a partially reset tile)."""
    w = 1 if 2 * L <= n else 0
    s = {0, n - 1} | set(range(w * L, min((w + 1) * L, n)))
    base = (w + 1) * L
    s |= {v for v in ((base + 1, base + L - 2) if L >= 4 else (base + 1,)) if v < n}
    return sorted(s)


def passed_form(voices):
    """The list as passed: unsorted, with repeats."""
    v = list(reversed(voices))
    return v + v[:3]


def events_by_voice(rt, shift=0):
    """The polled events by voice; voices at or past `shift` (> 0) are reported as voice - shift (the twin half of a runtime)."""
    out = {}
    for e in rt.process_queued_events():
        v = e["event"]["voice"]
        if shift and v >= shift:
            e = {"type": e["type"], "event": dict(e["event"], voice=v - shift)}
            v -= shift
            out.setdefault(("twin", v), []).append(e)
        else:
            out.setdefault(v, []).append(e)
    return out


def run(fam, L, niter, build, inputs, resets=(), start=0, stop=len(CALLS), poll=False, twin=False):
    """Calls CALLS[start:stop] (sample STARTS[start] on); before call c in `resets`, resets those voices.  twin: the runtime holds a second
    copy of the N_VOICES voices behind the first, with the same values and inputs and never reset — the un-reset twin in the same launch.
    Returns the voices and, per call, the events by voice (poll: after every call except the one before a reset)."""
    n_voices = 2 * N_VOICES if twin else N_VOICES
    rt = make_runtime(fam, L, niter, build, n_voices=n_voices)
    if twin:
        fam.setup(rt, N_VOICES, N_VOICES)                  # voice N_VOICES + v gets voice v's keyed values and seeds
        inputs = None if inputs is None else np.concatenate([inputs, inputs])
    if start:
        rt.set_current_time(int(STARTS[start]))
    vs, evs = [], []
    for c in range(start, stop):
        n, s = CALLS[c], int(STARTS[c])
        if c in resets:
            assert rt.reset_voices(passed_form(resets[c])) == 0, rt.last_error()
        v, mix = rt.process_voices(None if inputs is None else inputs[:, :, s:s + n], fam.n_out, n)
        assert_mix(mix, mix_model(v, rt.describe()["groups"]), f"{fam.name} L={L} {build} call {c}")
        vs.append(v)
        evs.append(events_by_voice(rt, N_VOICES if twin else 0) if poll and c + 1 not in RESET_CALLS else None)
    if build != "interp":
        assert rt.describe()["groups"][0].get("spec_state") == 2
    return np.concatenate(vs, axis=2), evs


# The specialised arms by default: an NVRTC compile of 10 to 60 s each on an H100 host; the delay family carries the hazard of unequal
# write indices inside a tile, in a wide and a narrow geometry.
SPEC_DEFAULT = {("delay", 32, 0, "spec"), ("delay", 4, 0, "dense"), ("oscillators", 1, 4, "spec")}


def _r1_params():
    """Each family interpreted in two of the nine K1 geometries, rotated so that every geometry meets three or four families, and the
    specialised arms of SPEC_DEFAULT.  ELEM_B200_CUTS_FULL=1: every family x geometry x build."""
    out = []
    n = len(GEOMETRIES)
    for i, f in enumerate(FAMILIES):
        for gi, (L, niter) in enumerate(GEOMETRIES):
            if FULL or gi in ((2 * i) % n, (2 * i + 1) % n):
                out.append(pytest.param(f, L, niter, "interp", id=f"{f}-L{L}n{niter}-interp"))
            for build in ("spec", "dense"):
                if (build == "spec" or (L in (2, 4, 8, 16) and niter == 0)) and (FULL or (f, L, niter, build) in SPEC_DEFAULT):
                    out.append(pytest.param(f, L, niter, build, id=f"{f}-L{L}n{niter}-{build}"))
    return out


@pytest.mark.parametrize("family,tile_width,niter,build", _r1_params())
def test_reset_voices_restart_as_fresh_instances(family, tile_width, niter, build):
    fam = z_family(FAMILIES[family])
    L = tile_width
    inputs = None if not fam.n_in else np.stack([fam.inputs(fam, v, int(STARTS[-1])) for v in range(N_VOICES)])
    R = reset_set(L)
    others = [v for v in range(N_VOICES) if v not in R]
    poll = family == "analysis"
    both, ea = run(fam, L, niter, build, inputs, resets={c: R for c in RESET_CALLS}, poll=poll, twin=True)
    a, t = both[:N_VOICES], both[N_VOICES:]
    what = f"{family} L={L} niter={niter} {build}"
    assert np.array_equal(a[others], t[others], equal_nan=True), f"{what}: voices outside the reset set changed"
    for k, c in enumerate(RESET_CALLS):
        end = RESET_CALLS[k + 1] if k + 1 < len(RESET_CALLS) else len(CALLS)
        b, eb = run(fam, L, niter, build, inputs, start=c, stop=end, poll=poll, twin=True)   # same layout: same specialised kernel
        seg = slice(int(STARTS[c]), int(STARTS[end]))
        got, want = a[R][:, :, seg], b[R]
        if not np.array_equal(got, want, equal_nan=True):
            bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))[0]
            raise AssertionError(f"{what}: reset before call {c}: voice {R[bad[0]]} out {bad[1]} sample {bad[2]} after the reset: "
                                 f"{got[tuple(bad)]!r}, fresh runtime {want[tuple(bad)]!r}")
        if poll:
            for j in range(c, end):
                if ea[j] is None:
                    continue
                for v in R:
                    mine = canon([e for e in ea[j].get(v, []) if e["type"] in EVENT_TYPES])
                    fresh = canon([e for e in eb[j - c].get(v, []) if e["type"] in EVENT_TYPES])
                    assert mine == fresh, f"{what}: call {j} voice {v}: events differ from a fresh runtime's"
    if poll:
        for j in range(len(CALLS)):
            if ea[j] is not None:
                for v in others:
                    assert canon(ea[j].get(v, [])) == canon(ea[j].get(("twin", v), [])), f"{what}: call {j} voice {v}: events differ from the twin's"


# ---- R2: convolver ------------------------------------------------------------------------------------------------------

IR = np.asarray(graphs.lcg_ir(4097), dtype=np.float32)
IRS = {"a": IR * 2.0, "b": IR[:700], "c": IR[:1500] * 0.5}


@pytest.mark.parametrize("form", ["shared", "per_channel", "fused"])
def test_convolver_reset_equals_set_path_per_voice(form):
    nv, R = 19, [0, 3, 4, 9, 18]
    names = list(IRS)
    idx = [v % 3 for v in range(nv)] if form == "per_channel" else [0] * nv
    x = np.random.default_rng(5).uniform(-0.5, 0.5, size=(nv, 1, 9 * 512)).astype(np.float32)

    def make():
        rt = Runtime(SR, 512, nv, device=0)
        for k, v in IRS.items():
            assert rt.add_shared_resource(k, v)
        cv = el.convolve({"path": "a", "key": "cv"}, el.in_(0))
        assert rt.apply_instructions(el.render(cv if form == "fused" else el.mul(1.0, cv))) == 0, rt.last_error()
        if form == "per_channel":
            assert rt.set_path_per_voice(cv.id(), names, idx) == 0, rt.last_error()
        return rt, cv.id()

    (a, cid), (b, _) = make(), make()
    outs = []
    for rt, reset in ((a, True), (b, False)):
        vs, s = [], 0
        for c, n in enumerate((512, 300, 200, 512, 100, 450, 512, 512)):
            if c == 3 and reset:
                assert rt.reset_voices(R) == 0, rt.last_error()
            elif c == 3:   # set_path_per_voice addresses a contiguous range: the voices one by one
                for v in R:
                    assert rt.set_path_per_voice(cid, names, [idx[v]], v) == 0, rt.last_error()
            v, _ = rt.process_voices(x[:, :, s:s + n], 1, n)
            vs.append(v)
            s += n
        outs.append(np.concatenate(vs, axis=2))
    assert np.array_equal(outs[0], outs[1])
    conv = [c for g in a.describe()["groups"] for c in g.get("convolvers", [])]
    assert conv and conv[0]["form"] == ("per_channel" if form == "per_channel" else "shared"), conv


# ---- R3: props replay ---------------------------------------------------------------------------------------------------

def _props_runtime(nv=40, seeds=None, armed=None, **opts):
    rt = Runtime(SR, 512, nv, device=0, tile_width=8, **opts)
    r = el.rand(seed=11, key="rr")
    o = el.once({"arm": False, "key": "oo"}, el.in_(0))
    assert rt.apply_instructions(el.Renderer(0.0).render(el.z(r), el.z(o))) == 0, rt.last_error()
    if seeds is not None:
        assert rt.set_property_per_voice(r.id(), "seed", seeds) == 0
    for v in armed or ():
        assert rt.apply_instructions([[3, o.id(), "arm", True]], voices=(v, v + 1)) == 0
    return rt, r.id(), o.id()


def _gate(nv, n, period=100):
    x = np.zeros((nv, 1, n), np.float32)
    x[:, :, (np.arange(n) % period) < period // 2] = 1.0
    return x


def test_rand_and_once_replay_their_props_across_a_cut():
    nv, n = 40, 512
    seeds = [1000 + 37 * v for v in range(nv)]
    armed = [2, 9, 17, 33]
    a, rid, oid = _props_runtime(nv, seeds, armed)
    g = _gate(nv, 4 * n)
    for k in range(2):
        a.process_voices(g[:, :, k * n:(k + 1) * n], 2, n)
    # a new seed after rendering, then a reset: restarts from the new seed; a reset, then a new seed: the new seed
    assert a.set_property_per_voice(rid, "seed", [77, 78], 10) == 0
    assert a.apply_instructions([[0, 0x7E000001, "sin"]], voices=(16, nv)) == 0, a.last_error()   # cut: the shadows move along
    assert len(a.describe()["groups"]) == 2
    R = [2, 3, 9, 10, 11, 17, 33, 39]
    assert a.reset_voices(R) == 0, a.last_error()
    assert a.set_property_per_voice(rid, "seed", [5], 39) == 0
    got, _ = a.process_voices(g[:, :, :n], 2, n)
    seeds2 = list(seeds)
    seeds2[10], seeds2[11], seeds2[39] = 77, 78, 5
    b, _, _ = _props_runtime(nv, seeds2, armed)
    want, _ = b.process_voices(g[:, :, :n], 2, n)
    assert np.array_equal(got[R], want[R])
    assert want[2, 1].any() and not want[3, 1].any()          # armed voices fire after the reset, never-armed ones stay silent


# ---- R4: launch paths ---------------------------------------------------------------------------------------------------

def _synth(nv, **opts):
    rt = Runtime(SR, 512, nv, device=0, **opts)
    assert rt.apply_instructions(graphs.subsynth32()) == 0, rt.last_error()
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(nv)])
    assert rt.set_property_per_voice(ida, "value", f0) == 0
    assert rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    return rt


def _fresh_after(rt_make, at, n_blocks):
    b = rt_make()
    b.set_current_time(at)
    got, _ = b.render_voices(n_blocks, 1)
    return got


def _same_after_fade(got, want, voices):
    """SUBSYNTH32's roots fade in over 20 ms in the fresh runtime (root fades are not restarted by a reset): bits from FADE_END on."""
    assert np.array_equal(got[voices][:, :, FADE_END:], want[voices][:, :, FADE_END:])
    assert np.abs(got[voices][:, :, FADE_END:]).max() > 0


@pytest.mark.parametrize("stages", [0, 3])
def test_one_voice_groups_in_the_many_groups_launch(stages):
    nv = 6
    def make():
        rt = _synth(nv, pipeline_stages=stages)
        for v in range(1, nv):   # one group per voice
            assert rt.apply_instructions([[0, 0x7E000000 + v, "sin"]], voices=(v, nv)) == 0, rt.last_error()
        return rt
    a = make()
    assert len(a.describe()["groups"]) == nv
    a.render_voices(3, 1)
    assert a.reset_voices([4, 1]) == 0, a.last_error()
    got, _ = a.render_voices(3, 1)
    want = _fresh_after(make, 3 * 512, 3)
    _same_after_fade(got, want, [1, 4])


def test_reset_with_a_commit_pending_and_then_offline():
    nv, R = 24, [0, 5, 6, 23]
    a = _synth(nv, tile_width=4)
    a.render_voices(2, 1)
    assert a.apply_instructions(graphs.subsynth32()[-2:]) == 0        # [[4, roots], [5]]: a program is queued
    assert a.reset_voices(R) == 0, a.last_error()
    _, got = a.process_offline(None, 1, 3 * 512, want_mix=False, want_voices=True)
    want = _fresh_after(lambda: _synth(nv, tile_width=4), 2 * 512, 3)
    _same_after_fade(got, want, R)


def test_reset_while_the_specialised_kernel_compiles():
    nv, R = 64, [3, 40, 41]
    a = _synth(nv, specialize=1)
    a.render_voices(1, 1)
    assert a.reset_voices(R) == 0
    got, _ = a.render_voices(3, 1)
    want = _fresh_after(lambda: _synth(nv, specialize=0), 512, 3)
    # the specialised kernel may take over during these blocks; its filters need not match the interpreter's bits (DESIGN.md section 4)
    g, w = got[R][:, :, FADE_END:].astype(np.float64), want[R][:, :, FADE_END:].astype(np.float64)
    assert np.abs(g - w).max() <= 1e-5 * np.abs(w).max() and np.abs(w).max() > 0
    # no compile is left running behind the test (the process may end right after it)
    t0 = time.monotonic()
    while a.describe()["groups"][0].get("spec_state", 2) == 0 and time.monotonic() - t0 < 300:
        time.sleep(0.05)
    assert a.describe()["groups"][0].get("spec_state") != 0


# ---- R5: launch count ---------------------------------------------------------------------------------------------------

def test_one_launch_per_call():
    a = _synth(64)
    a.render_voices(1, 1)
    l0 = a.kernel_launches
    assert a.reset_voices([]) == 0
    assert a.kernel_launches == l0
    assert a.reset_voices(list(range(0, 64, 3)) + [5, 5]) == 0
    assert a.kernel_launches == l0 + 1
