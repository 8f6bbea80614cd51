"""GPU: elem_b200_process_offline_events (Runtime.process_offline(on_event=...)) against its twin — a second runtime built the same
way that runs process() / process_voices() and process_queued_events(voices=...) once per block.  For every block the event lists
must be equal (type and event, in order; fft included: both run the same host transform), the audio bit for bit what
process_offline returns without events, and one more block with a full poll afterwards must give the same events on both runtimes
(the state left behind is the same)."""
import json

import numpy as np
import pytest

from elementary_b200 import Runtime, el, graphs
from events_common import noise, scenarios
from k1_families import BUILDS, FAMILIES, GEOMETRIES, family_inputs

pytestmark = pytest.mark.gpu
SR, BS = 48000.0, 512
SCEN = scenarios()


def _voice_inputs(n_voices, n_in, n, seed=0):
    if not n_in:
        return None
    return np.stack([np.stack([noise(n, 7919 * seed + 7 * v + c) for c in range(n_in)]) for v in range(n_voices)])


def _evts(lst):
    return [(t, json.dumps(e)) for t, e in lst]


def _twin_block(rt, x, k, n_out, voices, t0):
    """One block of the twin: process_voices (per-voice inputs) or process (shared clock), then the poll."""
    seg = None
    if x is not None:
        seg = np.zeros(x.shape[:-1] + (BS,), np.float32)
        part = x[..., k * BS:(k + 1) * BS]
        seg[..., :part.shape[-1]] = part
    if t0 is None:
        rt.process_voices(seg, n_out, BS)
    else:
        rt.process(seg, n_out, BS, sample_time=t0 + k * BS)
    return _evts((e["type"], e["event"]) for e in rt.process_queued_events(voices=voices))


def check_against_twin(make, n_out, n, x=None, chunk=0, voices=None, t0=None, pre=0, want_voices=True):
    """make() -> a fresh runtime; x: per-voice inputs [voice, n_in, n] (or, with t0, shared inputs [n_in, n]).  `pre` un-polled
    process() blocks run on every runtime first, so the call starts with a backlog.  Returns the per-block event lists."""
    off, twin, plain = make(), make(), make()
    nv = off.num_voices
    for k in range(pre):
        xp = _voice_inputs(nv, 0 if x is None else x.shape[-2], BS, seed=100 + k) if t0 is None else None
        for r in (off, twin, plain):
            r.process_voices(xp, n_out, BS)
    shared = t0 is not None
    kw = dict(num_outputs=n_out, num_samples=n, chunk_blocks=chunk, want_voices=want_voices, sample_time=t0)
    if x is not None:
        kw["inputs" if shared else "voice_inputs"] = x
    blocks = -(-n // BS)
    got = [[] for _ in range(blocks)]
    order = []

    def on_event(k, t, e):
        order.append(k)
        got[k].append((t, json.dumps(e)))

    m1, v1 = off.process_offline(on_event=on_event, event_voices=voices, **kw)
    m0, v0 = plain.process_offline(**kw)
    assert np.array_equal(m1.view(np.uint32), m0.view(np.uint32)), "events changed the mix"
    if want_voices:
        assert np.array_equal(v1.view(np.uint32), v0.view(np.uint32)), "events changed the per-voice outputs"
    assert order == sorted(order)
    want = [_twin_block(twin, x, k, n_out, voices, t0) for k in range(blocks)]
    for k in range(blocks):
        assert got[k] == want[k], f"block {k}: {str(got[k])[:400]} != {str(want[k])[:400]}"
    # the state left behind: one more block, then a full poll, on both
    after = []
    for r in (off, twin):
        r.process_voices(_voice_inputs(nv, 0 if x is None or shared else x.shape[-2], BS, seed=999), n_out, BS)
        after.append(_evts((e["type"], e["event"]) for e in r.process_queued_events()))
    assert after[0] == after[1], f"state after the call differs: {str(after[0])[:300]} != {str(after[1])[:300]}"
    return got


@pytest.mark.parametrize("pre", [0, 21], ids=["fresh", "backlog"])
@pytest.mark.parametrize("sc", SCEN, ids=[s["name"] for s in SCEN])
def test_scenarios_match_the_poll_per_block_twin(sc, pre):
    batch = el.render(*sc["graph"])

    def make():
        rt = Runtime(SR, BS, 35, device=0, tile_width=16)
        assert rt.apply_instructions(batch) == 0, rt.last_error()
        return rt
    n = sc["blocks"] * BS
    got = check_against_twin(make, len(sc["graph"]), n, _voice_inputs(35, sc["n_in"], n), pre=pre)
    assert any(got) != bool(sc.get("silent"))


def _geoms():
    out = []
    for L, niter in GEOMETRIES:
        out.append(pytest.param(L, niter, "interp", id=f"L{L}n{niter}-interp"))
        out.append(pytest.param(L, niter, "spec", id=f"L{L}n{niter}-spec"))
    return out


@pytest.mark.parametrize("L,niter,build", _geoms())
def test_analysis_family_in_every_geometry(L, niter, build):
    fam = FAMILIES["analysis"]
    n = 9 * BS

    def make():
        opts = dict(BUILDS[build], tile_width=L)
        if niter:
            opts["niter"] = niter
        rt = Runtime(SR, BS, 45, device=0, **opts)
        assert rt.apply_instructions(fam.batch) == 0, rt.last_error()
        fam.setup(rt)
        return rt
    got = check_against_twin(make, fam.n_out, n, family_inputs(fam, 45, n), chunk=3, pre=2)
    kinds = {t for blk in got for t, _ in blk}
    assert {"meter", "snapshot", "scope", "capture", "fft"} <= kinds, kinds


@pytest.mark.parametrize("voices", [None, (5, 29), (17, 18), (9, 9)], ids=["all", "across-tiles", "one", "empty"])
def test_voice_ranges(voices):
    fam = FAMILIES["analysis"]
    n = 8 * BS

    def make():
        rt = Runtime(SR, BS, 45, device=0, tile_width=8)
        assert rt.apply_instructions(fam.batch) == 0
        fam.setup(rt)
        return rt
    got = check_against_twin(make, fam.n_out, n, family_inputs(fam, 45, n), voices=voices, pre=3)
    seen = {json.loads(e)["voice"] for blk in got for _, e in blk}
    if voices is None:
        assert seen == set(range(45))
    elif voices[0] == voices[1]:
        assert not seen
    else:
        assert seen <= set(range(*voices)) and seen


@pytest.mark.parametrize("chunk,n", [(1, 7 * BS), (3, 7 * BS), (0, 19 * BS), (50, 7 * BS), (3, 4 * BS + 300), (0, 0)],
                         ids=["chunk1", "chunk3", "default", "chunk-past-blocks", "ragged", "empty"])
def test_chunking_and_lengths(chunk, n):
    g = (el.meter({"name": "m"}, el.mul(0.5, el.in_(0))), el.capture({"name": "c"}, el.le(el.phasor(31.0), 0.3), el.in_(0)),
         el.scope({"name": "s", "size": 700}, el.in_(0)))
    batch = el.render(*g)

    def make():
        rt = Runtime(SR, BS, 12, device=0)
        assert rt.apply_instructions(batch) == 0
        return rt
    got = check_against_twin(make, 3, n, _voice_inputs(12, 1, n), chunk=chunk)
    assert len(got) == -(-n // BS)


@pytest.mark.parametrize("t0", [None, 123456])
def test_sample_time_with_metro(t0):
    batch = el.render(el.metro({"name": "tick", "interval": 25.0}), el.meter({"name": "t"}, el.time()))

    def make():
        rt = Runtime(SR, BS, 6, device=0)
        assert rt.apply_instructions(batch) == 0
        return rt
    got = check_against_twin(make, 2, 9 * BS, None, t0=t0, chunk=4, want_voices=False)
    assert any(t == "metro" for blk in got for t, _ in blk)


def test_several_voice_groups():
    ir = (np.exp(-np.arange(900) / 90.0) * noise(900, 3)).astype(np.float32)
    gate = el.le(el.phasor(23.0), 0.4)
    parts = [
        ((0, 10), el.render(el.meter({"name": "g0"}, el.mul(0.5, el.in_(0))))),
        ((10, 20), el.render(el.add(el.scope({"name": "g1", "size": 600}, el.in_(0)), el.capture({"name": "g1c"}, gate, el.in_(0))))),
        ((20, 30), el.render(el.mul(0.25, el.in_(0)))),
        ((30, 40), el.render(el.meter({"name": "gone"}, el.in_(0)))),
        ((40, 48), el.render(el.convolve({"path": "ir"}, el.meter({"name": "g4"}, el.in_(0))))),
    ]

    def make():
        rt = Runtime(SR, BS, 48, device=0)
        assert rt.add_shared_resource("ir", ir)
        for voices, b in parts:
            assert rt.apply_instructions(b, voices) == 0, rt.last_error()
        assert rt.apply_instructions(el.render(el.mul(0.5, el.cycle(330.0))), (30, 40)) == 0    # the meter's root fades out
        return rt
    n = 8 * BS
    got = check_against_twin(make, 1, n, _voice_inputs(48, 1, n), chunk=3, pre=1)
    seen = {(json.loads(e)["source"], json.loads(e)["voice"] // 10) for blk in got for _, e in blk}
    assert not any(s == "gone" for s, _ in seen)
    assert {s for s, _ in seen} >= {"g0", "g1", "g1c", "g4"}


def test_many_voices_each_under_a_meter():
    n_voices, blocks = 4096, 16
    batch = el.render(el.meter({"name": "v"}, graphs.subsynth32_graph()))
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(n_voices)])

    def make():
        rt = Runtime(SR, BS, n_voices, device=0)
        assert rt.apply_instructions(batch) == 0
        assert rt.set_property_per_voice(ida, "value", f0) == 0
        assert rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
        return rt
    got = check_against_twin(make, 1, blocks * BS, None, want_voices=False)
    assert all(len(blk) == n_voices for blk in got)
