"""GPU: meter / snapshot readouts as arrays (elem_b200_poll_readouts, elem_b200_process_offline_readouts) against the JSON poll.

Two runtimes are built the same way and fed the same blocks.  One is polled with process_queued_events, the other with poll_readouts
over the same voices: for every poll and voice, fresh marks exactly the voices with an event, and a / b hold the event's numbers as
float32.  The offline form is checked against a process() + poll_readouts loop block for block, and against process_offline_events."""
import json

import numpy as np
import pytest

from elementary_b200 import Runtime, el, graphs
from elementary_b200.runtime import FLAG_MIX
from events_common import noise, scenarios

pytestmark = pytest.mark.gpu
SR, BS = 48000.0, 512
READOUT_SCEN = [s for s in scenarios() if s["name"].startswith(("meter", "snapshot", "several"))]


def analysis_nodes(graph):
    """[(node id, type, source name)] of the meter / snapshot nodes of a graph, each once."""
    out, seen = [], set()

    def walk(n):
        if not isinstance(n, el.Node) or n.id() in seen:
            return
        seen.add(n.id())
        if n.type in ("meter", "snapshot"):
            out.append((n.id(), n.type, n.props.get("name")))
        for c in n.children:
            walk(c)
    for g in graph:
        walk(g)
    return out


def voice_inputs(nv, n_in, k):
    if not n_in:
        return None
    return np.stack([np.stack([noise(BS, 1000 * k + 7 * v + c) for c in range(n_in)]) for v in range(nv)])


def json_readouts(events, nodes, vb, ve):
    """The JSON poll's events as the arrays poll_readouts fills: {node id: (a, b, fresh)} for voices [vb, ve)."""
    by_source = {(t, s): i for i, t, s in nodes}
    assert len(by_source) == len(nodes), "sources must tell the nodes apart"
    out = {i: (np.zeros(ve - vb, np.float32), np.zeros(ve - vb, np.float32), np.zeros(ve - vb, np.uint8)) for i, _, _ in nodes}
    for e in events:
        ev = e["event"]
        a, b, fresh = out[by_source[(e["type"], ev["source"])]]
        i = ev["voice"] - vb
        assert 0 <= i < ve - vb and not fresh[i], f"unexpected or repeated event {e}"
        fresh[i] = 1
        num = (lambda x: np.float32(np.nan) if x is None else np.float32(x))
        if e["type"] == "meter":
            a[i], b[i] = num(ev["min"]), num(ev["max"])
        else:
            a[i] = num(ev["data"])
    return out


def same_readouts(got, want, what):
    """got: poll_readouts' dict; want: (a, b, fresh) from json_readouts."""
    a, b, fresh = want
    assert np.array_equal(got["fresh"], fresh), f"{what}: fresh {got['fresh']} != {fresh}"
    m = fresh == 1
    ga, gb = (got["min"], got["max"]) if "min" in got else (got["data"], None)
    assert np.array_equal(ga[m], a[m], equal_nan=True), f"{what}: {ga[m]} != {a[m]}"
    if gb is not None:
        assert np.array_equal(gb[m], b[m], equal_nan=True), f"{what}: {gb[m]} != {b[m]}"
    assert not ga[~m].any() and (gb is None or not gb[~m].any()), f"{what}: values written where nothing is fresh"


def array_poll(rt, nodes, vb, ve):
    return {i: rt.poll_readouts(i, voices=(vb, ve)) for i, _, _ in nodes}


def check_twins(make, nodes, steps, ranges, n_in, n_out):
    """steps: ("block", k) | ("poll", range index) | ("do", fn(rt)).  Runs both twins; compares every poll.  Returns the fresh count."""
    js, ar = make(), make()
    nv = js.num_voices
    fresh = 0
    for st in steps:
        if st[0] == "block":
            x = voice_inputs(nv, n_in, st[1])
            for r in (js, ar):
                r.process_voices(x, n_out, BS)
        elif st[0] == "do":
            for r in (js, ar):
                st[1](r)
        else:
            vb, ve = ranges[st[1]]
            want = json_readouts(js.process_queued_events(voices=(vb, ve)), nodes, vb, ve)
            got = array_poll(ar, nodes, vb, ve)
            for i, t, s in nodes:
                same_readouts(got[i], want[i], f"{t} {s} voices {vb}..{ve}")
                fresh += int(want[i][2].sum())
    # what either poll left behind is the same: one more block, then a JSON poll of every voice on both
    x = voice_inputs(nv, n_in, 999)
    after = []
    for r in (js, ar):
        r.process_voices(x, n_out, BS)
        after.append(sorted(json.dumps(e, sort_keys=True) for e in r.process_queued_events()))
    assert after[0] == after[1]
    return fresh


@pytest.mark.parametrize("tile_width", [1, 2, 4, 32, 0], ids=["L1", "L2", "L4", "L32", "auto"])
@pytest.mark.parametrize("sc", READOUT_SCEN, ids=[s["name"] for s in READOUT_SCEN])
def test_scenarios_match_the_json_poll(sc, tile_width):
    nv = 35
    batch = el.render(*sc["graph"])
    nodes = analysis_nodes(sc["graph"])

    def make():
        rt = Runtime(SR, BS, nv, device=0, **({"tile_width": tile_width} if tile_width else {}))
        assert rt.apply_instructions(batch) == 0, rt.last_error()
        return rt
    ranges = [(0, nv), (3, 30), (5, 6), (17, 35)]    # all, inside tiles at both ends, one voice, to the end
    steps = []
    for k in range(sc["blocks"]):
        steps.append(("block", k))
        if sc["poll"](k):
            steps += [("poll", 1), ("poll", 2), ("poll", 3), ("poll", 0)]
    fresh = check_twins(make, nodes, steps, ranges, sc["n_in"], len(sc["graph"]))
    assert (fresh == 0) == bool(sc.get("silent"))


def _cut_runtime(tile_width, graph):
    """35 voices in two voice groups, cut at voice 20."""
    rt = Runtime(SR, BS, 35, device=0, tile_width=tile_width)
    rt.renderer = el.Renderer()             # later renders send only what changed, as the reference's renderer does
    batch = rt.renderer.render(*graph)
    assert rt.apply_instructions(batch, (0, 20)) == 0
    assert rt.apply_instructions(batch, (20, 35)) == 0
    return rt


@pytest.mark.parametrize("tile_width", [4, 32])
def test_range_across_a_voice_group_cut_with_resets_and_an_inactive_root(tile_width):
    m = el.meter({"name": "m"}, el.mul(0.5, el.in_(0)))
    s = el.snapshot({"name": "s"}, el.train(210.0), el.in_(0))
    other = el.mul(0.25, el.cycle(220.0))
    graph = (m, s)
    nodes = analysis_nodes(graph)
    ranges = [(0, 35), (13, 27), (18, 22)]
    steps = [("block", 0), ("poll", 1), ("block", 1), ("poll", 2), ("poll", 0)]
    steps += [("do", lambda r: r.reset_voices([14, 19, 20, 33]) == 0 or pytest.fail("reset")), ("poll", 1),
              ("block", 2), ("do", lambda r: r.reset_voices([2, 21])), ("poll", 1), ("poll", 0)]
    # the meter's root goes inactive (a render without it): nothing is fresh and its queue stays for later
    steps += [("do", lambda r: r.apply_instructions(r.renderer.render(other, s)) == 0 or pytest.fail(r.last_error())),
              ("block", 3), ("block", 4), ("block", 5), ("poll", 1), ("poll", 0)]
    steps += [("do", lambda r: r.apply_instructions(r.renderer.render(*graph)) == 0 or pytest.fail(r.last_error())),
              ("block", 6), ("poll", 2)]
    fresh = check_twins(lambda: _cut_runtime(tile_width, graph), nodes, steps, ranges, 1, 2)
    assert fresh > 0


def test_inactive_root_leaves_the_queue_for_a_json_poll():
    m = el.meter({"name": "m"}, el.in_(0))
    rt = Runtime(SR, BS, 9, device=0, tile_width=4)
    ren = el.Renderer()
    assert rt.apply_instructions(ren.render(m)) == 0
    x = voice_inputs(9, 1, 0)
    rt.process_voices(x, 1, BS)
    rt.process_voices(x, 1, BS)            # the root has faded in
    assert rt.apply_instructions(ren.render(el.cycle(100.0))) == 0
    rt.process_voices(voice_inputs(9, 1, 1), 1, BS)
    got = rt.poll_readouts(m.id())
    assert not got["fresh"].any() and not got["min"].any()
    assert rt.process_queued_events() == []              # not reachable from an active root: no JSON event either
    assert rt.apply_instructions(ren.render(m)) == 0     # active again, without a block in between: the queue is still there
    ev = rt.process_queued_events(voices=(2, 7))
    assert sorted(e["event"]["voice"] for e in ev) == [2, 3, 4, 5, 6]
    got = rt.poll_readouts(m.id())
    assert got["fresh"].tolist() == [1, 1, 0, 0, 0, 0, 0, 1, 1]


def test_json_and_array_polls_take_turns():
    """On one runtime the polls of overlapping ranges alternate; a twin polls everything as JSON at the same points.  Each poll sees what
    the polls before it left, and the nodes it does not address keep their events."""
    graph = (el.meter({"name": "a"}, el.snapshot({"name": "b"}, el.train(97.0), el.in_(0))), el.meter({"name": "c"}, el.cycle(440.0)))
    nodes = analysis_nodes(graph)
    ids = {s: i for i, _, s in nodes}
    batch = el.render(*graph)
    nv = 40
    mixed, twin = (Runtime(SR, BS, nv, device=0, tile_width=8) for _ in range(2))
    for r in (mixed, twin):
        assert r.apply_instructions(batch) == 0
    total = 0
    for k in range(6):
        x = voice_inputs(nv, 1, k)
        for r in (mixed, twin):
            r.process_voices(x, 2, BS)
        everything = twin.process_queued_events()
        rest = list(everything)

        def take(pred):
            nonlocal rest
            hit = [e for e in rest if pred(e)]
            rest = [e for e in rest if not pred(e)]
            return hit

        def in_range(lo, hi):
            return lambda e: lo <= e["event"]["voice"] < hi

        # array: meter "a" over [3, 21)
        want = json_readouts(take(lambda e: e["event"]["source"] == "a" and in_range(3, 21)(e)), nodes, 3, 21)
        same_readouts(mixed.poll_readouts(ids["a"], voices=(3, 21)), want[ids["a"]], f"block {k} array a")
        # JSON over [10, 30): everything there except what the array poll drained
        got = mixed.process_queued_events(voices=(10, 30))
        want_js = take(in_range(10, 30))
        assert sorted(json.dumps(e, sort_keys=True) for e in got) == sorted(json.dumps(e, sort_keys=True) for e in want_js)
        # array: snapshot "b" over [0, 40)
        want = json_readouts(take(lambda e: e["event"]["source"] == "b"), nodes, 0, nv)
        same_readouts(mixed.poll_readouts(ids["b"]), want[ids["b"]], f"block {k} array b")
        # JSON over everything: the rest
        got = mixed.process_queued_events()
        assert sorted(json.dumps(e, sort_keys=True) for e in got) == sorted(json.dumps(e, sort_keys=True) for e in rest)
        total += len(everything)
    assert total > 0


def test_device_mode_loop_equals_host_mode():
    torch = pytest.importorskip("torch")
    nv, blocks = 300, 64
    gate = el.train(el.const(35.0, key="rate"))
    graph = (el.meter({"name": "m"}, el.mul(el.const(1.0, key="amp"), el.cycle(el.const(100.0, key="f")))),
             el.snapshot({"name": "s"}, gate, el.phasor(3.0)))
    nodes = analysis_nodes(graph)
    batch = el.render(*graph)
    f_id, amp_id, rate_id = el.const(100.0, key="f").id(), el.const(1.0, key="amp").id(), el.const(35.0, key="rate").id()

    def make():
        rt = Runtime(SR, BS, nv, device=0)
        assert rt.apply_instructions(batch) == 0
        v = np.arange(nv)
        assert rt.set_const_table([f_id, amp_id, rate_id], np.stack([50.0 + 7.0 * v, 0.5 + (v % 5) * 0.1, 20.0 + (v % 41) * 3.0])) == 0
        return rt
    dev, host = make(), make()
    vb, ve = 7, 291
    n = ve - vb
    a = {i: torch.full((blocks, n), -1.0, device="cuda:0") for i, _, _ in nodes}
    b = torch.full((blocks, n), -1.0, device="cuda:0")
    fresh = {i: torch.full((blocks, n), 7, dtype=torch.uint8, device="cuda:0") for i, _, _ in nodes}
    torch.cuda.synchronize()
    want = []
    for k in range(blocks):
        dev.enqueue_block(0, 2, BS, FLAG_MIX)
        for i, t, _ in nodes:
            dev.poll_readouts_device(i, a[i][k].data_ptr(), b[k].data_ptr() if t == "meter" else None, fresh[i][k].data_ptr(), voices=(vb, ve))
        host.enqueue_block(0, 2, BS, FLAG_MIX)
        want.append(array_poll(host, nodes, vb, ve))
    dev.synchronize()
    fresh_seen = 0
    for i, t, _ in nodes:
        f = fresh[i].cpu().numpy()
        ga = a[i].cpu().numpy()
        for k in range(blocks):
            w = want[k][i]
            assert np.array_equal(f[k], w["fresh"]), f"{t} block {k}"
            m = f[k] == 1
            assert np.array_equal(ga[k][m], (w["min"] if t == "meter" else w["data"])[m])
            assert (ga[k][~m] == -1.0).all(), "a written where nothing is fresh"
            if t == "meter":
                gb = b.cpu().numpy()[k]
                assert np.array_equal(gb[m], w["max"][m]) and (gb[~m] == -1.0).all()
            fresh_seen += int(m.sum())
    assert fresh_seen > blocks * n


@pytest.mark.parametrize("n_voices", [4096, 131072])
def test_meter_readouts_are_each_voices_block_min_and_max(n_voices):
    batch = el.render(el.meter({"name": "v"}, graphs.subsynth32_graph()))
    meter = analysis_nodes((el.meter({"name": "v"}, graphs.subsynth32_graph()),))[0][0]
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(n_voices)])
    rt = Runtime(SR, BS, n_voices, device=0)
    assert rt.apply_instructions(batch) == 0
    assert rt.set_property_per_voice(ida, "value", f0) == 0
    assert rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    for _ in range(2):                      # the root's 20 ms fade-in ends inside the second block
        rt.process_voices(None, 1, BS, want_voices=False, want_mix=False)
    ov, _ = rt.process_voices(None, 1, BS, want_mix=False)
    got = rt.poll_readouts(meter)
    assert got["fresh"].all()
    assert np.array_equal(got["min"], ov[:, 0].min(axis=1)) and np.array_equal(got["max"], ov[:, 0].max(axis=1))
    again = rt.poll_readouts(meter)
    assert not again["fresh"].any()


def _offline_graph():
    gate = el.le(el.phasor(31.0), 0.3)
    return (el.meter({"name": "m"}, el.mul(0.5, el.in_(0))), el.snapshot({"name": "s"}, el.train(160.0), el.in_(0)),
            el.capture({"name": "c"}, gate, el.in_(0)), el.scope({"name": "sc", "size": 700}, el.in_(0)),
            el.meter({"name": "m2"}, el.cycle(330.0)))


@pytest.mark.parametrize("chunk,n", [(1, 7 * BS), (3, 7 * BS + 300), (0, 19 * BS - 5)], ids=["chunk1", "chunk3-ragged", "default-ragged"])
def test_offline_readouts_equal_the_poll_loop(chunk, n):
    graph = _offline_graph()
    nodes = analysis_nodes(graph)
    listed = [nodes[2][0], nodes[0][0]]                   # m2, then m; the snapshot is left alone
    batch = el.render(*graph)
    nv = 30

    def make():
        rt = Runtime(SR, BS, nv, device=0, tile_width=4)
        assert rt.apply_instructions(batch, (0, 20)) == 0
        assert rt.apply_instructions(batch, (20, nv)) == 0
        return rt
    off, loop, plain = make(), make(), make()
    x = np.stack([noise(n, 11)])
    vb, ve = 6, 27
    m1, _, ro = off.process_offline(x, 5, readouts=listed, readout_voices=(vb, ve), chunk_blocks=chunk)
    m0, _ = plain.process_offline(x, 5, chunk_blocks=chunk)
    assert np.array_equal(m1.view(np.uint32), m0.view(np.uint32)), "readouts changed the mix"
    blocks = -(-n // BS)
    for k in range(blocks):
        seg = np.zeros((1, BS), np.float32)
        part = x[:, k * BS:(k + 1) * BS]
        seg[:, :part.shape[1]] = part
        mk = loop.process(seg, 5, BS)
        width = min(BS, n - k * BS)
        assert np.array_equal(mk[:, :width].view(np.uint32), m1[:, k * BS:k * BS + width].view(np.uint32)), f"mix block {k}"
        for i in listed:
            w = loop.poll_readouts(i, voices=(vb, ve))
            for key in w:
                assert np.array_equal(ro[i][key][k].view(np.uint32) if key != "fresh" else ro[i][key][k],
                                      w[key].view(np.uint32) if key != "fresh" else w[key]), f"node {i} {key} block {k}"
    assert all(ro[i]["fresh"].any() for i in listed)
    # what was left behind: the snapshot's queue was not polled, the meters' were; a JSON poll of every voice agrees on both
    after = [sorted(json.dumps(e, sort_keys=True) for e in r.process_queued_events()) for r in (off, loop)]
    assert after[0] == after[1]


@pytest.mark.parametrize("chunk", [1, 3, 0])
def test_offline_readouts_equal_offline_events(chunk):
    graph = _offline_graph()
    nodes = analysis_nodes(graph)
    batch = el.render(*graph)
    nv, n = 26, 9 * BS - 100

    def make():
        rt = Runtime(SR, BS, nv, device=0, tile_width=8)
        assert rt.apply_instructions(batch) == 0
        return rt
    ev_rt, ro_rt = make(), make()
    x = np.stack([np.stack([noise(n, 31 * v)]) for v in range(nv)])
    per_block = [[] for _ in range(-(-n // BS))]
    m0, v0 = ev_rt.process_offline(voice_inputs=x, num_outputs=5, want_voices=True, chunk_blocks=chunk,
                                   on_event=lambda k, t, e: per_block[k].append({"type": t, "event": e}))
    m1, v1, ro = ro_rt.process_offline(voice_inputs=x, num_outputs=5, want_voices=True, chunk_blocks=chunk,
                                       readouts=[i for i, _, _ in nodes])
    assert np.array_equal(m0.view(np.uint32), m1.view(np.uint32)) and np.array_equal(v0.view(np.uint32), v1.view(np.uint32))
    for k, evs in enumerate(per_block):
        want = json_readouts([e for e in evs if e["type"] in ("meter", "snapshot")], nodes, 0, nv)
        for i, t, s in nodes:
            same_readouts({key: arr[k] for key, arr in ro[i].items()}, want[i], f"block {k} {t} {s}")


def test_snapshot_never_writes_b_through_the_c_abi():
    """For a snapshot, b is never written: in host mode, in device mode and offline, even where the staging record or the chunk log held
    a meter's b values just before (the meter is polled first into the same buffers, and the offline calls swap the node order)."""
    import ctypes as C
    torch = pytest.importorskip("torch")
    from elementary_b200.runtime import READOUT_DEVICE, _f32p
    graph = (el.meter({"name": "m"}, el.in_(0)), el.snapshot({"name": "s"}, el.train(300.0), el.in_(0)))
    (mid, _, _), (sid, _, _) = analysis_nodes(graph)
    nv, sentinel = 21, np.float32(-7.5)
    rt = Runtime(SR, BS, nv, device=0, tile_width=4)
    assert rt.apply_instructions(el.render(*graph)) == 0
    lib, h = rt._lib, rt._h
    seen = 0
    for k in range(4):
        rt.process_voices(voice_inputs(nv, 1, k), 2, BS)
        a, b, f = np.zeros(nv, np.float32), np.zeros(nv, np.float32), np.zeros(nv, np.uint8)
        assert lib.elem_b200_poll_readouts(h, mid, 0, nv, a.ctypes.data, b.ctypes.data, f.ctypes.data, 0) == 0
        assert f.all() and (b >= a).all()
        a, b, f = np.zeros(nv, np.float32), np.full(nv, sentinel), np.zeros(nv, np.uint8)
        assert lib.elem_b200_poll_readouts(h, sid, 0, nv, a.ctypes.data, b.ctypes.data, f.ctypes.data, 0) == 0
        assert (b == sentinel).all(), "host mode wrote b for a snapshot"
        seen += int(f.sum())
    assert seen > 0
    rt.process_voices(voice_inputs(nv, 1, 9), 2, BS)
    da, db, df = (torch.zeros(nv, device="cuda:0"), torch.full((nv,), float(sentinel), device="cuda:0"),
                  torch.zeros(nv, dtype=torch.uint8, device="cuda:0"))
    assert lib.elem_b200_poll_readouts(h, sid, 0, nv, da.data_ptr(), db.data_ptr(), df.data_ptr(), READOUT_DEVICE) == 0
    rt.synchronize()
    assert df.any().item() and (db == float(sentinel)).all().item(), "device mode wrote b for a snapshot"
    blocks = 5
    m = np.zeros((2, blocks * BS), np.float32)
    mix = (_f32p * 2)(*[m[i].ctypes.data_as(_f32p) for i in range(2)])
    x = np.stack([noise(blocks * BS, 5)])
    inp = (_f32p * 1)(x[0].ctypes.data_as(_f32p))
    for order in ([mid, sid], [sid, mid]):
        ids = np.asarray(order, np.int32)
        a, b, f = np.zeros((2, blocks, nv), np.float32), np.full((2, blocks, nv), sentinel), np.zeros((2, blocks, nv), np.uint8)
        assert lib.elem_b200_process_offline_readouts(h, inp, 1, None, mix, None, 2, blocks * BS, 2, None,
                                                      ids.ctypes.data_as(C.POINTER(C.c_int32)), 2, 0, nv,
                                                      a.ctypes.data, b.ctypes.data, f.ctypes.data) == 0
        js, jm = order.index(sid), order.index(mid)
        assert f[js].any() and (b[js] == sentinel).all(), f"offline wrote b for a snapshot (order {order})"
        assert f[jm].all() and (b[jm] >= a[jm]).all()
