"""elem_b200_poll_readouts and elem_b200_process_offline_readouts on plan-only engines (no GPU): every argument error returns its code
(-2, NodeNotFound, InvalidPropertyType) and changes nothing; a well-formed call fails with -1 because the engine cannot render or read
the device; the Python wrappers pass shapes and NULL pointers through."""
import ctypes as C

import numpy as np
import pytest

from elementary_b200 import Runtime, el
from elementary_b200.runtime import READOUT_DEVICE, _f32p

BS, V = 64, 8
METER = el.meter({"name": "m"}, el.in_(0))
SNAP = el.snapshot({"name": "s"}, el.train(10.0), el.in_(0))
CONST = el.const(0.25, key="k")
SCOPE = el.scope({"name": "sc"}, el.in_(0))
SAMPLE = el.sample({"path": "buf"}, el.train(2.0))
GRAPH = el.render(METER, el.add(SNAP, CONST), SCOPE, SAMPLE)
M, S, K, SC, SA = METER.id(), SNAP.id(), CONST.id(), SCOPE.id(), SAMPLE.id()


@pytest.fixture()
def rt():
    r = Runtime(48000.0, BS, V, device=-1)
    assert r.add_shared_resource("buf", np.ones(100, np.float32))
    assert r.apply_instructions(GRAPH) == 0
    return r


def _state(rt):
    return rt.describe(), [rt.snapshot(v) for v in range(V)], [rt.program_words(v).tolist() for v in range(V)]


def _poll(rt, node, vb=0, count=V, a=True, b=True, fresh=True, flags=0):
    bufs = [np.zeros(max(1, count), np.float32), np.zeros(max(1, count), np.float32), np.zeros(max(1, count), np.uint8)]
    ptrs = [x.ctypes.data if want else None for x, want in zip(bufs, (a, b, fresh))]
    return rt._lib.elem_b200_poll_readouts(rt._h, node, vb, count, *ptrs, flags)


def _offline(rt, nodes, vb=0, count=V, a=True, b=True, fresh=True, n=100, n_out=1, num_nodes=None):
    ids = np.asarray(nodes, np.int32)
    blocks = max(1, -(-n // BS))
    bufs = [np.zeros(max(1, ids.size * blocks * max(1, count)), dt) for dt in (np.float32, np.float32, np.uint8)]
    ptrs = [x.ctypes.data if want else None for x, want in zip(bufs, (a, b, fresh))]
    m = np.zeros((max(1, n_out), max(1, n)), np.float32)
    mix_ptrs = (_f32p * max(1, n_out))(*[m[i].ctypes.data_as(_f32p) for i in range(max(1, n_out))])
    return rt._lib.elem_b200_process_offline_readouts(rt._h, None, 0, None, mix_ptrs, None, n_out, n, 0, None,
                                                      ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.size if num_nodes is None else num_nodes,
                                                      vb, count, *ptrs)


POLL_ERRORS = [
    (dict(vb=-1), -2), (dict(vb=V - 2, count=3), -2), (dict(count=-1), -2), (dict(vb=V + 1, count=0), -2),
    (dict(a=False), -2), (dict(fresh=False), -2), (dict(a=False, flags=READOUT_DEVICE), -2),
    (dict(node=12345), 2), (dict(node=K), 5), (dict(node=SC), 5), (dict(node=SA), 5),
]


@pytest.mark.parametrize("case,code", POLL_ERRORS, ids=["begin-negative", "past-end", "count-negative", "empty-past-end", "null-a",
                                                        "null-fresh", "null-a-device", "missing-node", "const", "scope", "sample"])
def test_poll_errors_change_nothing(rt, case, code):
    case = dict(case)
    node = case.pop("node", M)
    before = _state(rt)
    assert _poll(rt, node, **case) == code
    assert _state(rt) == before


OFFLINE_ERRORS = [
    (dict(nodes=[]), -2), (dict(nodes=[M], num_nodes=0), -2), (dict(nodes=[M, S, M]), -2),
    (dict(count=0), -2), (dict(count=-1), -2), (dict(a=False), -2), (dict(fresh=False), -2), (dict(vb=V - 1, count=2), -2),
    (dict(vb=-1), -2), (dict(n_out=0), -2), (dict(n_out=4097), -2),
    (dict(nodes=[M, 777]), 2), (dict(nodes=[S, K]), 5), (dict(nodes=[SC]), 5), (dict(nodes=[SA]), 5),
]


@pytest.mark.parametrize("case,code", OFFLINE_ERRORS, ids=["no-nodes", "num-nodes-0", "repeated", "count-0", "count-negative", "null-a",
                                                           "null-fresh", "past-end", "begin-negative", "nout-0", "nout-4097",
                                                           "missing-node", "const", "scope", "sample"])
def test_offline_errors_render_nothing(rt, case, code):
    case = dict(case)
    nodes = case.pop("nodes", [M])
    before = _state(rt)
    assert _offline(rt, nodes, **case) == code
    assert _state(rt) == before and rt.current_time() == 0


def test_node_missing_in_one_of_two_groups():
    rt = Runtime(48000.0, BS, V, device=-1)
    assert rt.apply_instructions(el.render(METER), (0, 4)) == 0
    assert rt.apply_instructions(el.render(el.meter({"name": "other"}, el.in_(0))), (4, 8)) == 0
    before = _state(rt)
    assert _poll(rt, M, 0, V) == 2 and _poll(rt, M, 2, 4) == 2
    assert _offline(rt, [M], 2, 4) == 2
    assert _state(rt) == before
    assert _poll(rt, M, 0, 4) == -1                 # the first group alone has it
    assert _offline(rt, [M], 1, 3) == -1


def test_meter_in_one_group_snapshot_in_another():
    rt = Runtime(48000.0, BS, V, device=-1)
    batch = el.render(METER)
    assert rt.apply_instructions(batch, (0, 4)) == 0
    assert rt.apply_instructions([[0, x[1], "snapshot"] if x[:1] == [0] and x[1] == M else x for x in batch], (4, 8)) == 0
    assert rt.node_type(M, 0) == "meter" and rt.node_type(M, 4) == "snapshot"
    before = _state(rt)
    assert _poll(rt, M, 0, V) == 5 and _offline(rt, [M], 2, 4) == 5
    assert _state(rt) == before
    assert _poll(rt, M, 4, 4) == -1


@pytest.mark.parametrize("node", [M, S])
@pytest.mark.parametrize("vb,count,flags", [(0, V, 0), (3, 2, 0), (1, 7, READOUT_DEVICE)])
def test_valid_polls_need_a_device(rt, node, vb, count, flags):
    assert _poll(rt, node, vb, count, flags=flags) == -1
    assert "plan-only" in rt.last_error()
    assert _poll(rt, node, vb, count, b=False, flags=flags) == -1


def test_empty_poll_is_a_no_op(rt):
    assert _poll(rt, M, 3, 0) == 0
    assert _poll(rt, M, V, 0, a=False, b=False, fresh=False) == 0
    assert _poll(rt, K, 0, 0) == 0                  # no voice group in the range: nothing to check


@pytest.mark.parametrize("nodes,vb,count,n", [([M], 0, V, 100), ([S, M], 2, 3, 0), ([M], 7, 1, 64)])
def test_valid_offline_calls_need_a_device(rt, nodes, vb, count, n):
    assert _offline(rt, nodes, vb, count, n=n) == -1
    assert "plan-only" in rt.last_error()
    assert _offline(rt, nodes, vb, count, b=False, n=n) == -1


class _Recorder:
    """Stands in for the library: records the arguments of the readout calls and answers with a code."""

    def __init__(self, lib, code):
        self._lib, self.code, self.calls = lib, code, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in ("elem_b200_poll_readouts", "elem_b200_process_offline_readouts"):
            return fn

        def rec(*args):
            self.calls.append((name, args))
            return self.code
        return rec


def test_wrappers_pass_shapes_and_nulls_through(rt):
    rec = _Recorder(rt._lib, 0)
    rt._lib = rec
    out = rt.poll_readouts(M, voices=(2, 7))
    assert set(out) == {"min", "max", "fresh"} and all(x.shape == (5,) for x in out.values())
    assert out["fresh"].dtype == np.uint8 and out["min"].dtype == np.float32
    name, args = rec.calls[-1]
    assert args[1:4] == (M, 2, 5) and all(args[4:7]) and args[7] == 0
    out = rt.poll_readouts(S)
    assert set(out) == {"data", "fresh"} and out["data"].shape == (V,)
    rt.poll_readouts_device(S, 0x1000, None, 0x2000, voices=(1, 3))
    assert rec.calls[-1][1][1:] == (S, 1, 2, 0x1000, None, 0x2000, READOUT_DEVICE)
    rt.poll_readouts_device(M, 0x1000, 0x3000, 0x2000)
    assert rec.calls[-1][1][1:] == (M, 0, V, 0x1000, 0x3000, 0x2000, READOUT_DEVICE)
    mix, ov, ro = rt.process_offline(num_samples=3 * BS + 5, readouts=[S, M], readout_voices=(1, 4))
    name, args = rec.calls[-1]
    assert name == "elem_b200_process_offline_readouts" and args[11:14] == (2, 1, 3)
    assert list(ro) == [S, M]
    assert set(ro[S]) == {"data", "fresh"} and set(ro[M]) == {"min", "max", "fresh"}
    assert all(x.shape == (4, 3) for d in ro.values() for x in d.values())
    assert mix.shape == (1, 3 * BS + 5) and ov is None
    rec.code = -2
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.poll_readouts(M)
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.poll_readouts_device(M, 0, None, 0)


def test_wrappers_against_the_library(rt):
    with pytest.raises(RuntimeError, match=r"rc=-1 .*plan-only"):
        rt.poll_readouts(M, voices=(0, 3))
    with pytest.raises(RuntimeError, match=r"rc=5 "):
        rt.poll_readouts(K)
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.poll_readouts_device(M, 0, None, 0)
    with pytest.raises(RuntimeError, match=r"rc=-1 .*plan-only"):
        rt.process_offline(num_samples=10, readouts=[M, S])
    with pytest.raises(RuntimeError, match=r"rc=2 "):
        rt.process_offline(num_samples=10, readouts=[4242])
    with pytest.raises(ValueError):
        rt.process_offline(num_samples=10, readouts=[M], on_event=lambda *a: None)
    assert rt.node_type(M) == "meter" and rt.node_type(S, V - 1) == "snapshot" and rt.node_type(99) is None
