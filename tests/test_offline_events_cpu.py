"""elem_b200_process_offline_events on a plan-only engine (no GPU): every argument error returns -2 before anything is rendered,
including a NULL callback and a voice range out of bounds; a well-formed call fails like elem_b200_process_offline does (-1, the
engine cannot render); Runtime.process_offline(on_event=...) passes both through."""
import ctypes as C

import numpy as np
import pytest

from elementary_b200 import Runtime, graphs
from elementary_b200.runtime import BLOCK_EVENT_CB, _f32p

BS, V = 64, 4
CALLED = []
CB = BLOCK_EVENT_CB(lambda block, type_, js, user: CALLED.append(block))


@pytest.fixture()
def rt():
    r = Runtime(48000.0, BS, V, device=-1)
    assert r.apply_instructions(graphs.subsynth32()) == 0
    CALLED.clear()
    return r


def _call(rt, n_in=0, shared=False, per_voice=False, n_out=1, n=100, vb=0, ve=-1, cb=CB):
    keep = []
    in_ptrs = vin = None
    if shared:
        a = np.zeros((max(1, n_in), n), np.float32); keep.append(a)
        in_ptrs = (_f32p * max(1, n_in))(*[a[i].ctypes.data_as(_f32p) for i in range(max(1, n_in))])
    if per_voice:
        a = np.zeros((V, max(1, n_in), n), np.float32); keep.append(a)
        vin = a.ctypes.data_as(_f32p)
    m = np.zeros((max(1, n_out), n), np.float32)
    mix_ptrs = (_f32p * max(1, n_out))(*[m[i].ctypes.data_as(_f32p) for i in range(max(1, n_out))])
    return rt._lib.elem_b200_process_offline_events(rt._h, in_ptrs, n_in, vin, mix_ptrs, None, n_out, n, 0, None, vb, ve,
                                                    cb if cb is not None else BLOCK_EVENT_CB(), None)


@pytest.mark.parametrize("case", [
    dict(n_in=1, shared=True, per_voice=True), dict(n_in=2), dict(n_out=0), dict(n_out=4097),
    dict(cb=None), dict(vb=-1), dict(vb=V + 1, ve=-1), dict(vb=0, ve=V + 1), dict(vb=3, ve=2), dict(cb=None, n=0),
], ids=["both-inputs", "nin-without-pointer", "nout-0", "nout-4097", "null-callback", "begin-negative", "begin-past-end",
        "end-past-end", "end-before-begin", "null-callback-n0"])
def test_argument_errors_return_bad_argument(rt, case):
    assert _call(rt, **case) == -2
    assert rt.current_time() == 0 and not CALLED


@pytest.mark.parametrize("case", [dict(), dict(vb=1, ve=3), dict(vb=2, ve=2), dict(vb=V, ve=-1), dict(n=0), dict(n_in=1, shared=True)],
                         ids=["all", "range", "empty-range", "begin-at-end", "n0", "shared-in"])
def test_valid_calls_need_a_device(rt, case):
    assert _call(rt, **case) == -1
    assert "plan-only" in rt.last_error() and not CALLED


def test_wrapper_passes_errors_through(rt):
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.process_offline(num_samples=10, on_event=lambda *a: None, event_voices=(3, 1))
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.process_offline(num_samples=10, num_outputs=0, on_event=lambda *a: None)
    with pytest.raises(RuntimeError, match=r"rc=-1 "):
        rt.process_offline(num_samples=10, on_event=lambda *a: None, event_voices=(0, 2))
