"""elem_b200_process_offline on a plan-only engine (no GPU): every argument error returns -2 before anything is rendered, a valid
call returns -1 (a plan-only engine cannot render), and Runtime.process_offline passes shapes and NULLs through as documented."""
import ctypes as C

import numpy as np
import pytest

from elementary_b200 import Runtime, graphs
from elementary_b200.runtime import _f32p

BS, V = 64, 4


@pytest.fixture()
def rt():
    r = Runtime(48000.0, BS, V, device=-1)
    assert r.apply_instructions(graphs.subsynth32()) == 0
    return r


def _call(rt, n_in=0, shared=False, per_voice=False, mix=True, voices=False, n_out=1, n=100, chunk=0, t0=None):
    keep = []
    in_ptrs = vin = mix_ptrs = vout = None
    if shared:
        a = np.zeros((max(1, n_in), n), np.float32); keep.append(a)
        in_ptrs = (_f32p * max(1, n_in))(*[a[i].ctypes.data_as(_f32p) for i in range(max(1, n_in))])
    if per_voice:
        a = np.zeros((V, max(1, n_in), n), np.float32); keep.append(a)
        vin = a.ctypes.data_as(_f32p)
    if mix:
        m = np.zeros((max(1, n_out), n), np.float32); keep.append(m)
        mix_ptrs = (_f32p * max(1, n_out))(*[m[i].ctypes.data_as(_f32p) for i in range(max(1, n_out))])
    if voices:
        o = np.zeros((V, max(1, n_out), n), np.float32); keep.append(o)
        vout = o.ctypes.data_as(_f32p)
    user = None if t0 is None else C.byref(C.c_int64(t0))
    return rt._lib.elem_b200_process_offline(rt._h, in_ptrs, n_in, vin, mix_ptrs, vout, n_out, n, chunk, user)


@pytest.mark.parametrize("case", [
    dict(n_in=1, shared=True, per_voice=True),                 # both input forms
    dict(n_in=2),                                              # nIn > 0 without an input pointer
    dict(n_out=0),                                             # no output channel
    dict(n_out=4097),                                          # past ELEM_B200_MAX_OUT_CHANNELS
    dict(n_out=9, voices=True),                                # per-voice outputs past 8 channels
    dict(n_out=9, voices=True, mix=False),
    dict(n_in=1, shared=True, per_voice=True, n=0),            # argument errors come before numSamples == 0
], ids=["both-inputs", "nin-without-pointer", "nout-0", "nout-4097", "voices-past-8", "voices-only-past-8", "both-inputs-n0"])
def test_argument_errors_return_bad_argument(rt, case):
    assert _call(rt, **case) == -2
    assert rt.current_time() == 0


@pytest.mark.parametrize("case", [
    dict(), dict(n_out=4096), dict(n_out=1250), dict(n_out=8, voices=True), dict(n_out=8, voices=True, mix=False),
    dict(n_in=1, shared=True), dict(n_in=3, per_voice=True, voices=True), dict(n_in=0, shared=True),
    dict(chunk=3, t0=1000), dict(mix=False), dict(n=0),
], ids=["mix", "mix-4096", "mix-1250", "both-8", "voices-8", "shared-in", "voice-in", "nin-0", "chunk-time", "no-outputs", "n0"])
def test_valid_calls_need_a_device(rt, case):
    assert _call(rt, **case) == -1
    assert "plan-only" in rt.last_error()


def test_wrapper_rejects_both_input_forms(rt):
    with pytest.raises(ValueError):
        rt.process_offline(np.zeros((1, 10), np.float32), voice_inputs=np.zeros((V, 1, 10), np.float32))


@pytest.mark.parametrize("kw", [
    dict(num_samples=100), dict(inputs=np.zeros((2, 77), np.float32)), dict(voice_inputs=np.zeros((V, 1, 77), np.float32)),
    dict(num_samples=100, want_voices=True, want_mix=False), dict(num_samples=10, num_outputs=1250, sample_time=5),
])
def test_wrapper_reaches_the_engine(rt, kw):
    """The wrapper forms a well-formed call (the engine's -1 of a plan-only runtime, not -2 for a malformed one)."""
    with pytest.raises(RuntimeError, match=r"rc=-1 "):
        rt.process_offline(**kw)


def test_wrapper_passes_argument_errors_through(rt):
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.process_offline(num_samples=10, num_outputs=9, want_voices=True)
    with pytest.raises(RuntimeError, match=r"rc=-2 "):
        rt.process_offline(num_samples=10, num_outputs=0)


def test_render_offline_keeps_its_checks(rt):
    out = np.zeros((V, 9, BS), np.float32)
    # a plan-only engine answers -1 first, as before; the argument checks are those of a device engine
    assert rt._lib.elem_b200_render_offline(rt._h, 9, 1, out.ctypes.data_as(_f32p), 0) == -1
