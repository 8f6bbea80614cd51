"""Python mirror of ``elem::Runtime<float>`` over the C ABI of ``libelem_b200.so``.

Same method names, argument meaning and error behaviour as the reference class
(runtime/elem/Runtime.h:44-110): ``apply_instructions`` returns the reference's integer return codes
(Types.h:51-60), ``process`` takes planar float32 inputs and fills planar outputs, shared resources are
insert-only, ``gc`` returns the pruned node ids.  New here is the voice axis: one :class:`Runtime` holds
``num_voices`` independent graph instances that render in one fused CUDA kernel per block.

This module only *binds*: all work happens in the CUDA library (``include/elem_b200.h``).  There is no CPU
fallback — if the shared library is missing it raises ImportError-like RuntimeError, and without a CUDA device
``Runtime(...)`` raises, except for ``device=-1`` which builds a *plan-only* runtime (host logic and graph
compilation only; every render call fails) used by the CPU test-suite.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Iterable, List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ELEM_B200_LIB") or os.path.join(_HERE, "libelem_b200.so")   # env override: A/B builds only

_f32p = C.POINTER(C.c_float)
_f32pp = C.POINTER(_f32p)

RETURN_CODES = {
    0: "Ok", 1: "UnknownNodeType", 2: "NodeNotFound", 3: "NodeAlreadyExists", 4: "NodeTypeAlreadyExists",
    5: "InvalidPropertyType", 6: "InvalidPropertyValue", 7: "InvariantViolation", 8: "InvalidInstructionFormat",
    -1: "CudaError", -2: "BadArgument",
}

FLAG_VOICE_IN, FLAG_VOICE_OUT, FLAG_MIX, FLAG_ALLREDUCE = 1, 2, 4, 8
READOUT_DEVICE = 1      # elem_b200_poll_readouts: the arrays are device memory

_lib = None


EVENT_CB = C.CFUNCTYPE(None, C.c_char_p, C.c_char_p, C.c_void_p)
BLOCK_EVENT_CB = C.CFUNCTYPE(None, C.c_size_t, C.c_char_p, C.c_char_p, C.c_void_p)


def load_library() -> C.CDLL:
    """Load ``libelem_b200.so`` (built in-tree by ``__graft_entry__.build()``).  Fails loudly when missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    lib.elem_b200_create.restype = C.c_void_p
    lib.elem_b200_create.argtypes = [C.c_double, C.c_int, C.c_int, C.c_int]
    lib.elem_b200_destroy.argtypes = [C.c_void_p]
    lib.elem_b200_apply_instructions.restype = C.c_int
    lib.elem_b200_apply_instructions.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_size_t]
    lib.elem_b200_apply_binary.restype = C.c_int
    lib.elem_b200_apply_binary.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_size_t]
    lib.elem_b200_set_const_table.restype = C.c_int
    lib.elem_b200_set_const_table.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int, _f32p, C.c_int, C.c_int]
    lib.elem_b200_set_property_per_voice.restype = C.c_int
    lib.elem_b200_set_property_per_voice.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.POINTER(C.c_double), C.c_int, C.c_int]
    lib.elem_b200_set_path_per_voice.restype = C.c_int
    lib.elem_b200_set_path_per_voice.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int]
    lib.elem_b200_set_seq_per_voice.restype = C.c_int
    lib.elem_b200_set_seq_per_voice.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int]
    lib.elem_b200_reset_voices.restype = C.c_int
    lib.elem_b200_reset_voices.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_size_t]
    lib.elem_b200_reset_bytes_written.restype = C.c_uint64
    lib.elem_b200_reset_bytes_written.argtypes = [C.c_void_p]
    lib.elem_b200_process.restype = C.c_int
    lib.elem_b200_process.argtypes = [C.c_void_p, _f32pp, C.c_size_t, _f32pp, C.c_size_t, C.c_size_t, C.c_void_p]
    lib.elem_b200_set_current_time.argtypes = [C.c_void_p, C.c_int64]
    lib.elem_b200_current_time.restype = C.c_int64
    lib.elem_b200_current_time.argtypes = [C.c_void_p]
    lib.elem_b200_process_voices.restype = C.c_int
    lib.elem_b200_process_voices.argtypes = [C.c_void_p, _f32p, C.c_size_t, _f32p, _f32p, C.c_size_t, C.c_size_t]
    lib.elem_b200_render_offline.restype = C.c_int
    lib.elem_b200_render_offline.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, _f32p, C.c_size_t]
    lib.elem_b200_process_offline.restype = C.c_int
    lib.elem_b200_process_offline.argtypes = [C.c_void_p, _f32pp, C.c_size_t, _f32p, _f32pp, _f32p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]
    lib.elem_b200_enqueue_block.restype = C.c_int
    lib.elem_b200_process_offline_events.restype = C.c_int
    lib.elem_b200_process_offline_events.argtypes = [C.c_void_p, _f32pp, C.c_size_t, _f32p, _f32pp, _f32p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                     C.c_void_p, C.c_int, C.c_int, BLOCK_EVENT_CB, C.c_void_p]
    lib.elem_b200_enqueue_block.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    lib.elem_b200_process_offline_readouts.restype = C.c_int
    lib.elem_b200_process_offline_readouts.argtypes = [C.c_void_p, _f32pp, C.c_size_t, _f32p, _f32pp, _f32p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                       C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                       C.c_void_p]
    lib.elem_b200_poll_readouts.restype = C.c_int
    lib.elem_b200_poll_readouts.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.elem_b200_node_type.restype = C.c_int
    lib.elem_b200_node_type.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_char_p, C.c_size_t]
    lib.elem_b200_peer_export.restype = C.c_int
    lib.elem_b200_peer_export.argtypes = [C.c_void_p, C.c_char_p]
    lib.elem_b200_peer_attach.restype = C.c_int
    lib.elem_b200_peer_attach.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
    lib.elem_b200_peer_status.restype = C.c_int
    lib.elem_b200_peer_status.argtypes = [C.c_void_p]
    lib.elem_b200_peer_barrier.restype = C.c_int
    lib.elem_b200_peer_barrier.argtypes = [C.c_void_p]
    lib.elem_b200_last_kernel_times.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    lib.elem_b200_synchronize.restype = C.c_int
    lib.elem_b200_synchronize.argtypes = [C.c_void_p]
    for name in ("elem_b200_mix_device", "elem_b200_voice_out_device"):
        getattr(lib, name).restype = C.c_void_p
        getattr(lib, name).argtypes = [C.c_void_p]
    for name in ("elem_b200_voice_in_device", "elem_b200_shared_in_device"):
        getattr(lib, name).restype = C.c_void_p
        getattr(lib, name).argtypes = [C.c_void_p, C.c_size_t]
    lib.elem_b200_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    lib.elem_b200_add_shared_resource.restype = C.c_int
    lib.elem_b200_add_shared_resource.argtypes = [C.c_void_p, C.c_char_p, _f32pp, C.c_size_t, C.c_size_t]
    lib.elem_b200_prune_shared_resources.argtypes = [C.c_void_p]
    lib.elem_b200_list_shared_resources.restype = C.c_int
    lib.elem_b200_list_shared_resources.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    lib.elem_b200_gc.restype = C.c_int
    lib.elem_b200_gc.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_size_t]
    lib.elem_b200_reset.argtypes = [C.c_void_p]
    lib.elem_b200_process_queued_events.argtypes = [C.c_void_p, EVENT_CB, C.c_void_p]
    lib.elem_b200_process_queued_events_range.restype = C.c_int
    lib.elem_b200_process_queued_events_range.argtypes = [C.c_void_p, C.c_int, C.c_int, EVENT_CB, C.c_void_p]
    lib.elem_b200_set_option.restype = C.c_int
    lib.elem_b200_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
    lib.elem_b200_register_node_type.restype = C.c_int
    lib.elem_b200_register_node_type.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_char_p]
    lib.elem_b200_has_node_type.restype = C.c_int
    lib.elem_b200_has_node_type.argtypes = [C.c_void_p, C.c_char_p]
    lib.elem_b200_snapshot.restype = C.c_int
    lib.elem_b200_snapshot.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    lib.elem_b200_describe.restype = C.c_int
    lib.elem_b200_describe.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    lib.elem_b200_program_words.restype = C.c_int
    lib.elem_b200_program_words.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_uint32), C.c_size_t]
    lib.elem_b200_specialize_dry_run.restype = C.c_long
    lib.elem_b200_specialize_dry_run.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    lib.elem_b200_kernel_launches.restype = C.c_uint64
    lib.elem_b200_kernel_launches.argtypes = [C.c_void_p]
    lib.elem_b200_take_kernel_time_ms.restype = C.c_double
    lib.elem_b200_take_kernel_time_ms.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.elem_b200_last_convolve_time_ms.restype = C.c_double
    lib.elem_b200_last_convolve_time_ms.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.elem_b200_last_error.restype = C.c_char_p
    lib.elem_b200_last_error.argtypes = [C.c_void_p]
    lib.elem_b200_describe_return_code.restype = C.c_char_p
    lib.elem_b200_describe_return_code.argtypes = [C.c_int]
    lib.elem_b200_device_count.restype = C.c_int
    _lib = lib
    return lib


def device_count() -> int:
    return load_library().elem_b200_device_count()


def describe_return_code(code: int) -> str:
    return load_library().elem_b200_describe_return_code(code).decode()


class DeviceArray:
    """Zero-copy view of an engine-owned device buffer (``__cuda_array_interface__``), e.g. for
    ``torch.as_tensor(rt.mix_device(), device='cuda')`` in the multi-GPU mix-bus reduce."""

    def __init__(self, ptr: int, shape):
        self.ptr, self.shape = ptr, tuple(shape)

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": "<f4", "data": (self.ptr, False), "version": 3, "strides": None}


class Runtime:
    """``elem::Runtime<float>`` with a voice axis.  See module docstring."""

    def __init__(self, sample_rate: float = 48000.0, block_size: int = 512, num_voices: int = 1, device: int = 0,
                 **options: float):
        self._lib = load_library()
        self.sample_rate, self.block_size, self.num_voices, self.device = float(sample_rate), int(block_size), int(num_voices), int(device)
        h = self._lib.elem_b200_create(self.sample_rate, self.block_size, self.num_voices, self.device)
        if not h:
            raise RuntimeError("elem_b200_create failed: " + self._lib.elem_b200_last_error(None).decode())
        self._h = C.c_void_p(h)
        if os.environ.get("ELEM_B200_SPECIALIZE") == "1":      # run anything (the GPU parity suite) on the experimental per-program kernels
            options.setdefault("specialize", 2)                 # 2 = wait for the compiler at COMMIT: no interpreter blocks in between
            options.setdefault("specialize_strict", 1)          # a specialisation that fails to compile or load is an error, never a silent fallback
        for k, v in options.items():
            self.set_option(k, v)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.elem_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- Runtime::applyInstructions (Runtime.h:48,170-218) ------------------------------------------------------
    def apply_instructions(self, batch, voices: Optional[Sequence[int]] = None) -> int:
        """Apply an instruction batch (list or JSON text) to voices ``[voices[0], voices[1])`` (default: all)."""
        s = batch if isinstance(batch, (str, bytes)) else json.dumps(batch)
        b = s.encode() if isinstance(s, str) else s
        vb, ve = (0, -1) if voices is None else (int(voices[0]), int(voices[1]))
        return self._lib.elem_b200_apply_instructions(self._h, vb, ve, b, len(b))

    def apply_binary(self, data: bytes, voices: Optional[Sequence[int]] = None) -> int:
        """Apply an instruction batch in the binary encoding (include/elem_b200.h; ``el.encode_binary`` writes it)."""
        vb, ve = (0, -1) if voices is None else (int(voices[0]), int(voices[1]))
        return self._lib.elem_b200_apply_binary(self._h, vb, ve, data, len(data))

    def set_const_table(self, node_ids, values, voice_begin: int = 0) -> int:
        """values[p][i] -> ``value`` of const node ``node_ids[p]`` for voice ``voice_begin + i`` (float32 table, one copy per row)."""
        ids = np.ascontiguousarray(np.asarray(node_ids, dtype=np.int32))
        v = np.ascontiguousarray(np.asarray(values, dtype=np.float32))
        assert v.ndim == 2 and v.shape[0] == ids.size
        return self._lib.elem_b200_set_const_table(self._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.size,
                                                   v.ctypes.data_as(_f32p), int(voice_begin), v.shape[1])

    def set_property_per_voice(self, node_id: int, key: str, values, voice_begin: int = 0) -> int:
        v = np.ascontiguousarray(np.asarray(values, dtype=np.float64))
        return self._lib.elem_b200_set_property_per_voice(self._h, int(node_id), key.encode(),
                                                          v.ctypes.data_as(C.POINTER(C.c_double)), int(voice_begin), v.size)

    def set_path_per_voice(self, node_id: int, names, index, voice_begin: int = 0) -> int:
        """Voice ``voice_begin + i`` of convolve or sample node ``node_id`` gets the impulse response or sample buffer
        ``names[index[i]]`` (shared resources), without cutting its voice group; the addressed voices restart from silence at the next
        block (a sample node keeps its voices' trigger edge detector and current reader)."""
        return self._set_per_voice(self._lib.elem_b200_set_path_per_voice, node_id,
                                   [n.encode() if isinstance(n, str) else bytes(n) for n in names], index, voice_begin)

    def set_seq_per_voice(self, node_id: int, seqs, index, voice_begin: int = 0) -> int:
        """Voice ``voice_begin + i`` of seq, seq2, sparseq or sparseq2 node ``node_id`` gets the sequence ``seqs[index[i]]`` (a Python
        value such as ``[1, 2, 3]`` or ``[{"tickTime": 0, "value": 1}]``, JSON-encoded here; bytes pass through as JSON text),
        without cutting its voice group: the same as single-voice ``[3, node_id, "seq", seqs[index[i]]]`` batches.  Each distinct
        sequence is parsed and uploaded once."""
        return self._set_per_voice(self._lib.elem_b200_set_seq_per_voice, node_id,
                                   [s if isinstance(s, bytes) else json.dumps(s).encode() for s in seqs], index, voice_begin)

    def _set_per_voice(self, fn, node_id, table, index, voice_begin):
        """fn(node, table of C strings, their count, int32 index per voice, first voice, voice count): a table plus an index."""
        tab = (C.c_char_p * max(1, len(table)))(*table)
        idx = np.ascontiguousarray(np.asarray(index, dtype=np.int32).reshape(-1))
        return fn(self._h, int(node_id), tab, len(table), idx.ctypes.data_as(C.POINTER(C.c_int32)), int(voice_begin), idx.size)

    def reset_voices(self, voices) -> int:
        """The given voices (runtime-global indices, any order, repeats allowed) restart as fresh instances from the next block on, as
        if a new Runtime had been given this runtime's instruction history; props are replayed as last set for each voice.  One kernel
        launch, stream-ordered, no voice group cut.  Returns 0, or -2 (nothing changed) when an index is outside [0, num_voices)."""
        v = np.ascontiguousarray(np.asarray(voices, dtype=np.int64).reshape(-1))
        if v.size and (v.min() < -2**31 or v.max() >= 2**31):
            return -2
        v = v.astype(np.int32)
        return self._lib.elem_b200_reset_voices(self._h, v.ctypes.data_as(C.POINTER(C.c_int32)), v.size)

    @property
    def reset_bytes_written(self) -> int:
        """Bytes the voice resets have written so far, counted from their plans."""
        return int(self._lib.elem_b200_reset_bytes_written(self._h))

    # -- Runtime::process (Runtime.h:51-57,275-290): out = mix bus over all voices -------------------------------
    def process(self, inputs: Optional[np.ndarray], num_outputs: int, num_samples: Optional[int] = None,
                sample_time: Optional[int] = None) -> np.ndarray:
        """``sample_time``: the int64 the reference's hosts pass as ``userData`` (wasm/Main.cpp:206-215); None lets the
        engine keep the clock itself."""
        n = int(num_samples if num_samples is not None else self.block_size)
        if inputs is None or len(inputs) == 0:
            n_in, in_ptrs, keep = 0, None, None
        else:
            keep = np.ascontiguousarray(np.asarray(inputs, dtype=np.float32))
            assert keep.ndim == 2 and keep.shape[1] >= n
            n_in = keep.shape[0]
            in_ptrs = (_f32p * n_in)(*[keep[i].ctypes.data_as(_f32p) for i in range(n_in)])
        out = np.zeros((num_outputs, n), dtype=np.float32)
        out_ptrs = (_f32p * max(1, num_outputs))(*[out[i].ctypes.data_as(_f32p) for i in range(num_outputs)])
        user = None if sample_time is None else C.byref(C.c_int64(int(sample_time)))
        rc = self._lib.elem_b200_process(self._h, in_ptrs, n_in, out_ptrs, num_outputs, n, user)
        self._check(rc, "process")
        return out

    def process_voices(self, inputs: Optional[np.ndarray], num_outputs: int, num_samples: Optional[int] = None,
                       want_voices: bool = True, want_mix: bool = True):
        """Per-voice I/O: ``inputs`` is [voice, n_in, n] or None.  Returns (voices [voice, n_out, n] | None, mix [n_out, n] | None)."""
        n = int(num_samples if num_samples is not None else self.block_size)
        if inputs is None:
            n_in, in_ptr, keep = 0, None, None
        else:
            keep = np.ascontiguousarray(np.asarray(inputs, dtype=np.float32))
            assert keep.ndim == 3 and keep.shape[0] == self.num_voices and keep.shape[2] == n
            n_in, in_ptr = keep.shape[1], keep.ctypes.data_as(_f32p)
        ov = np.zeros((self.num_voices, num_outputs, n), dtype=np.float32) if want_voices else None
        mix = np.zeros((num_outputs, n), dtype=np.float32) if want_mix else None
        rc = self._lib.elem_b200_process_voices(self._h, in_ptr, n_in,
                                                ov.ctypes.data_as(_f32p) if ov is not None else None,
                                                mix.ctypes.data_as(_f32p) if mix is not None else None, num_outputs, n)
        self._check(rc, "process_voices")
        return ov, mix

    def render_voices(self, n_blocks: int, num_outputs: int = 1, inputs: Optional[np.ndarray] = None):
        """Run ``n_blocks`` blocks; returns (voices [voice, n_out, n_blocks*bs], mix [n_out, n_blocks*bs])."""
        bs = self.block_size
        vs, ms = [], []
        for b in range(n_blocks):
            inp = None if inputs is None else np.asarray(inputs)[:, :, b * bs:(b + 1) * bs]
            v, m = self.process_voices(inp, num_outputs, bs)
            vs.append(v)
            ms.append(m)
        return np.concatenate(vs, axis=2), np.concatenate(ms, axis=1)

    def render_offline(self, n_blocks: int, num_outputs: int = 1, chunk_blocks: int = 0, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Offline render: ``n_blocks`` blocks of every voice with no host round trip per block; returns [voice, n_out, n_blocks*bs]."""
        if out is None:
            out = np.empty((self.num_voices, num_outputs, n_blocks * self.block_size), dtype=np.float32)
        assert out.flags["C_CONTIGUOUS"] and out.dtype == np.float32 and out.shape == (self.num_voices, num_outputs, n_blocks * self.block_size)
        self._check(self._lib.elem_b200_render_offline(self._h, num_outputs, n_blocks, out.ctypes.data_as(_f32p), chunk_blocks), "render_offline")
        return out

    def process_offline(self, inputs: Optional[np.ndarray] = None, num_outputs: int = 1, num_samples: Optional[int] = None,
                        voice_inputs: Optional[np.ndarray] = None, want_mix: bool = True, want_voices: bool = False,
                        chunk_blocks: int = 0, sample_time: Optional[int] = None, on_event=None,
                        event_voices: Optional[Sequence[int]] = None, readouts: Optional[Sequence[int]] = None,
                        readout_voices: Optional[Sequence[int]] = None):
        """OfflineRenderer.process (js/packages/offline-renderer/index.ts:87-133): ceil(n / block_size) full blocks in one call, with
        ``inputs`` [n_in, n] broadcast to every voice or ``voice_inputs`` [voice, n_in, n] (zero past n), no host round trip per block.
        ``num_samples`` defaults to the inputs' length (one block without inputs).  ``sample_time``: as for :meth:`process`, for the
        first block.  Returns (mix [n_out, n] | None, voices [voice, n_out, n] | None), truncated to n.

        ``on_event(block, type, event_dict)``: every block's events, as :meth:`process_queued_events` (``voices`` = ``event_voices``)
        would report them right after the block (elem_b200_process_offline_events); called in block order before the call returns,
        and it must not call into this runtime.  An exception it raises is re-raised once the call has returned.

        ``readouts``: meter / snapshot node ids whose readouts are read after every block as :meth:`poll_readouts` would read them,
        polled in the order given, for the voices ``readout_voices`` = (begin, end) (default: all); no other event node is polled
        (elem_b200_process_offline_readouts).  The call then returns a third element, ``{node_id: {...}}`` with the arrays of
        :meth:`poll_readouts` shaped [blocks, voices].  Not together with ``on_event``."""
        if inputs is not None and voice_inputs is not None:
            raise ValueError("process_offline: give inputs or voice_inputs, not both")
        if readouts is not None and on_event is not None:
            raise ValueError("process_offline: give readouts or on_event, not both")
        src = inputs if inputs is not None else voice_inputs
        keep = None if src is None else np.ascontiguousarray(np.asarray(src, dtype=np.float32))
        n = int(num_samples if num_samples is not None else (keep.shape[-1] if keep is not None else self.block_size))
        in_ptrs, vin_ptr, n_in = None, None, 0
        if inputs is not None:
            assert keep.ndim == 2 and keep.shape[1] == n
            n_in = keep.shape[0]
            if n_in:
                in_ptrs = (_f32p * n_in)(*[keep[i].ctypes.data_as(_f32p) for i in range(n_in)])
        elif voice_inputs is not None:
            assert keep.ndim == 3 and keep.shape[0] == self.num_voices and keep.shape[2] == n
            n_in = keep.shape[1]
            vin_ptr = keep.ctypes.data_as(_f32p) if n_in else None
        mix = np.zeros((num_outputs, n), dtype=np.float32) if want_mix else None
        ov = np.zeros((self.num_voices, num_outputs, n), dtype=np.float32) if want_voices else None
        mix_ptrs = (_f32p * max(1, num_outputs))(*[mix[i].ctypes.data_as(_f32p) for i in range(num_outputs)]) if want_mix else None
        user = None if sample_time is None else C.byref(C.c_int64(int(sample_time)))
        ov_ptr = ov.ctypes.data_as(_f32p) if ov is not None else None
        if readouts is not None:
            ids = np.ascontiguousarray(np.asarray(readouts, dtype=np.int32).reshape(-1))
            vb, ve = (0, self.num_voices) if readout_voices is None else (int(readout_voices[0]), int(readout_voices[1]))
            shape = (ids.size, -(-n // self.block_size), max(0, ve - vb))
            a, b, fresh = np.zeros(shape, np.float32), np.zeros(shape, np.float32), np.zeros(shape, np.uint8)
            rc = self._lib.elem_b200_process_offline_readouts(self._h, in_ptrs, n_in, vin_ptr, mix_ptrs, ov_ptr, num_outputs, n,
                                                              int(chunk_blocks), user, ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.size,
                                                              vb, ve - vb, a.ctypes.data, b.ctypes.data, fresh.ctypes.data)
            self._check(rc, "process_offline")
            return mix, ov, {int(i): self._readout_dict(int(i), vb, a[j], b[j], fresh[j]) for j, i in enumerate(ids)}
        if on_event is None:
            rc = self._lib.elem_b200_process_offline(self._h, in_ptrs, n_in, vin_ptr, mix_ptrs, ov_ptr, num_outputs, n, int(chunk_blocks), user)
            self._check(rc, "process_offline")
            return mix, ov
        import json as _json
        raised: List[BaseException] = []

        def _cb(block, type_, js, _user):
            if raised:
                return
            try:
                on_event(int(block), type_.decode(), _json.loads(js.decode()))
            except BaseException as exc:    # ctypes cannot unwind through C: keep the first one for after the call
                raised.append(exc)

        cb = BLOCK_EVENT_CB(_cb)
        vb, ve = (0, -1) if event_voices is None else (int(event_voices[0]), int(event_voices[1]))
        rc = self._lib.elem_b200_process_offline_events(self._h, in_ptrs, n_in, vin_ptr, mix_ptrs, ov_ptr, num_outputs, n,
                                                        int(chunk_blocks), user, vb, ve, cb, None)
        if raised:
            raise raised[0]
        self._check(rc, "process_offline")
        return mix, ov

    # -- device-resident stepping -----------------------------------------------------------------------------
    def enqueue_block(self, n_in: int = 0, n_out: int = 1, num_samples: Optional[int] = None, flags: int = FLAG_MIX) -> None:
        n = int(num_samples if num_samples is not None else self.block_size)
        self._check(self._lib.elem_b200_enqueue_block(self._h, n_in, n_out, n, flags), "enqueue_block")

    # -- cross-GPU mix bus over peer memory (include/elem_b200.h: elem_b200_peer_*) ------------------------------------
    def peer_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._check(self._lib.elem_b200_peer_export(self._h, buf), "peer_export")
        return buf.raw

    def peer_attach(self, rank: int, handles: Sequence[bytes]) -> None:
        blob = b"".join(handles)
        assert len(blob) == 64 * len(handles)
        self._check(self._lib.elem_b200_peer_attach(self._h, int(rank), len(handles), blob), "peer_attach")

    def peer_status(self) -> int:
        return int(self._lib.elem_b200_peer_status(self._h))

    def peer_barrier(self) -> None:
        """Enqueue a cross-GPU barrier on the render stream (no-op without attached peers)."""
        self._check(self._lib.elem_b200_peer_barrier(self._h), "peer_barrier")

    def synchronize(self) -> None:
        self._check(self._lib.elem_b200_synchronize(self._h), "synchronize")

    def set_stream(self, cuda_stream_handle: int) -> None:
        self._lib.elem_b200_set_stream(self._h, C.c_void_p(cuda_stream_handle))

    def mix_device(self, n_out: int = 1) -> DeviceArray:
        return DeviceArray(self._lib.elem_b200_mix_device(self._h), (n_out, self.block_size))

    def voice_out_device(self, n_out: int = 1) -> DeviceArray:
        return DeviceArray(self._lib.elem_b200_voice_out_device(self._h), (self.num_voices, n_out, self.block_size))

    def voice_in_device(self, n_in: int) -> DeviceArray:
        return DeviceArray(self._lib.elem_b200_voice_in_device(self._h, n_in), (self.num_voices, n_in, self.block_size))

    def shared_in_device(self, n_in: int) -> DeviceArray:
        return DeviceArray(self._lib.elem_b200_shared_in_device(self._h, n_in), (n_in, self.block_size))

    # -- shared resources (Runtime.h:83-94) -----------------------------------------------------------------------
    def add_shared_resource(self, name: str, data) -> bool:
        a = np.ascontiguousarray(np.asarray(data, dtype=np.float32))
        if a.ndim == 1:
            a = a[None, :]
        ptrs = (_f32p * a.shape[0])(*[a[i].ctypes.data_as(_f32p) for i in range(a.shape[0])])
        return bool(self._lib.elem_b200_add_shared_resource(self._h, name.encode(), ptrs, a.shape[0], a.shape[1]))

    def prune_shared_resources(self) -> None:
        self._lib.elem_b200_prune_shared_resources(self._h)

    def get_shared_resource_map_keys(self) -> List[str]:
        buf = C.create_string_buffer(1 << 16)
        self._lib.elem_b200_list_shared_resources(self._h, buf, len(buf))
        return [s for s in buf.value.decode().split("\n") if s]

    # -- gc / reset / events ------------------------------------------------------------------------------------
    def gc(self, voice: int = 0) -> List[int]:
        buf = (C.c_int32 * 65536)()
        n = self._lib.elem_b200_gc(self._h, voice, buf, 65536)
        return [buf[i] for i in range(min(n, 65536))]

    def reset(self) -> None:
        """Runtime::reset(): both readers of every `sample` node of every voice get noteOff, as in the reference."""
        self._lib.elem_b200_reset(self._h)

    # -- ElementaryAudioProcessor::setCurrentTime (wasm/Main.cpp:232-241) ---------------------------------------------
    def set_current_time(self, sample_time: int) -> None:
        self._lib.elem_b200_set_current_time(self._h, int(sample_time))

    def current_time(self) -> int:
        return int(self._lib.elem_b200_current_time(self._h))

    def process_queued_events(self, callback=None, voices: Optional[Sequence[int]] = None) -> List[dict]:
        """Runtime::processQueuedEvents (Runtime.h:64,438-446).  ``callback(type, event_dict)`` is called per event like
        the reference's handler; the events are also returned as ``[{"type": ..., "event": {...}}, ...]`` — the batch
        shape of wasm/Main.cpp:220-231.  Every event dict carries the reference's keys plus ``"voice"``."""
        import json as _json
        events: List[dict] = []

        def _cb(type_, js, _user):
            evt = _json.loads(js.decode())
            events.append({"type": type_.decode(), "event": evt})
            if callback is not None:
                callback(type_.decode(), evt)

        cb = EVENT_CB(_cb)
        vb, ve = (0, -1) if voices is None else (int(voices[0]), int(voices[1]))
        self._check(self._lib.elem_b200_process_queued_events_range(self._h, vb, ve, cb, None), "process_queued_events")
        return events

    def poll_readouts(self, node_id: int, voices: Optional[Sequence[int]] = None) -> dict:
        """The poll of one meter or snapshot node over ``voices`` = (begin, end) (default: all) into arrays, index i = voice begin + i
        (elem_b200_poll_readouts): ``{"min", "max", "fresh"}`` for a meter, ``{"data", "fresh"}`` for a snapshot.  ``fresh[i]`` is 1 where
        :meth:`process_queued_events` would have reported an event for that voice, with the same side effects; elsewhere the values are 0."""
        vb, ve = (0, self.num_voices) if voices is None else (int(voices[0]), int(voices[1]))
        n = max(0, ve - vb)
        a, b, fresh = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.uint8)
        rc = self._lib.elem_b200_poll_readouts(self._h, int(node_id), vb, ve - vb, a.ctypes.data, b.ctypes.data, fresh.ctypes.data, 0)
        self._check(rc, "poll_readouts")
        return self._readout_dict(int(node_id), vb, a, b, fresh)

    def poll_readouts_device(self, node_id: int, a_ptr: int, b_ptr: Optional[int], fresh_ptr: int,
                             voices: Optional[Sequence[int]] = None) -> None:
        """:meth:`poll_readouts` into device memory (float32 ``a`` and ``b``, uint8 ``fresh``, e.g. ``tensor.data_ptr()``; ``b_ptr`` may
        be None): enqueued on the runtime's stream, no synchronisation.  ``a`` is the min or the value, ``b`` the max."""
        vb, ve = (0, self.num_voices) if voices is None else (int(voices[0]), int(voices[1]))
        rc = self._lib.elem_b200_poll_readouts(self._h, int(node_id), vb, ve - vb, a_ptr or None, b_ptr or None, fresh_ptr or None, READOUT_DEVICE)
        self._check(rc, "poll_readouts_device")

    def node_type(self, node_id: int, voice: int = 0) -> Optional[str]:
        """The type name of ``node_id`` in the voice group containing ``voice``, or None."""
        buf = C.create_string_buffer(64)
        n = self._lib.elem_b200_node_type(self._h, int(voice), int(node_id), buf, len(buf))
        return buf.value.decode() if n else None

    def _readout_dict(self, node_id, voice, a, b, fresh) -> dict:
        if self.node_type(node_id, voice) == "snapshot":
            return {"data": a, "fresh": fresh}
        return {"min": a, "max": b, "fresh": fresh}

    # -- introspection ------------------------------------------------------------------------------------------
    def set_option(self, key: str, value: float) -> None:
        self._check(self._lib.elem_b200_set_option(self._h, key.encode(), float(value)), f"set_option({key})")

    def describe(self) -> dict:
        n = self._lib.elem_b200_describe(self._h, None, 0)
        buf = C.create_string_buffer(n + 16)
        self._lib.elem_b200_describe(self._h, buf, len(buf))
        return json.loads(buf.value.decode())

    def register_node_type(self, type_name: str, num_inputs: int, num_state: int, cuda_body: str) -> int:
        """Runtime::registerNodeType (Runtime.h:105-106) for device code: ``cuda_body`` is the body of
        ``float node(float* s, const float* in, const float sr)``; returns the reference's codes (4 = name taken)."""
        return self._lib.elem_b200_register_node_type(self._h, type_name.encode(), int(num_inputs), int(num_state), cuda_body.encode())

    def has_node_type(self, type_name: str) -> bool:
        return bool(self._lib.elem_b200_has_node_type(self._h, type_name.encode()))

    def snapshot(self, voice: int = 0) -> dict:
        """Runtime::snapshot() (Runtime.h:110,490-499): {"0x<hex node id>": props} of the voice group containing ``voice``."""
        n = self._lib.elem_b200_snapshot(self._h, int(voice), None, 0)
        buf = C.create_string_buffer(n + 16)
        self._lib.elem_b200_snapshot(self._h, int(voice), buf, len(buf))
        return json.loads(buf.value.decode())

    def debug_opprof(self, reset: bool = True) -> np.ndarray:
        """A/B builds with -DEB_OPPROF only: [64, 2] uint64 (cycles, dispatches) per opcode of the K1 interpreter; zeros otherwise."""
        buf = np.zeros(128, dtype=np.uint64)
        self._lib.elem_b200_debug_opprof.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        rc = self._lib.elem_b200_debug_opprof(self._h, buf.ctypes.data_as(C.c_void_p), 1 if reset else 0)
        self._check(rc, "debug_opprof")
        return buf.reshape(64, 2)

    def program_words(self, voice: int = 0) -> np.ndarray:
        """The encoded render program of the voice group containing ``voice`` (uint32 words, csrc/program.h)."""
        n = self._lib.elem_b200_program_words(self._h, int(voice), None, 0)
        buf = np.zeros(max(1, n), dtype=np.uint32)
        self._lib.elem_b200_program_words(self._h, int(voice), buf.ctypes.data_as(C.POINTER(C.c_uint32)), n)
        return buf[:n]

    def specialize_dry_run(self, voice: int = 0):
        """EXPERIMENTAL: NVRTC-compile (only) the specialised K1 of the voice group containing ``voice``.  Returns
        (cubin_bytes | -1, compiler_log)."""
        buf = C.create_string_buffer(1 << 16)
        n = self._lib.elem_b200_specialize_dry_run(self._h, int(voice), buf, len(buf))
        return int(n), buf.value.decode(errors="replace")

    @property
    def kernel_launches(self) -> int:
        return int(self._lib.elem_b200_kernel_launches(self._h))

    def take_kernel_time_ms(self):
        """(summed device ms of the K1 launches since the last call, number of launches); needs time_kernels=1."""
        n = C.c_uint64(0)
        ms = self._lib.elem_b200_take_kernel_time_ms(self._h, C.byref(n))
        return float(ms), int(n.value)

    def last_kernel_times(self) -> dict:
        """{"K1": (ms, n), "K2": ..., "K3": ..., "K4": ...} gathered by the latest take_kernel_time_ms()."""
        ms = (C.c_double * 4)()
        n = (C.c_uint64 * 4)()
        self._lib.elem_b200_last_kernel_times(self._h, ms, n)
        return {k: (float(ms[i]), int(n[i])) for i, k in enumerate(("K1", "K2", "K3", "K4"))}

    def last_convolve_time_ms(self):
        """(summed device ms of the K3 launches, count) gathered by the latest take_kernel_time_ms()."""
        n = C.c_uint64(0)
        ms = self._lib.elem_b200_last_convolve_time_ms(self._h, C.byref(n))
        return float(ms), int(n.value)

    def last_error(self) -> str:
        return self._lib.elem_b200_last_error(self._h).decode()

    def _check(self, rc: int, what: str) -> None:
        if rc != 0:
            raise RuntimeError(f"{what} failed: rc={rc} ({RETURN_CODES.get(rc, '?')}): {self.last_error()}")
