"""Engine option spec_opprof: the per-opcode cycle counters of -DEB_OPPROF compiled into the NVRTC-specialised K1
(spec_host.cpp: the -DEB_OPPROF define, the name expression &eb::g_opprof and its lowered name; tools/spec_opprof.py reads them)."""
import numpy as np
import pytest

from elementary_b200 import Runtime, graphs
from elementary_b200.runtime import FLAG_MIX

OP_SVF, OP_DELAY, LOOP = 18, 21, 63        # program.h; slot 63 = the whole sample loop of a warp


def test_spec_opprof_compiles_without_a_gpu():
    """The compile step (NVRTC only) with and without the counters: both succeed, and the counters add code.  A failed lookup of
    the counters' lowered name fails the compilation."""
    sizes = {}
    for opprof in (0, 1):
        rt = Runtime(48000.0, 512, 4096, device=-1, spec_opprof=opprof)
        assert rt.apply_instructions(graphs.subsynth32()) == 0
        n, log = rt.specialize_dry_run(0)
        assert n > 50_000, log
        sizes[opprof] = n
    assert sizes[1] > sizes[0]


@pytest.mark.gpu
def test_spec_opprof_counts_every_op_of_the_specialised_kernel():
    n, blocks = 64, 3
    rt = Runtime(48000.0, 512, n, device=0, specialize=2, specialize_strict=1, spec_opprof=1, tile_width=2)
    assert rt.apply_instructions(graphs.subsynth32()) == 0
    rt.enqueue_block(0, 1, 512, FLAG_MIX)
    rt.synchronize()
    assert rt.describe()["groups"][0].get("spec_state") == 2
    rt.debug_opprof(True)
    for _ in range(blocks):
        rt.enqueue_block(0, 1, 512, FLAG_MIX)
    rt.synchronize()
    p = rt.debug_opprof(True).reshape(64, 2)
    warps, tiles = n // 2, 512 // 64                # L = 2: 64-sample tiles
    assert p[LOOP, 1] == warps * blocks
    for op in (OP_SVF, OP_DELAY):
        assert p[op, 1] == warps * blocks * tiles and p[op, 0] > 0
    assert p[:63, 0].sum() <= p[LOOP, 0]
    assert not rt.debug_opprof(False).any()          # reset
