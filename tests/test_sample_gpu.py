"""The `sample` node on the GPU: every voice bit for bit (np.array_equal) against SampleModel (tests/sample_common.py, pinned to the
compiled reference by tests/test_sample_cpu.py), in the K1 tile geometries, interpreted and specialised, through process() calls of
odd lengths.  The scenarios (tests/sample_common.py): trigger / gate / loop, retriggers inside the 10 ms fade,
rates that are fractional, > 1, 0, negative, moving or a constant, start and stop offsets, buffers of 1, 2, 7, 13, 1000 and 3001
samples, a path changed while playing or set late, one child or none, a live edit, a voice-group cut, reset_voices, reset(),
prune_shared_resources, reads outside the buffer; plus 4096 voices choosing among 64 buffers in one voice group, and one-voice
graphs in the batched launch.  The mix bus is checked against the float64 sum of the model's voices.

By default each scenario runs the interpreter in every geometry and the specialised kernels in rotated geometries (as
tests/test_kernel_matrix_gpu.py does); the trigger and loop scenarios, and ELEM_B200_MATRIX_FULL=1, run the whole cross product."""
import os

import numpy as np
import pytest

from elementary_b200 import Runtime, el
from k1_families import BUILDS, DENSE_WIDTHS, GEOMETRIES, assert_build, assert_exact, check_mix
from oracle import oracle as orc
import sample_common
from sample_common import BS, SR

FULL = os.environ.get("ELEM_B200_MATRIX_FULL") == "1"
SCENARIOS = {sc.name: sc for sc in sample_common.scenarios() + [sample_common.many_voices()]}
ALWAYS_FULL = ("trigger", "loop")
_REF = {}


def _reference(sc):
    if sc.name not in _REF:
        _REF[sc.name] = sc.model()
    return _REF[sc.name]


def _params():
    out = []
    for i, name in enumerate(SCENARIOS):
        full = FULL or name in ALWAYS_FULL
        spec_geoms = GEOMETRIES if full else [GEOMETRIES[(i + 4 * j) % len(GEOMETRIES)] for j in range(2)]
        dense = DENSE_WIDTHS if full else [DENSE_WIDTHS[i % len(DENSE_WIDTHS)]]
        for L, niter in GEOMETRIES:
            out.append(pytest.param(name, L, niter, "interp", id=f"{name}-L{L}n{niter}-interp"))
            if (L, niter) in spec_geoms:
                out.append(pytest.param(name, L, niter, "spec", id=f"{name}-L{L}n{niter}-spec"))
        for L in dense:
            out.append(pytest.param(name, L, 0, "dense", id=f"{name}-L{L}n0-dense"))
    return out


def _runtime(sc, L, niter, build, **extra):
    opts = dict(BUILDS[build], tile_width=L, **extra)
    if niter:
        opts["niter"] = niter
    rt = Runtime(SR, BS, sc.n_voices, device=0, **opts)
    sc.setup_gpu(rt)
    rt.build = build
    assert rt.describe()["groups"][0]["tile_width"] == L
    return rt


@pytest.mark.gpu
@pytest.mark.parametrize("name,tile_width,niter,build", _params())
def test_sample_scenario(name, tile_width, niter, build):
    sc = SCENARIOS[name]
    ref, inputs = _reference(sc)
    rt = _runtime(sc, tile_width, niter, build)
    got, mix = sc.run_gpu(rt, inputs)
    assert_build(rt)
    assert_exact(got, ref, f"{name} L={tile_width} niter={niter} {build}")
    check_mix(mix, ref, f"{name} mix")


@pytest.mark.gpu
def test_failed_per_voice_calls_change_nothing():
    """A rejected set_path_per_voice / set_property_per_voice leaves every voice rendering what it rendered without the call."""
    sc = SCENARIOS["trigger"]
    ref, inputs = _reference(sc)
    rt = _runtime(sc, 4, 0, "interp")
    assert rt.set_path_per_voice(sc.sid, ["len7", "no such resource"], np.arange(sc.n_voices) % 2) == 6
    assert rt.set_property_per_voice(sc.sid, "startOffset", np.where(np.arange(sc.n_voices) == 30, -1.0, 1.0)) == 6
    assert rt.set_property_per_voice(sc.sid, "stopOffset", [-2.0] * 5, 10) == 6
    got, _ = sc.run_gpu(rt, inputs)
    assert_exact(got, ref, "after failed per-voice calls")


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [0, 3])
def test_one_voice_graphs_in_the_batched_launch(stages):
    """BASELINE config 5 shape: one voice group per graph, launched together (render_groups_kernel), bit for bit what each graph
    renders alone in a single-group launch (and, where oracle/_ref is built, what the reference renders).  The warp pipeline
    (render_groups_pipe_kernel) does not cut a program with `sample`, whatever pipeline_stages says: like the control nodes, the op
    decodes its operands out of line, without the ring slots a cut would put between the stages (DESIGN.md section 4)."""
    n = 24
    sc = SCENARIOS["trigger"]
    names = sc.names
    rt = Runtime(SR, BS, n, device=0, pipeline_stages=stages)
    for name, data in sc.resources.items():
        assert rt.add_shared_resource(name, data)
    batches = [el.render(sample_common.one_voice_graph(v, names)) for v in range(n)]
    for v in range(n):
        assert rt.apply_instructions(batches[v], (v, v + 1)) == 0, rt.last_error()
    calls = (512, 7, 100, 333, 512, 65)
    got = np.concatenate([rt.process_voices(None, 1, c)[0] for c in calls], axis=2)
    groups = rt.describe()["groups"]
    assert len(groups) == n
    assert all(g.get("pipeline_stages", 1) == 1 for g in groups), [g.get("pipeline_stages") for g in groups]
    for v in range(n):
        alone = Runtime(SR, BS, 1, device=0)
        for name, data in sc.resources.items():
            assert alone.add_shared_resource(name, data)
        assert alone.apply_instructions(batches[v]) == 0
        want = np.concatenate([alone.process_voices(None, 1, c)[0] for c in calls], axis=2)
        assert_exact(got[v:v + 1], want, f"one-voice graph {v} batched, pipeline_stages={stages}")
        if orc.ref_available():
            o = orc.RefRuntime(SR, BS)
            for name, data in sc.resources.items():
                assert o.add_shared_resource(name, data)
            assert o.apply(batches[v]) == 0
            ref = np.concatenate([o.process(None, 1, c) for c in calls], axis=1)
            assert_exact(got[v:v + 1], ref[None], f"one-voice graph {v} against the reference")
