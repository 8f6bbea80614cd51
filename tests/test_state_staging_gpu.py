"""K1's staging of state and parameter rows (render_kernel.cu, the prologue and the state write-back of render_tile): all 32 lanes
of a warp take part, 32 / L state entries and as many parameters per pass, and an entry's shared-memory row is found by a warp
vote over the doubles before it.  This graph has more state entries and parameters than one pass holds at every tile width, with
double-precision state (svf, mm1p: 8-byte aligned, so padding rows appear) between float rows, and per-voice parameter values, so a
row staged to the wrong place, for the wrong voice, or written back wrongly changes the output of the next process() call.
Checked against per-voice reference instances in every K1 geometry, interpreted and specialised, and cut into pipeline stages,
where each stage stages only the state rows of its own ops."""
import numpy as np
import pytest

from elementary_b200 import Runtime, el
from helpers import block_peak_tolerance_check, oracle_cls
from k1_families import (BS, CALLS, DENSE_WIDTHS, GEOMETRIES, SR, Family, assert_build, assert_exact, check_family, make_runtime,
                         reference, run_calls)

IN0, IN1 = el.in_(0), el.in_(1)


def _k(key, v):
    return el.const(v, key=key)


_KEYED = {f"sg_p{i}": [0.5 + 0.03 * i, 0.9 - 0.02 * i, 0.0, 0.99, -0.4 + 0.05 * i] for i in range(12)}
_KEYED.update({f"sg_r{i}": [0.1 * (i % 9), 0.95, 0.7 - 0.04 * i] for i in range(12)})
_KEYED.update({f"sg_f{i}": [55.0 * (i + 1), 440.0 + i, 3.5 * i + 1.0, -120.0] for i in range(6)})
_KEYED.update({
    "sg_fc0": [1000.0, 120.0, 8000.0, 23000.0], "sg_q0": [0.7, 3.0, 0.3],
    "sg_fc1": [300.0, 5000.0, 45.0], "sg_q1": [1.0, 0.5, 12.0],
    "sg_b0": [0.2, 1.0, 0.06], "sg_b1": [0.4, 0.0, 0.12], "sg_b2": [0.2, 0.0, 0.06], "sg_b3": [-0.5, 0.0, -1.6], "sg_b4": [0.3, 0.0, 0.8],
    "sg_m": [2000.0, 150.0, 12000.0], "sg_ea": [0.9, 0.1], "sg_er": [0.99, 0.5, 0.999],
})


def _roots(x0, x1):
    return [
        el.add(*[el.pole(_k(f"sg_p{i}", 0.5), x0) for i in range(12)]),
        el.svf({"mode": "lowpass"}, _k("sg_fc0", 1000.0), _k("sg_q0", 0.7), x0),
        el.biquad(*[_k(f"sg_b{i}", 0.0) for i in range(5)], x1),
        el.mm1p({"mode": "lowpass"}, el.prewarp(_k("sg_m", 2000.0)), x0),
        el.add(*[el.pole(_k(f"sg_r{i}", 0.5), x1) for i in range(12)]),
        el.svf({"mode": "highpass"}, _k("sg_fc1", 300.0), _k("sg_q1", 1.0), x1),
        el.add(*[el.phasor(_k(f"sg_f{i}", 100.0)) for i in range(6)]),
        el.env(_k("sg_ea", 0.9), _k("sg_er", 0.99), x0),
    ]


FAM = Family("state_staging", _roots(IN0, IN1), 2, "filter", keyed=_KEYED)


def _params():
    out = []
    for L, niter in GEOMETRIES:
        for build in ("interp", "spec"):
            out.append(pytest.param(L, niter, build, id=f"L{L}n{niter}-{build}"))
    for L in DENSE_WIDTHS:
        out.append(pytest.param(L, 0, "dense", id=f"L{L}n0-dense"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width,niter,build", _params())
def test_state_staging_every_geometry(tile_width, niter, build):
    ref, inputs = reference(FAM)
    rt = make_runtime(FAM, tile_width, niter, build)
    g = rt.describe()["groups"][0]
    assert g["state_rows"] > 32 and g["params"] > 32, g          # more than one staging pass at every tile width
    got, mix = run_calls(rt, FAM, inputs, CALLS)
    assert_build(rt)
    check_family(FAM, got, mix, ref, inputs, f"state_staging L={tile_width} niter={niter} {build}")


PIPE_VOICES = 4


def _pipe_run(batch, stages):
    rt = Runtime(SR, BS, PIPE_VOICES, device=0, specialize=0, pipeline_stages=stages)
    for v in range(PIPE_VOICES):
        assert rt.apply_instructions(batch, voices=(v, v + 1)) == 0, rt.last_error()
        assert rt.apply_instructions(FAM.voice_batch(v), voices=(v, v + 1)) == 0, rt.last_error()
    got = np.concatenate([rt.process_voices(None, 1, n)[0] for n in CALLS], axis=2)
    return got, rt.describe()["groups"]


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [2, 3, 4])
def test_state_staging_pipeline_stages(stages):
    saw = lambda f: el.sub(el.mul(2.0, el.phasor(f)), 1.0)            # one voice per group, no host inputs: oscillators drive the filters
    batch = el.render(el.add(*_roots(saw(110.0), saw(37.0))))
    got, groups = _pipe_run(batch, stages)
    assert all(g["pipeline_stages"] == stages for g in groups), groups
    base, _ = _pipe_run(batch, 0)
    what = f"state_staging pipelined W={stages}"
    assert_exact(got, base, what + " against pipeline_stages=0")
    refs = []
    for v in range(PIPE_VOICES):
        o = oracle_cls()(SR, BS)
        assert o.apply(batch) == 0 and o.apply(FAM.voice_batch(v)) == 0
        refs.append(np.concatenate([o.process(None, 1, n) for n in CALLS], axis=1))
    ok, worst, exact = block_peak_tolerance_check(got, np.stack(refs), BS)   # the sum of the roots: the svf's ulp is not the sum's
    assert ok, f"{what}: worst err/tol {worst:.3g}, bit-exact {exact:.4f}"
