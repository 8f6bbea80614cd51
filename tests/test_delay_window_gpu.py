"""Delay lines on both sides of OP_DELAY's hoisted read window (render_ops.inc; the predicate is proven in
tests/test_delay_window_cpu.py), bit for bit against the reference in every K1 geometry, interpreted and specialised.

Lengths that take the hoisted window (per-voice constant, readFrac exact at the ring's magnitude, every lane of the warp agreeing)
and lengths that must not: fractional bits beyond the ring's magnitude, audio-rate lengths, lengths at the hazard bounds
hz + 1 / size - hz - 1 of every geometry, rings shorter than a sample tile, sizes that are not powers of two, and warps whose
voices disagree.  Lengths above the sample tile T take the tile-wide window (the ring loads of the whole tile issued ahead of its
stores), lengths up to T the per-element form; lengths near size - T read positions that later samples of the same tile
overwrite.  The process() sequence wraps the write and read indices inside slices and tiles many times."""
import pytest

from elementary_b200 import el
from k1_families import (CALLS, DENSE_WIDTHS, GEOMETRIES, Family, assert_build, assert_exact, check_family, make_runtime, reference,
                         run_calls)

IN0, IN1 = el.in_(0), el.in_(1)
BIG = (1 << 21) + 5           # 1000.5 fits its magnitude (1 fractional bit: sizes up to 2^22), 1000.125 does not (3 bits: 2^20)


def _k(key, v):
    return el.const(v, key=key)


FAM = Family("delay_window", [
    # hoistable lengths: SUBSYNTH32's 3001.5 among integers, halves and quarters (17.5 is a hazard where a slice holds 32 samples)
    el.delay({"size": 4800}, _k("dw_a", 3001.5), _k("dw_fa", 0.35), IN0),
    # warps mixing hoistable and inexact lengths (1234.5678: 13 fractional bits), pass-through and hazardous ones
    el.delay({"size": 4800}, _k("dw_b", 3001.5), 0.5, IN0),
    # a ring that is not a power of two, lengths at the hazard bounds of every slice length PER = 1 .. 32
    el.delay({"size": 300}, _k("dw_c", 100.0), _k("dw_fc", -0.6), IN0),
    # a ring shorter than the sample tile of the wide geometries (T = 128, 256): the per-element form
    el.delay({"size": 64}, _k("dw_d", 40.0), 0.7, IN0),
    # a ring past 2^21: 1000.5 hoisted, 1000.125 rejected
    el.delay({"size": BIG}, _k("dw_e", 1000.5), 0.25, IN0),
    # audio-rate length (integers 2999 .. 3002): the per-element form
    el.delay({"size": 4800}, el.add(3001.0, el.round_(el.mul(1.5, IN1))), 0.3, IN0),
    # constant length, audio-rate feedback
    el.delay({"size": 1000}, _k("dw_f", 500.5), el.mul(0.9, IN1), IN0),
], 2, "exact", keyed={
    "dw_a": [3001.5, 3001.5, 100.0, 2000.25, 4767.0, 33.0, 17.5, 4766.5, 3001.5, 1024.0, 4095.75],
    "dw_fa": [0.35, -0.9, 1.0, 0.0],
    "dw_b": [3001.5, 1234.5678, 3001.5, 0.0, 3001.5, 2.5, 4799.5, 4800.0, 3001.5, 1e-9, 6000.0, 4767.25],
    "dw_c": [2.0, 3.0, 5.0, 9.0, 17.0, 33.0, 267.0, 283.0, 291.0, 295.0, 297.0, 298.0, 17.5, 282.5, 150.75, 100.0, 266.5, 33.5],
    "dw_fc": [-0.6, 0.8],
    "dw_d": [17.0, 31.5, 40.0, 46.0, 46.5, 20.125, 30.0],
    "dw_e": [1000.5, 1000.125, 4096.0, 1000.5, 1000.5],
    "dw_f": [500.5, 999.0, 34.0, 500.5],
})


def _params():
    out = []
    for L, niter in GEOMETRIES:
        for build in ("interp", "spec"):
            out.append(pytest.param(L, niter, build, id=f"L{L}n{niter}-{build}"))
    for L in DENSE_WIDTHS:
        out.append(pytest.param(L, 0, "dense", id=f"L{L}n0-dense"))
    return out


_INTERP = {}


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width,niter,build", _params())
def test_delay_window_bit_exact(tile_width, niter, build):
    ref, inputs = reference(FAM)
    rt = make_runtime(FAM, tile_width, niter, build)
    got, mix = run_calls(rt, FAM, inputs, CALLS)
    assert_build(rt)
    what = f"delay_window L={tile_width} niter={niter} {build}"
    check_family(FAM, got, mix, ref, inputs, what)
    if build == "interp":
        _INTERP[(tile_width, niter)] = got
    elif (tile_width, niter) in _INTERP:
        assert_exact(got, _INTERP[(tile_width, niter)], what + " against the interpreter")
