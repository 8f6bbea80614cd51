"""The K1 test matrix: every node family, in every tile geometry, in the interpreter and in the per-program specialised kernel,
against the reference, to the exactness DESIGN.md section 4 documents.

K1 has six tile geometries (L = 1, 2, 4, 8, 16, 32 voices per warp), three `niter` variants and two builds of the same text (the
interpreter and the NVRTC specialisation, plus its dense 64-register variant).  Many node bodies take a different code path per
geometry: the rand jump, the column walks of pole / env / biquad with their partial-tile bound, the svf scan and its serial form,
the delay fast path with its hazard window, the phasor run.  Each family below is one multi-root graph (<= 8 outputs) with its own
contract, rendered for 45 voices (a ragged last tile for every L) that differ in their keyed constants, seeds and input noise, through
a sequence of process() lengths that hits cnt < T, cnt == T and cnt == T +- 1 for every tile length T.

Contracts (DESIGN.md section 4, "Numerics"):

* ``exact``  -- np.array_equal against the reference for every voice and sample (NaN equals only NaN).  The kernels are compiled
  without FTZ, without fast math and without FMA contraction, and these nodes are sequences of IEEE float operations in the order
  of the reference: nothing may differ.  The interpreter and the specialised kernel must also be identical to each other.
* ``filter`` -- svf / svfshelf / mm1p compute in double.  The departures from the reference (Taylor tan, (pi fc) * (1 / sr) for
  pi fc / sr, rcp.approx + Newton, FMA contraction, the warp scan) are about 1e-16 relative (5e-13 for tan) of the double state.
  Three things amplify them: tan's condition number near Nyquist (fc at the sr / 2.0001 clamp: about 2e4), the resonance (q up
  to 20) and the cancellation of a highpass whose cutoff sits above the signal.  Measured on an H100, the worst case (highpass, fc
  at the clamp) is 1.7e-9 of the block peak, so: |gpu - ref| <= 1 ulp_f32(|ref|) + 1e-8 * block peak (DESIGN.md section 4).  The 1e-5 * block peak bound of the rest of the
  suite must also hold.
* ``math``   -- element-wise functions against a float64 NumPy evaluation of the same function on the same float32 inputs, within
  the maximum ulp error the CUDA 12 Math API documentation states for the single-precision function; results that are exact in
  IEEE arithmetic (sqrt, abs, floor, ceil, round, + - * /, fmod, min, max, compares) bit-exact against the reference.  A build with
  fast math (__sinf and friends) or FTZ (subnormal inputs and outputs flushed) breaks it.
* ``peak``   -- blep oscillators: |gpu - ref| <= 1e-5 * block peak, as in tests/test_parity_gpu.py.

The mix bus is compared with the float64 sum of the per-voice references in every run.  The families, their references and the
checks live in tests/k1_families.py.
"""
import os
import re

import numpy as np
import pytest

from elementary_b200 import Runtime, graphs
from elementary_b200.runtime import FLAG_VOICE_IN, FLAG_VOICE_OUT
from helpers import block_peak_tolerance_check, oracle_cls
from k1_families import (BS, CALLS, DENSE_WIDTHS, FADE_END, FAMILIES, GEOMETRIES, MATH_FAMILIES, N_VOICES, RATE_FAMILIES, SR,
                         assert_build, assert_exact, check_family, family_inputs, make_runtime, reference, run_calls)


# ---- A/B/C: families x geometries x builds ----------------------------------------------------------------------------

# Every (family, geometry) pair of a specialised arm is one NVRTC compile of a few seconds.  By default each family runs the
# interpreter in every geometry and the specialised kernel in three geometries (the dense build in one width), rotated over the
# families so that together they cover every geometry several times; ELEM_B200_MATRIX_FULL=1 runs the whole cross product.
FULL = os.environ.get("ELEM_B200_MATRIX_FULL") == "1"


def _matrix_params():
    out = []
    for i, (f, fam) in enumerate(FAMILIES.items()):
        spec_geoms = GEOMETRIES if FULL else [GEOMETRIES[(i + 3 * j) % len(GEOMETRIES)] for j in range(3)]
        dense_widths = DENSE_WIDTHS if FULL else [DENSE_WIDTHS[i % len(DENSE_WIDTHS)]]
        for L, niter in GEOMETRIES:
            out.append(pytest.param(f, L, niter, "interp", id=f"{f}-L{L}n{niter}-interp"))
            if (L, niter) in spec_geoms:
                out.append(pytest.param(f, L, niter, "spec", id=f"{f}-L{L}n{niter}-spec"))
        if fam.contract != "math":       # the element-wise layout is the least geometry-specific: no dense arm
            for L in dense_widths:
                out.append(pytest.param(f, L, 0, "dense", id=f"{f}-L{L}n0-dense"))
    return out


_INTERP_OUT = {}


def _interp_output(fam, L, niter, ref_inputs):
    key = (fam.name, L, niter)
    if key not in _INTERP_OUT:
        rt = make_runtime(fam, L, niter, "interp")
        _INTERP_OUT[key] = run_calls(rt, fam, ref_inputs, CALLS)[0]
    return _INTERP_OUT[key]


@pytest.mark.gpu
@pytest.mark.parametrize("family,tile_width,niter,build", _matrix_params())
def test_family_matrix(family, tile_width, niter, build):
    """One family, one geometry, one build, 45 voices through the short / ragged process() sequence CALLS, against the reference."""
    fam = FAMILIES[family]
    ref, inputs = reference(fam)
    rt = make_runtime(fam, tile_width, niter, build)
    got, mix = run_calls(rt, fam, inputs, CALLS)
    assert_build(rt)
    what = f"{family} L={tile_width} niter={niter} {build}"
    check_family(fam, got, mix, ref, inputs, what)
    if build == "interp":
        _INTERP_OUT[(family, tile_width, niter)] = got
    elif fam.contract == "exact":
        assert_exact(got, _interp_output(fam, tile_width, niter, inputs), what + " against the interpreter")
    if family == "subnormal":
        tiny = np.abs(got[:, :, FADE_END:])
        for c in range(2):
            assert ((tiny[:, c] > 0) & (tiny[:, c] < 1.1754944e-38)).sum() > 100, f"{what}: no subnormal outputs on root {c}"


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(FAMILIES))
def test_family_single_partial_tile(family, build="interp"):
    """5 voices at L = 32: one warp whose tile is mostly empty lanes."""
    fam = FAMILIES[family]
    ref, inputs = reference(fam, n_voices=5)
    rt = make_runtime(fam, 32, 0, build, n_voices=5)
    got, mix = run_calls(rt, fam, inputs, CALLS)
    assert_build(rt)
    check_family(fam, got, mix, ref, inputs, f"{family} 5 voices L=32 {build}")


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width", [1, 2, 8, 32])
def test_families_as_voice_groups_in_one_launch(tile_width):
    """Every family on its own voice range of ONE runtime: one batched render_groups_kernel launch (+ one mix reduce) per
    process() call renders them all, with tables read from global memory instead of the shared-memory copy."""
    per = max(8, tile_width)
    names = list(FAMILIES)
    n_in = max(f.n_in for f in FAMILIES.values())
    rt = Runtime(SR, BS, per * len(names), device=0, tile_width=tile_width, specialize=0)
    for f in FAMILIES.values():
        for name, data in f.resources.items():
            assert rt.add_shared_resource(name, data)
    inputs = np.zeros((per * len(names), n_in, sum(CALLS)), dtype=np.float32)
    refs = {}
    for i, name in enumerate(names):
        fam = FAMILIES[name]
        assert rt.apply_instructions(fam.batch, voices=(per * i, per * (i + 1))) == 0, rt.last_error()
        fam.setup(rt, per * i, per)
        ref, fin = reference(fam)
        refs[name] = ref[:per]
        if fin is not None:
            inputs[per * i:per * (i + 1), :fam.n_in] = fin[:per]
    groups = rt.describe()["groups"]
    assert len(groups) == len(names) and all(g["tile_width"] == tile_width for g in groups), groups
    l0 = rt.kernel_launches
    got, mix = run_calls(rt, None, inputs, CALLS, n_out=8)
    assert rt.kernel_launches - l0 == 2 * len(CALLS), "one K1 launch for all groups + one mix reduce per process() call"
    for i, name in enumerate(names):
        fam = FAMILIES[name]
        g = got[per * i:per * (i + 1), :fam.n_out]
        check_family(fam, g, None, refs[name], None if fam.n_in == 0 else inputs[per * i:per * (i + 1), :fam.n_in],
                     f"{name} group L={tile_width}")


@pytest.mark.gpu
@pytest.mark.parametrize("sr,bs", [(48000.0, 480), (44100.0, 441), (96000.0, 1024)])
@pytest.mark.parametrize("tile_width", [1, 4, 32])
@pytest.mark.parametrize("family", RATE_FAMILIES)
def test_filter_and_delay_families_at_other_rates_and_block_sizes(family, tile_width, sr, bs):
    fam = FAMILIES[family]
    calls = (bs, bs, 7, bs - 7, 1, bs, bs)
    ref, inputs = reference(fam, calls, sr, bs)
    rt = make_runtime(fam, tile_width, 0, "interp", sr=sr, bs=bs)
    got, mix = run_calls(rt, fam, inputs, calls)
    check_family(fam, got, mix, ref, inputs, f"{family} L={tile_width} sr={sr:g} bs={bs}", bs)


# ---- D: the benchmarked kernels at scale ------------------------------------------------------------------------------

def _subsynth_class_refs(n_blocks):
    vb = [graphs.subsynth32_voice_props(v) for v in range(40)]
    outs = []
    for v in range(40):
        o = oracle_cls()(SR, BS)
        assert o.apply(graphs.subsynth32()) == 0 and o.apply(vb[v]) == 0
        outs.append(o.render(n_blocks, 1)[0])
    return np.stack(outs)


@pytest.mark.gpu
@pytest.mark.parametrize("n_voices,tile_width,dense", [(4096, 2, False), (8192, 2, True), (16384, 4, True)])
def test_subsynth32_specialised_at_scale(n_voices, tile_width, dense):
    """SUBSYNTH32 through the specialised kernels the benchmark times, in the geometry the engine picks on its own: L = 2 at 4096
    voices; from 8192 voices up the dense mid range (4096 warps, kernels compiled for 8 CTAs per SM, at most 64 registers).
    Every voice, block by block, against its class reference."""
    n_blocks = 12
    rt = Runtime(SR, BS, n_voices, device=0, specialize=2, specialize_strict=1)
    assert rt.apply_instructions(graphs.subsynth32()) == 0, rt.last_error()
    ida, idb = graphs.subsynth32_param_ids()
    f0 = np.array([graphs.subsynth32_f0(v) for v in range(n_voices)])
    assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    ref = _subsynth_class_refs(n_blocks)
    cls = np.arange(n_voices) % 40
    worst = 0.0
    for b in range(n_blocks):
        got, mix = rt.process_voices(None, 1, BS)
        if b == 0:
            g = rt.describe()["groups"][0]
            assert g["tile_width"] == tile_width and g.get("spec_state") == 2, g
            if dense:
                assert 0 < g["spec_regs"] <= 64, g
        r = ref[:, b * BS:(b + 1) * BS]
        ok, w, ex = block_peak_tolerance_check(got[:, 0], r[cls], BS)
        assert ok, f"block {b}: worst err/tol {w:.3g}, bit-exact {ex:.4f}"
        worst = max(worst, w)
        want = r[cls].astype(np.float64).sum(axis=0)
        assert np.abs(mix[0] - want).max() <= 1e-5 * np.abs(want).max() + 1e-7
    print(f"MATRIX subsynth32 {n_voices} voices L={tile_width} spec: worst_err_over_tol={worst:.3g} regs={g.get('spec_regs')}")


# ---- E: chain fusion is bit-identical ---------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("tile_width", [1, 8])
def test_fuse_chains_off_is_bit_identical(tile_width):
    """DESIGN.md section 2.4: fusing element-wise runs into one OP_CHAIN keeps every operation and its order, so the samples are the
    same bits as with fusion off."""
    cases = [(FAMILIES[f], None) for f in MATH_FAMILIES] + [(None, graphs.random_graph(s, 48)) for s in (7, 8, 9)]
    for fam, batch in cases:
        n_voices = 33
        outs = []
        for fuse in (1, 0):
            rt = Runtime(SR, BS, n_voices, device=0, tile_width=tile_width, specialize=0, fuse_chains=fuse)
            if fam is not None:
                assert rt.apply_instructions(fam.batch) == 0
                fam.setup(rt)
                inputs = family_inputs(fam, n_voices, sum(CALLS))
                outs.append(run_calls(rt, fam, inputs, CALLS))
            else:
                assert rt.apply_instructions(batch) == 0
                outs.append(rt.render_voices(5, 1))
        (va, ma), (vb, mb) = outs
        what = fam.name if fam is not None else "random graph"
        assert np.array_equal(va, vb, equal_nan=True), what
        assert np.array_equal(ma, mb, equal_nan=True), what


# ---- E: every opcode and chain function has a matrix entry (CPU) --------------------------------------------------------

EXCLUDED_OPCODES = {
    "OP_END": "terminates every program",
    "OP_PROMOTE": "tap promotion records behind the program",
    "OP_STOREBUF": "stage boundary around convolve: tests/test_convolve_gpu.py",
    "OP_LOADBUF": "stage boundary around convolve: tests/test_convolve_gpu.py",
    "OP_CUSTOM": "registered node types: tests/test_parity_gpu.py",
}


def _enum(name):
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "..", "elementary_b200", "csrc", "program.h")) as f:
        text = f.read()
    body = re.search(r"enum " + name + r"\s*:\s*uint32_t\s*\{(.*?)\};", text, re.S).group(1)
    body = re.sub(r"//[^\n]*", "", body)
    values, nxt = {}, 0
    for item in [s.strip() for s in body.split(",") if s.strip()]:
        m = re.match(r"(\w+)\s*(?:=\s*(\w+))?$", item)
        nm, val = m.group(1), m.group(2)
        nxt = int(val, 0) if val is not None else nxt
        values[nm] = nxt
        nxt += 1
    return values


def program_ops(words):
    """(opcode, chain fns) of every op of a program: [8 header words][operand words], ended by OP_END."""
    ops, fns, pc = [], set(), 0
    while pc < len(words):
        w0 = int(words[pc])
        opcode, nwords = w0 & 0xFF, (w0 >> 8) & 0xFF
        if opcode == 0:
            break
        ops.append(opcode)
        if opcode == 5:                                     # OP_CHAIN: operand 0, then (fn word, operand word) per step
            for s in range(int(words[pc + 6])):
                fns.add(int(words[pc + 8 + 1 + 2 * s]) & 0xFF)
        pc += 8 + nwords
    return ops, fns


def test_matrix_families_emit_every_opcode_and_chain_fn():
    """A node added to the engine without an entry in the matrix fails here, on a CPU: the families' programs (plan-only runtime)
    together contain every opcode of program.h except the named exclusions, and every chain function."""
    opcodes = {k: v for k, v in _enum("Opcode").items() if k != "OP_COUNT_"}
    chain_fns = _enum("ChainFn")
    assert opcodes["OP_CHAIN"] == 5 and opcodes["OP_END"] == 0
    seen_ops, seen_fns = set(), set()
    for fam in FAMILIES.values():
        rt = Runtime(SR, BS, N_VOICES, device=-1, tile_width=4, plan_dry_run=1)
        for name, data in fam.resources.items():
            assert rt.add_shared_resource(name, data)
        assert rt.apply_instructions(fam.batch) == 0, (fam.name, rt.last_error())
        assert fam.n_out <= 8
        if fam.n_in:       # host-input reads are compiled once a block says how many channels there are (host side only here)
            rt.enqueue_block(fam.n_in, fam.n_out, BS, flags=FLAG_VOICE_IN | FLAG_VOICE_OUT)
        ops, fns = program_ops(rt.program_words(0))
        assert ops, fam.name
        seen_ops |= set(ops)
        seen_fns |= fns
    missing = sorted(k for k, v in opcodes.items() if v not in seen_ops and k not in EXCLUDED_OPCODES)
    assert not missing, f"opcodes without a matrix family: {missing}"
    missing_fns = sorted(k for k, v in chain_fns.items() if v not in seen_fns)
    assert not missing_fns, f"chain functions without a matrix family: {missing_fns}"
    assert set(EXCLUDED_OPCODES) <= set(opcodes)
