"""CPU: the exact reference and the contract of K3 (tests/conv_exact.py) are right and sharp.

* `trim` drops exactly the taps the convolver drops (checked against the CPU restatement, oracle/libelem_oracle.so);
* `exact` reproduces the compiled reference's stored convolver outputs (tests/golden) within their float rounding;
* the float32 model of K3's algorithm stays at or below 0.25 of the bound on every signal of the GPU matrix;
* every planted fault of the model exceeds the bound by at least 4x on at least one of those signals — the evidence that the GPU
  contract of tests/test_convolve_exact_gpu.py would catch it."""
import os

import numpy as np
import pytest

import conv_exact as ce
from elementary_b200 import graphs
from oracle import oracle as orc

SR, BS = 48000.0, 512
LEAD = 1024
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_cases.npz"))


def root_fade(y):
    """The root's 20 ms fade-in (GainFade.h as restated in oracle/elem_oracle.cpp) applied per 512-sample block in float32: the
    gains, so that exact * gain is the fixture's faded convolution before its final rounding."""
    step = np.float32(1.0 / (SR * 20.0 / 1000.0))
    g = np.empty(y.shape[-1], np.float32)
    cur = np.float32(0.0)
    for b in range(0, y.shape[-1], BS):
        i = np.arange(min(BS, y.shape[-1] - b), dtype=np.float32)
        g[b:b + i.size] = 1.0 if cur == 1.0 else np.clip(cur + step * i, np.float32(0), np.float32(1))
        cur = np.clip(cur + step * np.float32(i.size), np.float32(0), np.float32(1))
    return g


@pytest.mark.parametrize("last", ["below", "at", "above"])
def test_trim_matches_the_port(last):
    v = {"below": np.nextafter(np.float32(1e-6), np.float32(0)), "at": np.float32(1e-6),
         "above": np.nextafter(np.float32(1e-6), np.float32(1))}[last]
    h = ce.make_ir("flat", 700, seed=5)
    h[-1] = v
    h[-2] = -v                                             # the tap before it survives only if the last one does not fall
    r = orc.PortRuntime(SR, BS)
    assert r.add_shared_resource("ir", h) and r.apply(graphs.convolve_channel("ir")) == 0
    x = np.zeros((1, 4 * BS), np.float32)
    x[0, LEAD] = 1.0                                       # an impulse after the root's fade-in: the output is the trimmed IR
    out = r.render(4, 1, BS, x)[0]
    kept = ce.trim(h).size
    assert kept == (700 if last != "below" else 698)
    assert abs(out[LEAD + 699]) > 5e-7 if kept == 700 else abs(out[LEAD + 699]) < 1e-9
    assert abs(out[LEAD + 698]) > 5e-7 if kept == 700 else abs(out[LEAD + 698]) < 1e-9
    assert abs(out[LEAD + 697]) > 1e-4


@pytest.mark.parametrize("taps", [16384, 700])
def test_exact_matches_the_reference_fixtures(taps):
    x = GOLD[f"convolve_{taps}_input"][0]
    want = GOLD[f"convolve_{taps}"][0].astype(np.float64)
    h = np.asarray(graphs.lcg_ir(16384)[:taps], dtype=np.float32)
    y = ce.exact(x, h)
    E = ce.bound(x, h)
    faded = y * root_fade(y)
    tol = ce.C * E + ce.U * ce.block_error(faded, np.zeros_like(faded))    # + the rounding of the fade's product
    r = ce.ratio(want, faded, tol)
    assert r.max() <= 1.0, r.max()
    assert np.abs(want).max() > 0.01


def matrix_signals(S):
    """The GPU matrix's inputs for an IR of S partitions, whole blocks."""
    n = LEAD + 3 * ce.P * len(ce.IMPULSE_OFFSETS) + (S + 2) * ce.P
    n = -(-n // ce.P) * ce.P
    kinds = [(k, 1) for k in ce.INPUT_KINDS] + [("noise", 2), ("impulses", 0)]
    return np.stack([ce.make_input(k, n, seed=s, lead=LEAD) for k, s in kinds])


def ratios(h, fault=None):
    x = matrix_signals(ce.partitions(h))
    return ce.ratio(ce.model(x, h, fault), ce.exact(x, h), ce.bound(x, h))


@pytest.mark.parametrize("kind", ce.IR_KINDS)
def test_faultless_model_stays_within_a_quarter_of_the_bound(kind):
    worst = max(ratios(ce.make_ir(kind, taps, seed=taps + 7, tail=tail)).max() for taps, tail in ce.LENGTHS)
    assert worst <= 0.25 * ce.C, worst


FAULT_IRS = [("flat", 4097), ("taps", 4097), ("lcg", 16384), ("flat", 1025)]


@pytest.mark.parametrize("fault", ce.FAULTS)
def test_every_planted_fault_exceeds_the_bound_four_times(fault):
    worst = max(ratios(ce.make_ir(kind, taps, seed=taps + 7), fault).max() for kind, taps in FAULT_IRS)
    assert worst >= 4.0 * ce.C, worst


@pytest.mark.parametrize("fault", ["bin0", "bin256", "bin512", "pack"])
def test_bin_faults_are_caught_by_the_input_that_excites_the_bin(fault):
    """The special-cased bins: DC (bin 0 and the packed pair), fs/4 (bin 256), Nyquist (bin 512), each through a flat IR, whose
    every partition carries energy in every bin."""
    kind = {"bin0": "dc", "bin256": "quarter", "bin512": "alternating", "pack": "dc"}[fault]
    h = ce.make_ir("flat", 4097, seed=9)
    x = ce.make_input(kind, LEAD + 16 * ce.P, lead=LEAD)[None]
    r = ce.ratio(ce.model(x, h, fault), ce.exact(x, h), ce.bound(x, h)).max()
    assert r >= 4.0 * ce.C, r
    assert ce.ratio(ce.model(x, h), ce.exact(x, h), ce.bound(x, h)).max() <= 0.25 * ce.C
