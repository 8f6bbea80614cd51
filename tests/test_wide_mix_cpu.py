"""The float32 model of the wide mix bus (tests/wide_mix_model.py) is right and sharp, on a CPU; the host side of the wide path on a
plan-only engine.

Right: it agrees bit for bit with the dense model (tests/mix_model.py) where the two must agree, and stays within the depth bound of
the exact float64 sum of every channel.  Sharp: on a designed input, each fault the compact layout could plausibly have changes the
bits of the model's output, so a GPU mix that equals the model bit for bit (tests/test_wide_mix_gpu.py) has none of them.
"""
import json

import numpy as np
import pytest

from elementary_b200 import Runtime, el
from elementary_b200.runtime import FLAG_MIX
from mix_model import k2_groups, mix_model
from wide_mix_model import (MAX_WIDE_OUT_CHANNELS, channel_bound, mix_channels, wide_k2, wide_mix_model, wide_rows)


def _layout(*groups):
    return [{"v0": v0, "nv": nv, "tile_width": L, "slots": 1, "mix_channels": list(ch)} for v0, nv, L, ch in groups]


def _designed(n_voices, n_out, n, salt=0):
    """Per-voice, per-channel gains +-2^k, k in [-20, 20], rotating with the sample (tests/test_mix_model_cpu.py, one salt per
    channel): every tile is among the largest terms of its channels at some sample, so every change of summation order shows."""
    v = np.arange(n_voices)[:, None, None]
    c = np.arange(n_out)[None, :, None]
    t = np.arange(n)[None, None, :]
    k = (7 * v + 13 * t + 5 * c + salt) % 41 - 20
    sign = np.where((v * 5 + c + salt) % 3 == 0, -1.0, 1.0)
    mant = 1.0 + ((v * 37 + t * 11 + c * 3 + salt) % 97) / 97.0
    return (sign * mant * np.exp2(k)).astype(np.float32)


def _random(n_voices, n_out, n, seed):
    rng = np.random.default_rng(seed)
    scale = 10.0 ** rng.uniform(-3.0, 3.0, size=(n_voices, 1, 1))
    return (rng.standard_normal((n_voices, n_out, n)) * scale).astype(np.float32)


N_OUT = 16
N = 64
# widths 4, 1, 8, 2 (150 + 300 + 50 + 350 tiles); |R_0| = 200 (G = 1), |R_3| = 800 (G = 4), |R_9| = 500 (G = 2), |R_12| = 400
# (G = 2), channel 20 is past nOut, the other channels have no rows.  1900 rows in all (G would be 8).
FAULT_LAYOUT = _layout((0, 600, 4, (0, 3, 9)), (600, 300, 1, (3, 9, 20)), (900, 400, 8, (0, 9, 12)), (1300, 700, 2, (3, 12)))


@pytest.fixture(scope="module")
def designed():
    x = _designed(2000, N_OUT, N)
    P, R = wide_rows(x, FAULT_LAYOUT, N_OUT)
    assert [len(r) for r in R][:13] == [200, 0, 0, 800, 0, 0, 0, 0, 0, 500, 0, 0, 400]
    assert P.shape[0] == 1900 and k2_groups(1900) == 8
    good = wide_mix_model(x, FAULT_LAYOUT, N_OUT)
    assert np.array_equal(good, wide_k2(P, R, N))
    return x, P, R, good


def _differs(a, b):
    return bool((np.asarray(a).view(np.uint32) != np.asarray(b).view(np.uint32)).any())


def test_mix_channels_of_a_group():
    g = {"v0": 0, "nv": 4, "tile_width": 2, "slots": 1, "mix_channels": [0, 3, 9, 20]}
    assert mix_channels(g, 16) == [0, 3, 9] and mix_channels(g, 21) == [0, 3, 9, 20] and mix_channels(g, 3) == [0]
    assert mix_channels({"v0": 0, "nv": 4, "tile_width": 0, "mix_channels": [1]}, 16) == []
    assert mix_channels({"v0": 0, "nv": 4, "tile_width": 2}, 16) == []                    # no program yet


def test_empty_channels_are_positive_zero(designed):
    x, P, R, good = designed
    for c in range(N_OUT):
        if not R[c]:
            assert (good[c].view(np.uint32) == 0).all(), c


@pytest.mark.parametrize("writers", [(0,), (1, 3), (0, 1, 2, 3)])
def test_agrees_with_the_dense_model_on_channel_zero(writers):
    """Every group writes channel 0 only (or nothing): channel 0 of the wide model equals mix_model over the groups that write it."""
    base = [(0, 600, 4), (600, 300, 1), (900, 400, 8), (1300, 700, 2)]
    lay = _layout(*[(v0, nv, L, (0,) if i in writers else (-1, 30)) for i, (v0, nv, L) in enumerate(base)])
    x = _designed(2000, N_OUT, N, salt=3)
    got = wide_mix_model(x, lay, N_OUT)
    want = mix_model(x[:, :1], [g for i, g in enumerate(lay) if i in writers])
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32))
    assert not got[1:].any()


@pytest.mark.parametrize("seed", range(4))
def test_within_the_depth_bound_of_the_exact_sum(seed):
    x = _random(2000, N_OUT, 48, seed)
    got = wide_mix_model(x, FAULT_LAYOUT, N_OUT).astype(np.float64)
    for c in range(N_OUT):
        bound, d = channel_bound(x, FAULT_LAYOUT, N_OUT, c)
        if bound is None:
            assert not got[c].any()
            continue
        exact = sum(x[g["v0"]:g["v0"] + g["nv"], c].astype(np.float64).sum(axis=0)
                    for g in FAULT_LAYOUT if c in mix_channels(g, N_OUT))
        err = np.abs(got[c] - exact)
        assert (err <= bound).all(), f"channel {c}: err / bound = {float((err / bound).max()):.3g} (d = {d})"


# ---- sharpness ------------------------------------------------------------------------------------------------------------

def test_fault_row_under_the_wrong_channel(designed):
    x, P, R, good = designed
    for a, b in ((0, 3), (3, 9), (9, 12), (12, 0), (3, 5)):
        for i in (0, len(R[a]) // 2, len(R[a]) - 1):
            Q = [list(r) for r in R]
            Q[b].append(Q[a].pop(i))
            Q[b].sort()
            assert _differs(wide_k2(P, Q, N), good), f"row {i} of channel {a} under channel {b} is invisible"


def test_fault_two_compact_indices_exchanged(designed):
    x, P, R, good = designed
    for gi, g in enumerate(FAULT_LAYOUT):
        nc = len(mix_channels(g, N_OUT))
        for k0 in range(nc):
            for k1 in range(k0 + 1, nc):
                Q, R2 = wide_rows(x, FAULT_LAYOUT, N_OUT, exchange=(gi, k0, k1))
                assert R2 == R
                assert _differs(wide_k2(Q, R, N), good), f"compact channels {k0} and {k1} of group {gi} exchanged is invisible"


def test_fault_group_rows_out_of_engine_order(designed):
    """One group's run of rows moved to the front of a channel's list (the groups of the channel in another order)."""
    x, P, R, good = designed
    for c in (0, 3, 9, 12):
        owners = [gi for gi, g in enumerate(FAULT_LAYOUT) if c in mix_channels(g, N_OUT)]
        bounds, base = [], 0
        for gi, g in enumerate(FAULT_LAYOUT):
            n_t = (g["nv"] + g["tile_width"] - 1) // g["tile_width"]
            if gi in owners:
                bounds.append((base, base + n_t))
                base += n_t
        for lo, hi in bounds[1:]:
            Q = [list(r) for r in R]
            Q[c] = R[c][lo:hi] + R[c][:lo] + R[c][hi:]
            assert _differs(wide_k2(P, Q, N), good), f"channel {c}: a group's rows out of engine order is invisible"


def test_fault_row_counted_twice(designed):
    x, P, R, good = designed
    for c in (0, 3, 9, 12):
        for i in range(0, len(R[c]), 37):
            Q = [list(r) for r in R]
            Q[c].insert(i + 1, R[c][i])
            assert _differs(wide_k2(P, Q, N), good), f"row {i} of channel {c} counted twice is invisible"


def test_fault_group_count_from_the_total_row_count(designed):
    x, P, R, good = designed
    total = P.shape[0]
    bad = wide_k2(P, R, N, groups_of=lambda c, rows: k2_groups(total))
    for c in (0, 3, 9, 12):
        assert k2_groups(len(R[c])) != k2_groups(total)
        assert _differs(bad[c], good[c]), f"channel {c}: G from the total row count is invisible"


# ---- plan-only engine: what the host reports and accepts --------------------------------------------------------------------

def _roots_batch(pairs):
    """One root per (channel, graph) — several may share a channel or aim outside [0, nOut)."""
    r = el.Renderer()
    batch = r.render(*[g for _, g in pairs])
    # the renderer numbers channels by position: rewrite the channel prop of each root in order
    roots = batch[-2][1]
    by_id = {}
    for ins in batch:
        if ins[0] == 3 and ins[2] == "channel" and ins[1] in roots:
            by_id[ins[1]] = ins
    for rid, (ch, _) in zip(roots, pairs):
        by_id[rid][3] = ch
    return batch


def _graphs(n):
    return [el.mul(float(i + 1), el.phasor(el.const(10.0 + i, key=f"wf{i}"))) for i in range(n)]


def test_describe_reports_mix_channels_plan_only():
    rt = Runtime(48000.0, 512, 12, device=-1, plan_dry_run=1)
    g = _graphs(4)
    assert rt.apply_instructions(_roots_batch([(3, g[0]), (3, g[1]), (9, g[2])]), voices=(0, 4)) == 0, rt.last_error()   # overlapping
    assert rt.apply_instructions(_roots_batch([(0, g[0]), (12, g[3])]), voices=(4, 8)) == 0, rt.last_error()           # disjoint
    assert rt.apply_instructions(_roots_batch([(-1, g[1]), (40, g[2]), (5, g[3])]), voices=(8, 12)) == 0, rt.last_error()  # out of range
    rt.enqueue_block(0, 16, 512, flags=FLAG_MIX)
    groups = rt.describe()["groups"]
    assert [(x["v0"], x["nv"]) for x in groups] == [(0, 4), (4, 4), (8, 4)]
    assert [x["mix_channels"] for x in groups] == [[3, 9], [0, 12], [5, 40]]
    assert [mix_channels(x, 16) for x in groups] == [[3, 9], [0, 12], [5]]


def test_channel_cap_plan_only():
    rt = Runtime(48000.0, 128, 4, device=-1, plan_dry_run=1)
    g = _graphs(2)
    assert rt.apply_instructions(_roots_batch([(0, g[0]), (MAX_WIDE_OUT_CHANNELS - 1, g[1])])) == 0, rt.last_error()
    lib, h = rt._lib, rt._h
    assert lib.elem_b200_enqueue_block(h, 0, MAX_WIDE_OUT_CHANNELS, 128, FLAG_MIX) == 0, rt.last_error()
    assert lib.elem_b200_enqueue_block(h, 0, MAX_WIDE_OUT_CHANNELS + 1, 128, FLAG_MIX) == -2
    assert "output channels" in rt.last_error()
    assert lib.elem_b200_enqueue_block(h, 0, 9, 128, FLAG_MIX | 2) == 0, rt.last_error()
    assert json.loads(json.dumps(rt.describe()))["groups"][0]["mix_channels"] == [0, MAX_WIDE_OUT_CHANNELS - 1]
