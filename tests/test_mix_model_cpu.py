"""The float32 model of the mix bus (tests/mix_model.py) is right and sharp, on a CPU.

Right: on random inputs it stays within the depth bound gamma_d * sum |x| of the exact (float64) sum, d derived from the summation
tree of the layout.  Sharp: on a designed input, each fault the engine could plausibly have in its mix path changes the bits of the
model's output, so a GPU mix that equals the model bit for bit (tests/test_voice_groups_gpu.py) has none of them.
"""
import numpy as np
import pytest

from mix_model import butterfly, depth, k2, k2_groups, k2_per_group, mix_bound, mix_model, tile_rows


def _layout(*groups):
    return [{"v0": v0, "nv": nv, "tile_width": L, "slots": 1} for v0, nv, L in groups]


def _random_voices(n_voices, n_out, n, seed):
    rng = np.random.default_rng(seed)
    scale = 10.0 ** rng.uniform(-3.0, 3.0, size=(n_voices, 1, 1))
    return (rng.standard_normal((n_voices, n_out, n)) * scale).astype(np.float32)


LAYOUTS = {
    "1 voice": _layout((0, 1, 1)),
    **{f"45 voices L={L}": _layout((0, 45, L)) for L in (1, 2, 4, 8, 16, 32)},
    "4096 voices L=2 (G=8)": _layout((0, 4096, 2)),
    "4097 tiles L=1 (G=16, last group empty)": _layout((0, 4097, 1)),
    "5000 voices L=1 (uneven last group)": _layout((0, 5000, 1)),
    "8192 voices L=1 (G=16)": _layout((0, 8192, 1)),
    "mixed widths": _layout((0, 33, 1), (33, 64, 32), (97, 40, 4), (137, 3, 2), (140, 100, 8), (240, 31, 16)),
    "no program / unset width": [{"v0": 0, "nv": 10, "tile_width": 0}, {"v0": 10, "nv": 20, "tile_width": 4},
                                 {"v0": 30, "nv": 40, "tile_width": 2, "slots": 3}],
}


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_model_is_within_the_depth_bound_of_the_exact_sum(name):
    layout = LAYOUTS[name]
    n_voices = max(g["v0"] + g["nv"] for g in layout)
    x = _random_voices(n_voices, 2, 32, seed=len(name))
    got = mix_model(x, layout).astype(np.float64)
    live = np.zeros(n_voices, dtype=bool)
    for g in layout:
        if g["tile_width"] and "slots" in g:
            live[g["v0"]:g["v0"] + g["nv"]] = True
    exact = x[live].astype(np.float64).sum(axis=0)
    bound, d = mix_bound(x[live], layout)
    err = np.abs(got - exact)
    assert (err <= bound).all(), f"{name}: err / bound = {float((err / bound).max()):.3g} (d = {d})"
    print(f"MIXMODEL {name}: d={d} G={k2_groups(sum((g['nv'] + g['tile_width'] - 1) // g['tile_width'] for g in layout if g['tile_width']))} "
          f"worst err/bound={float((err / bound).max()):.3g}")


def test_k2_group_counts():
    assert [k2_groups(n) for n in (1, 256, 257, 2048, 4096, 4097, 8192)] == [1, 1, 2, 8, 16, 16, 16]
    assert k2_per_group(4097, 16) == 288 and 15 * 288 >= 4097          # 4097 tiles: the 16th K2 group is empty
    assert k2_per_group(5000, 16) == 320 and 5000 - 15 * 320 == 200     # 5000 tiles: a short last group
    # 2048 tiles at L = 2: G = 8 groups of 256, 8 rows per lane, 2 per accumulator
    assert depth(_layout((0, 4096, 2))) == 1 + 2 + 2 + 31 + 8


# ---- sharpness -----------------------------------------------------------------------------------------------------------

# Four groups of widths 4, 1, 8 and 2: 150 + 300 + 50 + 350 = 850 tiles, so G = 4 groups of 224 rows (the last one short).
FAULT_LAYOUT = _layout((0, 600, 4), (600, 300, 1), (900, 400, 8), (1300, 700, 2))
N_SAMPLES = 96


def _designed(n_voices, n, salt=0):
    """Per-voice gains +-2^k, k in [-20, 20], rotating with the sample: voice v has exponent ((7 v + 13 t + salt) mod 41) - 20 at
    sample t, times a mantissa in [1, 2).  Every voice (so every tile) is among the largest terms at some sample, and the 41
    binades make every change of summation order visible in the rounding of the float32 sums."""
    v = np.arange(n_voices)[:, None]
    t = np.arange(n)[None, :]
    k = (7 * v + 13 * t + salt) % 41 - 20
    sign = np.where((v * 5 + salt) % 3 == 0, -1.0, 1.0)
    mant = 1.0 + ((v * 37 + t * 11 + salt) % 97) / 97.0
    return (sign * mant * np.exp2(k)).astype(np.float32)[:, None, :]


def _partial(x, layout=FAULT_LAYOUT, **kw):
    return np.concatenate(tile_rows(x, layout, **kw), axis=0)


def _differs(a, b):
    return bool((np.asarray(a).view(np.uint32) != np.asarray(b).view(np.uint32)).any())


@pytest.fixture(scope="module")
def designed():
    n_voices = 2000
    x = _designed(n_voices, N_SAMPLES)
    P = _partial(x)
    assert P.shape[0] == 850 and k2_groups(850) == 4
    good = mix_model(x, FAULT_LAYOUT)
    assert np.array_equal(good, k2(P))
    return x, P, good


def test_fault_every_tile_dropped_or_counted_twice(designed):
    x, P, good = designed
    for r in range(P.shape[0]):
        Q = P.copy()
        Q[r] = 0.0
        assert _differs(k2(Q), good), f"dropping tile {r} is invisible"
        Q[r] = P[r] + P[r]
        assert _differs(k2(Q), good), f"counting tile {r} twice is invisible"


def test_fault_two_k2_groups_exchanged(designed):
    """The final sum over the K2 groups in another order.  (Exchanging groups 0 and 1 alone is invisible in ANY float arithmetic:
    0 + s0 + s1 == 0 + s1 + s0.)"""
    x, P, good = designed
    G = k2_groups(P.shape[0])
    for a in range(G):
        for b in range(a + 1, G):
            if (a, b) == (0, 1):
                continue
            order = list(range(G))
            order[a], order[b] = order[b], order[a]
            assert _differs(k2(P, group_order=order), good), f"K2 groups {a} and {b} exchanged is invisible"


def test_fault_stale_row_from_the_previous_call(designed):
    x, P, good = designed
    prev = _partial(_designed(x.shape[0], N_SAMPLES, salt=17))
    for r in range(P.shape[0]):
        Q = P.copy()
        Q[r] = prev[r]
        assert _differs(k2(Q), good), f"a stale row {r} is invisible"


def test_fault_k2_group_count_off_by_one(designed):
    x, P, good = designed
    G = k2_groups(P.shape[0])
    for g in (G - 1, G + 1):
        assert _differs(k2(P, G=g), good), f"G = {g} instead of {G} is invisible"


def test_fault_butterfly_replaced_by_a_serial_sum(designed):
    """(At L = 2 the butterfly IS the serial sum; the L = 4 and L = 8 groups of the layout tell them apart.)"""
    x, P, good = designed

    def serial(t):
        s = t[:, 0]
        for j in range(1, t.shape[1]):
            s = s + t[:, j]
        return s

    for i, g in enumerate(FAULT_LAYOUT):
        if g["tile_width"] < 4:
            continue
        rows = tile_rows(x, FAULT_LAYOUT)
        rows[i] = tile_rows(x, [g], reduce_tile=serial)[0]
        assert _differs(k2(np.concatenate(rows)), good), f"a serial tile sum in group {i} (L = {g['tile_width']}) is invisible"
    assert np.array_equal(serial(np.ones((1, 2, 3), np.float32)), butterfly(np.ones((1, 2, 3), np.float32)))


def test_fault_tile_base_off_by_one_at_a_group_boundary(designed):
    x, P, good = designed
    rows = tile_rows(x, FAULT_LAYOUT)
    n = P.shape[0]
    for i in range(1, len(rows)):
        base, m = sum(len(r) for r in rows[:i]), len(rows[i])
        for shift in (-1, 1):
            Q = P.copy()
            Q[base:base + m] = 0.0                          # what group i should have written is not there (zeroed rows) ...
            lo, hi = max(0, base + shift), min(n, base + shift + m)
            Q[lo:hi] = rows[i][lo - base - shift:hi - base - shift]     # ... it went one tile early / late, over a neighbour's row
            assert _differs(k2(Q), good), f"tileBase of group {i} off by {shift} is invisible"
