"""A float32 model of the mix bus: the K1 tile epilogue (render_kernel.cu, `mixPartial`) followed by K2 (`mix_reduce_kernel`).

The mix is a fixed summation tree over the per-voice outputs, so the engine's mix bus must equal this model BIT FOR BIT (NaN equal to
NaN) for any layout of voice groups (DESIGN.md sections 4 and 5):

1. Partial rows.  The voice groups, in engine order (`describe()["groups"]`), own consecutive runs of rows: group i starts at
   tileBase_i = sum of ceil(nv_j / L_j) over the groups j < i (a group whose tile width is still 0 owns no rows).  Row
   tileBase_i + t is the sum over the L voices of tile t, formed by the xor butterfly over the voice bits of the lane id:
   x[j] <- x[j] + x[j + h] for h = L/2, L/4, ..., 1, starting from the voices' outputs (voices past nv count as +0.0).  A group
   without a program writes rows of zeros.  A fused `convolve -> root` group (L = 1) writes one row per voice, which is the same thing.
2. K2.  With nTiles rows, G = min(16, ceil(nTiles / 256)) groups of perGroup = roundup(ceil(nTiles / G), 32) rows each (the last
   ones may be short or empty).  In group g, lane j (0..31) sums rows tBegin + j, tBegin + j + 32, ... into four accumulators a0..a3
   (item k of the lane goes to a_(k mod 4) while four items remain, the rest to a0), combines (a0 + a1) + (a2 + a3), then the
   group sum is 0 + lane 0 + lane 1 + ... + lane 31.  With G = 1 that is the mix; otherwise the mix is 0 + s_0 + s_1 + ... + s_(G-1).
   Every sum is a float32 sum that starts from +0.0.
"""
import math

import numpy as np

MAX_GROUPS = 16      # kernels.h MIX_REDUCE_MAX_GROUPS
LANES = 32


def k2_groups(n_tiles):
    """The number of K2 tile groups for n_tiles partial rows (launch_mix_reduce)."""
    return max(1, min(MAX_GROUPS, (n_tiles + 255) // 256))


def k2_per_group(n_tiles, G):
    return ((n_tiles + G - 1) // G + LANES - 1) // LANES * LANES


def butterfly(x):
    """x: [tiles, L, ...] float32 -> [tiles, ...]: the xor butterfly of the tile epilogue, as lane 0 sees it."""
    while x.shape[1] > 1:
        h = x.shape[1] // 2
        x = x[:, :h] + x[:, h:]
    return x[:, 0]


def group_active(g):
    """describe() reports a program's shape ("slots", ...) only for a group that has one."""
    return g.get("active", "slots" in g)


def tile_rows(voice_out, layout, reduce_tile=butterfly):
    """The partial rows of every group, in engine order: a list of [ceil(nv / L), nOut, n] float32 arrays."""
    voice_out = np.asarray(voice_out, dtype=np.float32)
    rows = []
    for g in layout:
        L, v0, nv = int(g["tile_width"]), int(g["v0"]), int(g["nv"])
        if L == 0:
            rows.append(np.zeros((0,) + voice_out.shape[1:], dtype=np.float32))
            continue
        nt = (nv + L - 1) // L
        x = np.zeros((nt * L,) + voice_out.shape[1:], dtype=np.float32)
        if group_active(g):
            x[:nv] = voice_out[v0:v0 + nv]
        rows.append(reduce_tile(x.reshape((nt, L) + voice_out.shape[1:])))
    return rows


def lane_sum(items):
    """One K2 lane: four interleaved accumulators while four items remain, then a0; (a0 + a1) + (a2 + a3)."""
    z = np.zeros(items.shape[1:], dtype=np.float32)
    a = [z.copy(), z.copy(), z.copy(), z.copy()]
    k = 0
    while k + 3 < len(items):
        for i in range(4):
            a[i] = a[i] + items[k + i]
        k += 4
    while k < len(items):
        a[0] = a[0] + items[k]
        k += 1
    return (a[0] + a[1]) + (a[2] + a[3])


def k2(partial, G=None, group_order=None):
    """mix_reduce_kernel on partial [nTiles, nOut, n] float32.  group_order permutes the final sum over the groups (default: in order)."""
    partial = np.asarray(partial, dtype=np.float32)
    n_tiles = partial.shape[0]
    G = k2_groups(n_tiles) if G is None else G
    per = k2_per_group(n_tiles, G)
    sums = []
    for g in range(G):
        t0, t1 = g * per, min(n_tiles, g * per + per)
        v = np.zeros(partial.shape[1:], dtype=np.float32)
        for j in range(LANES):
            v = v + lane_sum(partial[t0 + j:t1:LANES] if t0 + j < t1 else partial[:0])
        sums.append(v)
    if G == 1:
        return sums[0]
    out = np.zeros(partial.shape[1:], dtype=np.float32)
    for g in (group_order if group_order is not None else range(G)):
        out = out + sums[g]
    return out


def mix_model(voice_out, layout, n_out=None, n=None):
    """The engine's mix bus for per-voice outputs voice_out [V, nOut, n] and the group layout (describe()["groups"])."""
    voice_out = np.asarray(voice_out, dtype=np.float32)
    if n_out is not None or n is not None:
        voice_out = voice_out[:, :n_out, :n]
    with np.errstate(over="ignore", invalid="ignore"):      # inf and NaN outputs propagate as on the GPU
        rows = tile_rows(voice_out, layout)
        partial = np.concatenate(rows, axis=0) if rows else np.zeros((0,) + voice_out.shape[1:], np.float32)
        if partial.shape[0] == 0:
            return np.zeros(voice_out.shape[1:], dtype=np.float32)
        return k2(partial)


def depth(layout):
    """The largest number of float additions between one voice output and the mix: log2 L of the butterfly, the longest K2
    accumulator chain, the two combines, the 31 lane additions and the G group additions (counted in full: an upper bound)."""
    n_tiles = sum((g["nv"] + g["tile_width"] - 1) // g["tile_width"] for g in layout if g["tile_width"])
    G = k2_groups(n_tiles)
    per = k2_per_group(n_tiles, G)
    items = math.ceil(per / LANES)                       # items of the fullest lane
    chain = items // 4 + items % 4                       # a0 gets one per round of four, then the remainder
    logl = max(int(math.log2(g["tile_width"])) for g in layout if g["tile_width"])
    return logl + chain + 2 + 31 + (G if G > 1 else 0)


def mix_bound(voice_out, layout):
    """|model - exact| <= gamma_d * sum |x| per output sample, gamma_d = d u / (1 - d u), u = 2^-24 (Higham, Accuracy and Stability
    of Numerical Algorithms, 2nd ed., Lemma 3.1 applied to the summation tree)."""
    d = depth(layout)
    u = 2.0 ** -24
    scale = np.abs(np.asarray(voice_out, dtype=np.float64)).sum(axis=0)
    return d * u / (1.0 - d * u) * scale, d


def assert_mix(got, want, what):
    """Bit-for-bit equality of a mix bus with the model, NaN equal to NaN."""
    got, want = np.asarray(got, dtype=np.float32), np.asarray(want, dtype=np.float32)
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        c, t = np.argwhere(~same)[0]
        raise AssertionError(f"{what}: mix bus differs from the model in {int((~same).sum())} samples; first out {c} sample {t}: "
                             f"gpu {got[c, t]!r} model {want[c, t]!r}")
