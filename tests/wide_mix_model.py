"""A float32 model of the wide mix bus (nOut > 8): compact partial rows reduced per channel by K2w (DESIGN.md sections 3 and 4).

The engine's mix bus must equal this model BIT FOR BIT (NaN equal to NaN) for any layout of voice groups:

1. Mix channels.  Group g's mix channels C_g are the distinct channels in [0, nOut) of its program's roots (describe() reports the
   non-negative ones as "mix_channels"), ascending; a group without a program has none.
2. Compact partial rows.  The groups, in engine order, own consecutive runs of rows: group g owns nTiles_g * |C_g| rows, row
   rowBase_g + t * |C_g| + k being tile t's sum of channel C_g[k] — the xor butterfly of mix_model.tile_rows over the tile's voices.
3. Row lists.  R_c lists the rows of channel c: groups in engine order, tiles in order.
4. K2w.  Channel c is mix_model.k2 over the rows of R_c (G_c = min(16, ceil(|R_c| / 256)) groups, the same lane and group sums);
   a channel with no rows is +0.0.
"""
import numpy as np

from mix_model import group_active, k2, k2_groups, mix_bound, tile_rows

MAX_OUT_CHANNELS = 8        # above this nOut the compact path runs
MAX_WIDE_OUT_CHANNELS = 4096


def mix_channels(g, n_out):
    """C_g: the group's mix channels for nOut = n_out (empty for a group without a program)."""
    if not g.get("tile_width") or not group_active(g):
        return []
    return sorted({int(c) for c in g.get("mix_channels", []) if 0 <= int(c) < n_out})


def wide_rows(voice_out, layout, n_out, exchange=None):
    """(P [rows, n] float32, R: list of n_out row lists).  exchange = (group index, k0, k1): a planted fault that writes compact
    channels k0 and k1 of that group into each other's rows."""
    voice_out = np.asarray(voice_out, dtype=np.float32)
    tiles = tile_rows(voice_out, layout)               # per group [nTiles, nOut, n]
    rows, R, base = [], [[] for _ in range(n_out)], 0
    for gi, (g, tr) in enumerate(zip(layout, tiles)):
        ch = mix_channels(g, n_out)
        src = list(ch)
        if exchange is not None and exchange[0] == gi:
            src[exchange[1]], src[exchange[2]] = src[exchange[2]], src[exchange[1]]
        for t in range(tr.shape[0]):
            for k, c in enumerate(src):
                rows.append(tr[t, c])
        for k, c in enumerate(ch):
            R[c].extend(base + t * len(ch) + k for t in range(tr.shape[0]))
        base += tr.shape[0] * len(ch)
    n = voice_out.shape[2]
    P = np.stack(rows) if rows else np.zeros((0, n), np.float32)
    return P, R


def wide_k2(P, R, n, groups_of=None):
    """K2w over row lists R: [len(R), n].  groups_of(c, rows) -> G_c (default k2_groups(|R_c|))."""
    out = np.zeros((len(R), n), dtype=np.float32)
    for c, rc in enumerate(R):
        if not rc:
            continue
        G = None if groups_of is None else groups_of(c, rc)
        out[c] = k2(P[np.asarray(rc, dtype=np.int64)][:, None, :], G=G)[0]
    return out


def wide_mix_model(voice_out, layout, n_out, n=None):
    """The engine's wide mix bus for per-voice outputs voice_out [V, nOut, n] and the group layout (describe()["groups"])."""
    voice_out = np.asarray(voice_out, dtype=np.float32)
    if n is not None:
        voice_out = voice_out[:, :, :n]
    with np.errstate(over="ignore", invalid="ignore"):
        P, R = wide_rows(voice_out, layout, n_out)
        return wide_k2(P, R, voice_out.shape[2])


def engine_mix_model(voice_out, layout, n_out, n=None):
    """Whichever path the engine selects for n_out: mix_model.mix_model up to 8 channels, the compact model above."""
    from mix_model import mix_model
    if n_out <= MAX_OUT_CHANNELS:
        return mix_model(voice_out, layout, n_out, n)
    return wide_mix_model(np.asarray(voice_out)[:, :n_out], layout, n_out, n)


def channel_bound(voice_out, layout, n_out, c):
    """The depth bound of channel c: mix_model.mix_bound over the groups that write c (their voices only)."""
    lay = [g for g in layout if c in mix_channels(g, n_out)]
    if not lay:
        return None, 0
    x = np.concatenate([np.asarray(voice_out)[g["v0"]:g["v0"] + g["nv"], c:c + 1] for g in lay])
    b, d = mix_bound(x, lay)
    return b[0], d
