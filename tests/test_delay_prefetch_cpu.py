"""OP_DELAY's window one tile ahead (render_ops.inc): the predicate under which tile k issues tile k + 1's read window with cp.async
before tile k + 1 runs, restated and checked against the reference index arithmetic (Delays.h: readFrac = (float) (size + w) -
offset, left = (int) readFrac mod size, right = left + 1 mod size) for every write position at which a launch can start.

Under the predicate (ceil(offset) > numSamples + T, offset <= size - PER - 1, the tile-wide window's own conditions), for every tile
of the launch: the T + 1 positions the kernel prefetches for the tile hold exactly the left / right positions of the reference for
each of its samples, and none of them was written earlier in the same launch, so the values fetched one tile early are the values
the reference reads.  Ring sizes and offsets around T, 2T, 3T, the block size and size - T."""
import math

import numpy as np

GEOMS = [(4, 1), (4, 2), (8, 1), (8, 3), (4, 0), (8, 5)]     # (NITER, LOGL) with NITER > 1: the tile-wide window exists


def _exact(offset, size):
    """readFrac exact for every write position (delay_offset_exact's contract), checked directly in float32."""
    o = np.float32(offset)
    w = np.arange(size, dtype=np.int64)
    rf = (np.float32(size) + w.astype(np.float32)) - o
    return bool(np.all(rf.astype(np.float64) == (size + w).astype(np.float64) - float(o)))


def _predicate(offset, size, n_samples, T, per):
    cf = math.ceil(offset)
    return (size >= T and size <= 1 << 23 and cf > T and _exact(offset, size)
            and cf > n_samples + T and offset <= size - per - 1)


def _check(offset, size, n_samples, T, per):
    o = np.float32(offset)
    cf = math.ceil(float(o))
    frac = np.float32(cf) - o
    for w_start in range(size):
        written = set()
        for s0 in range(0, n_samples, T):
            cnt = min(T, n_samples - s0)
            w0 = (w_start + s0) % size
            if s0 > 0:       # the kernel's prefetch for this tile, issued by the tile before (w0 = w0_prev + T)
                rn = (w0 - cf) % size
                window = [(rn + t) % size for t in range(T + 1)]
                assert not written.intersection(window), (offset, size, n_samples, w_start, s0)
                for t in range(cnt):
                    w = (w0 + t) % size
                    rf = np.float32(np.float32(size + w) - o)
                    left = int(rf) % size
                    right = (left + 1) % size
                    assert window[t] == left and window[t + 1] == right, (offset, size, w_start, s0, t)
                    assert np.float32(rf - np.floor(rf)) == frac
            written.update((w0 + t) % size for t in range(cnt))


def test_prefetch_window_matches_reference_and_is_never_written_before():
    checked = 0
    for niter, logl in GEOMS:
        L = 1 << logl
        T, per = 32 * niter // L, 32 // L
        for n_samples in (T + 1, 3 * T - 5, 512):
            if n_samples > 4 * T and T < 64:
                continue
            for size in (3 * T + 7, n_samples + T + 40, 2 * (n_samples + T) + 1):
                cands = [T, 2 * T, 3 * T, n_samples, n_samples + T, n_samples + T + 0.5, n_samples + T + 1, size - T, size - T + 0.5,
                         size - per - 1, size - per - 0.5, size - per - 1.5]
                for off in cands:
                    if off <= 0 or off > size:
                        continue
                    if _predicate(off, size, n_samples, T, per):
                        _check(off, size, n_samples, T, per)
                        checked += 1
    assert checked > 20, checked

