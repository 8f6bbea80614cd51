"""OP_DELAY's hoisted read window (render_ops.inc, render_kernel.cu delay_offset_exact), proven on the CPU.

The fast path of a delay with a per-voice constant length forms, per element,
    readFrac = (float) (size + w) - offset,  readLeft = (int) readFrac,  frac = readFrac - floorf(readFrac)
and reduces readLeft / readLeft + 1 into [0, size).  When delay_offset_exact(offset, size) holds, the kernel instead sets up once
per tile  c = ceilf(offset), frac = c - offset  and reads at (w - c) mod size and the position after it.  These tests restate both
forms in numpy float32 and check, for every write position w in [0, size), that every (size, offset) the predicate admits gives the
same indices and the same frac bits — and that the predicate admits the SUBSYNTH32 delay (size 4800, length 3001.5)."""
import numpy as np
import pytest

K_EPS = np.float32(np.finfo(np.float32).eps)
MAX_FULL_SWEEP = 1 << 23      # every size the predicate can admit (2 size <= 2^24) is swept in full


def offset_exact(offset, size):
    """delay_offset_exact restated: integer ops on the float's bits."""
    b = int(np.float32(offset).view(np.uint32))
    e = (b >> 23) - 127
    m = b | 0x800000
    tz = (m & -m).bit_length() - 1            # __ffs(m) - 1
    f = max(0, 23 - e - tz)
    return f <= 23 and ((size - 1) >> (23 - f)) == 0


def per_element(offset, size):
    """The per-element form (render_ops.inc, OP_DELAY fast path) for every w in [0, size)."""
    w = np.arange(size, dtype=np.int64)
    read_frac = (size + w).astype(np.float32) - np.float32(offset)
    assert read_frac.dtype == np.float32
    left = read_frac.astype(np.int64)                   # (int) truncates; readFrac >= 0 here
    frac = read_frac - np.floor(read_frac)
    right = left + 1
    left = np.where(left >= size, left - size, left)
    right = np.where(right >= size, right - size, right)
    right = np.where(right >= size, right - size, right)
    return left, right, frac


def hoisted(offset, size):
    """The hoisted form: c and frac once, the read index moves by one per sample."""
    w = np.arange(size, dtype=np.int64)
    c = np.ceil(np.float32(offset))
    frac = np.float32(c - np.float32(offset))
    left = (w - int(c)) % size
    right = np.where(left + 1 == size, 0, left + 1)
    return left, right, np.full(size, frac, dtype=np.float32)


def offsets_for(size):
    """Integers, halves, offsets with many fractional bits, 0, kEps, size, and the values just inside the hazard bounds
    (hz + 1 and size - hz - 1 for the slice lengths PER = 1 .. 32 of the K1 geometries) and their float neighbours."""
    fs = np.float32(size)
    cands = [0.0, K_EPS, 1.0, 1.5, 2.0, 3001.5, fs, fs - 0.5, fs / 3, fs * 0.7071, np.float32(np.pi) * 1000]
    for hz in ((1, 2, 4, 8, 16, 32) if size <= 1 << 16 else (16, 32)):   # (fewer full sweeps of the large rings)
        cands += [hz + 1, size - hz - 1]
    cands += [size / 2, size // 2 + 0.25, size // 2 + 0.125, size // 3 + 1 / 1024, size - 1 + 1 / 8]
    out = set()
    for v in cands:
        v = np.float32(v)
        for x in (v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(0))):
            if np.float32(0) <= x <= fs:
                out.add(float(x))
    return sorted(out)


def sizes():
    s = set(range(1, 70)) | {4800, 3001, 3002, 48000, 96000, 100003}
    for k in range(1, 25):
        s |= {(1 << k) - 1, 1 << k, (1 << k) + 1}
    return sorted(s)


def check(size, offset):
    left0, right0, frac0 = per_element(offset, size)
    left1, right1, frac1 = hoisted(offset, size)
    return (np.array_equal(left0, left1) and np.array_equal(right0, right1)
            and np.array_equal(frac0.view(np.uint32), frac1.view(np.uint32)))


@pytest.mark.parametrize("size", sizes())
def test_predicate_never_admits_an_inexact_window(size):
    for offset in offsets_for(size):
        if offset <= K_EPS or not offset_exact(offset, size):
            continue        # the kernel passes the input through (<= kEps) or keeps the per-element form
        assert size <= MAX_FULL_SWEEP
        assert check(size, offset), (size, offset)


def test_predicate_on_random_offsets():
    rng = np.random.default_rng(1)
    admitted = 0
    for size in (64, 65, 100, 4800, 4095, 4096, 4097, 65536, 1 << 20):
        fs = np.float32(size)
        offs = np.concatenate([rng.uniform(1.0, size, 40).astype(np.float32),                      # many fractional bits
                               (np.floor(rng.uniform(1.0, size, 20)) + rng.integers(0, 16, 20) / 16).astype(np.float32)])
        for offset in offs:
            if not (1.0 <= offset <= fs) or not offset_exact(float(offset), size):
                continue
            admitted += 1
            assert check(size, float(offset)), (size, float(offset))
    assert admitted > 50


def test_predicate_admits_subsynth32_and_common_lengths():
    assert offset_exact(3001.5, 4800)
    assert check(4800, 3001.5)
    for size in (512, 4800, 48000, 1 << 20, 1 << 21):
        for offset in (17.0, 100.0, 255.5, size // 2 + 0.25):
            assert offset_exact(offset, size), (size, offset)
    assert offset_exact(4000.0, 1 << 23) and offset_exact(4000.5, 1 << 22) and not offset_exact(4000.25, 1 << 22)


def test_predicate_rejects_where_the_float_form_rounds():
    """The predicate guards real cases: past its bound the per-element float computation and the hoisted one part ways."""
    differ = 0
    for size, offset in (((1 << 23) + 1, 1000.5), ((1 << 22) + 1, 3.25), ((1 << 21) + 3, 7.125), (1 << 24, 5.0),
                         (4800, float(np.float32(1234.5678))), (1 << 16, float(np.float32(np.pi) * 1000))):
        assert not offset_exact(offset, size), (size, offset)
        if not check(size, offset):
            differ += 1
    assert differ >= 4


def test_predicate_bound_is_tight_in_size():
    # with f fractional bits the largest admitted size is 2^(23 - f): one more is rejected
    for f in range(0, 12):
        offset = 2.0 + 2.0 ** -f if f else 3.0
        top = 1 << (23 - f)
        assert offset_exact(offset, top) and not offset_exact(offset, top + 1), f
