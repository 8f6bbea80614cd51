"""The exact reference of K3 (`convolve_chunk_tm_kernel`), its error contract, and a float32 model of its algorithm.

K3 computes the linear convolution of each channel's float32 input with its trimmed float32 impulse response, as one uniformly
partitioned frequency-domain delay line: partition P = 512, real FFT N = 1024, S = ceil(len(trim(h)) / 512) partitions.  For output
block b (samples [512 b, 512 b + 512) of the stream, on the grid that starts with the runtime's first sample):

    y_b = first half of IFFT(Y_b) + second half of IFFT(Y_{b-1}),    Y_b = sum_{i<S} H_i . X_{b-i},

with X_j = FFT([x_j, 0]) the spectrum of input block j and H_i = FFT([h_i, 0]) that of IR partition i.

`exact` evaluates the same convolution in float64 (relative error ~1e-15: the reference, not a model).  `bound` is the contract:

    max over block b of |gpu - exact|  <=  C * E_b,
    E_b = u * sqrt(S) * sum_{i<S} ||h_i||_2 * (||x_{b-i}||_2 + ||x_{b-i-1}||_2),     u = 2^-24.

Derivation of C.  Model every float rounding as an independent error of relative size at most u, i.e. standard deviation at most
u / sqrt(3) (uniform rounding error).  Write sigma for the per-sample standard deviation of the error in y_b.  The sources are:

1. Forward transform of x_j (10 radix-2 or 5 radix-4 + 1 radix-2 passes, float twiddles): each pass adds, per bin, an error of at
   most about 2u times the rms bin magnitude (one complex product with a rounded twiddle, one complex sum), so after log2 N = 10
   passes the rms bin error is at most sqrt(10 * 4 / 3) u rms(X_j) < 3.7 u rms(X_j).  By Parseval, rms(X_j) = ||x_j||_2
   (the FFT is unnormalised, N bins, ||X_j||_2^2 = N ||x_j||_2^2).
2. The IR spectra, computed in double and rounded once: rms error u / sqrt(3) rms(H_i) = 0.58 u ||h_i||_2 per bin.
3. The complex MAC over the S partitions: one complex product (2 roundings) and one complex sum per term.  Recursive summation of S
   terms adds rounding errors proportional to the running sums; with random signs their rms grows like sqrt(S) times the rms of one
   term: at most sqrt(S) * sqrt(3 * 2 / 3) u = 1.5 sqrt(S) u per unit of the terms' rms magnitude.
4. Inverse transform: as 1, 3.7 u relative to rms(Y_b); the 1/512 scale and the 0.5 factors of the split pass are exact.
5. Overlap-add of the two halves: one float sum, u / sqrt(3) relative.

An error delta in bin k of the product H_i . X_j reaches the time domain through the inverse transform, which divides by N: a bin
error of rms e spread over N bins gives a per-sample rms of e / sqrt(N).  Source 1 enters as |H_i| . delta X_j, so its time-domain
rms is 3.7 u ||h_i|| ||x_j|| / sqrt(N) (rms(H_i) = ||h_i||_2 by Parseval); the same holds for 2 (0.58), 3 (1.5 sqrt(S)) and 4
(3.7, since rms(Y_b) <= sum_i ||h_i|| (||x_{b-i}||)).  Summing the standard deviations over all partitions and both halves (the
triangle inequality, which also covers correlated errors), and bounding 1 <= sqrt(S):

    sigma <= (3.7 + 0.58 + 1.5 + 3.7 + 0.58) u sqrt(S) sum_i ||h_i|| (||x_{b-i}|| + ||x_{b-i-1}||) / sqrt(1024)
          = 10.1 / 32 * E_b = 0.32 E_b.

The largest of the 512 samples of a block lies within about sqrt(2 ln 1024) = 3.7 standard deviations, and a whole test matrix
(~10^8 samples) within about 6: the spread errors contribute at most 6 sigma = 1.9 E_b.

The estimate above spreads every error evenly over the block.  When the output is concentrated in a few samples (an impulse
through a one- or two-tap IR), the roundings fall on the peak sample itself.  The inverse transform's pass s holds the peak with
magnitude up to 2^s / 512 of its final value, so the sum of its roundings over the passes is at most about 2 u |y[n]|; the forward
transform and the product, bounded the same way, add as much each: 6 u |y[n]|.  By Cauchy-Schwarz,
|y[n]| <= sum_i ||h_i|| (||x_{b-i}|| + ||x_{b-i-1}||) = E_b / (u sqrt(S)), so this term adds at most 6 E_b (S = 1).  Together:
max |err| <= (1.9 + 6) E_b; C = 8.

`model(x, h)` is the float32 algorithm (uniform partitions, float32 real FFTs, float32 MAC) with optional planted faults.  Its
faultless worst ratio |err| / E_b on the matrix's signals is 1.5: one ulp of a two-tap IR's output for an impulse, a value just
above a power of two (one ulp is then 2u relative, and E_b = u |y|); on dense signals it stays below 0.5.
`test_convolve_exact_cpu.py` holds it at or below 0.25 C and shows that every planted fault exceeds C E_b by at least 4x.  K3's
own worst ratio on an H100 is in DESIGN.md section 4.
"""
from __future__ import annotations

import numpy as np
from scipy import fft as sfft
from scipy import signal as ssig

P = 512                  # partition
N = 1024                 # real FFT length
U = 2.0 ** -24           # unit roundoff of float32
C = 8.0                  # contract constant (module docstring)


# ---- impulse responses and inputs of the GPU matrix -------------------------------------------------------------------------
IR_KINDS = ("flat", "taps", "lcg")
INPUT_KINDS = ("noise", "impulses", "dc", "alternating", "quarter", "tone", "burst")
# IR lengths of the matrix (taps, trailing taps below 1e-6): around one and two partitions, config 4's 16384 and 65 partitions
LENGTHS = ((1, 0), (2, 0), (511, 0), (512, 0), (513, 0), (1023, 0), (1024, 0), (1025, 0), (1025, 300), (4097, 0), (4097, 700),
           (16383, 0), (16384, 0), (16385, 0), (32769, 0))
IMPULSE_OFFSETS = (0, 1, 255, 256, 511, 512, 513)
TAP_OFFSETS = (0, 1, 255, 256, 511)


def make_ir(kind, taps, seed=1, tail=0):
    """`taps` taps of one IR kind, then `tail` taps below 1e-6 in magnitude (trimmed away):
    flat: white noise with no decay; taps: one tap of gain +-1 per partition at offset 0, 1, 255, 256, 511 in turn;
    lcg: the decaying noise of `graphs.lcg_ir` (BASELINE config 4)."""
    rng = np.random.default_rng(seed)
    if kind == "flat":
        h = rng.uniform(-0.01, 0.01, taps).astype(np.float32)
        if taps:
            h[-1] = 0.01
    elif kind == "taps":
        h = np.zeros(taps, dtype=np.float32)
        for i in range((taps + P - 1) // P):
            h[min(i * P + TAP_OFFSETS[i % len(TAP_OFFSETS)], taps - 1)] = 1.0 if i % 2 == 0 else -1.0
    elif kind == "lcg":
        from elementary_b200 import graphs
        h = np.asarray(graphs.lcg_ir(taps, seed=seed), dtype=np.float32)
        if taps and abs(h[-1]) < 1e-6:
            h[-1] = 1e-5                     # keep S = ceil(taps / 512)
    else:
        raise ValueError(kind)
    if tail:
        h = np.concatenate([h, rng.uniform(-9.9e-7, 9.9e-7, tail).astype(np.float32)])
    return h


def make_input(kind, n, seed=0, lead=0):
    """`n` samples of one input kind; the first `lead` samples are silent (and the patterns count from the stream's first sample,
    so an impulse at offset k lands k samples into a partition when `lead` is a multiple of 512)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    if kind == "noise":
        x = rng.uniform(-0.5, 0.5, n)
    elif kind == "impulses":        # unit impulses at partition offsets 0, 1, 255, 256, 511, 512, 513, two partitions apart
        x = np.zeros(n)
        for k, off in enumerate(IMPULSE_OFFSETS):
            p = lead + 3 * P * k + off
            if p < n:
                x[p] = 1.0 if (k + seed) % 2 == 0 else -1.0
    elif kind == "dc":              # bin 0
        x = np.full(n, 0.5 + 0.01 * (seed % 7))
    elif kind == "alternating":     # bin 512 (Nyquist)
        x = np.where(t % 2 == 0, 1.0, -1.0)
    elif kind == "quarter":         # 1, 0, -1, 0: bin 256 (fs/4)
        x = np.array([1.0, 0.0, -1.0, 0.0])[t % 4]
    elif kind == "tone":            # bin 1 of the 1024-point transform
        x = np.cos(2.0 * np.pi * (t + 37 * seed) / N)
    elif kind == "burst":           # silence -> noise burst -> silence
        x = np.zeros(n)
        b0 = lead + 2 * P + 100 + 37 * (seed % 5)
        x[b0:b0 + 700] = rng.uniform(-1.0, 1.0, max(0, min(700, n - b0)))
    elif kind == "silence":
        x = np.zeros(n)
    else:
        raise ValueError(kind)
    x = x.astype(np.float32)
    x[:lead] = 0.0
    return x


# ---- the reference and the bound ------------------------------------------------------------------------------------------
def trim(h):
    """Drop trailing taps with fabs(h) < 1e-6f in float32, as the convolver does before partitioning."""
    h = np.asarray(h, dtype=np.float32).reshape(-1)
    keep = np.nonzero(np.abs(h) >= np.float32(0.000001))[0]
    return h[:keep[-1] + 1] if keep.size else h[:0]


def partitions(h):
    return (trim(h).size + P - 1) // P


def _rows(x, start):
    """float64 copy of x as [rows, n], samples before each row's start index set to zero (a restart from silence)."""
    x = np.asarray(x, dtype=np.float32)
    x2 = x.reshape(-1, x.shape[-1]).astype(np.float64)
    if start is not None:
        st = np.broadcast_to(np.asarray(start, dtype=np.int64), (x2.shape[0],))
        x2[np.arange(x2.shape[1])[None, :] < st[:, None]] = 0.0
    return x2, x.shape


def _groups(h, rows):
    """(trimmed float64 IR, row indices) per distinct IR: `h` is one IR for every row or a sequence of one IR per row."""
    if isinstance(h, np.ndarray) and h.ndim == 1 and h.dtype != object:
        return [(trim(h).astype(np.float64), np.arange(rows))]
    assert len(h) == rows, (len(h), rows)
    by = {}
    for r, hr in enumerate(h):
        by.setdefault(id(hr), (hr, []))[1].append(r)
    return [(trim(hr).astype(np.float64), np.asarray(rs)) for hr, rs in by.values()]


def exact(x, h, start=None, chunk=64):
    """Linear convolution of the float32 input rows with the trimmed float32 IR(s), in float64, truncated to the input length.
    `start`: per-row index before which the input counts as zero."""
    x2, shape = _rows(x, start)
    y = np.zeros_like(x2)
    for ht, rs in _groups(h, x2.shape[0]):
        if ht.size == 0:
            continue
        for k in range(0, rs.size, chunk):
            r = rs[k:k + chunk]
            y[r] = ssig.fftconvolve(x2[r], ht[None, :], axes=-1)[:, :x2.shape[1]]
    # where every input block an output block depends on is silent the convolution is exactly 0 (fftconvolve leaves ~1e-16)
    quiet = np.repeat(_silent_blocks(_pair_norms(x2), h, x2.shape[0]), P, axis=1)[:, :x2.shape[1]]
    y[quiet] = 0.0
    return y.reshape(shape)


def _block_norms(a):
    n = a.shape[-1]
    nb = (n + P - 1) // P
    a = np.pad(a, [(0, 0)] * (a.ndim - 1) + [(0, nb * P - n)])
    return np.sqrt(np.square(a.reshape(a.shape[:-1] + (nb, P))).sum(axis=-1))


def bound(x, h, start=None):
    """E_b of the module docstring, per row and 512-sample output block: [..., ceil(n / 512)] (multiply by C for the contract)."""
    x2, shape = _rows(x, start)
    t = _pair_norms(x2)
    E = np.zeros_like(t)
    for ht, rs in _groups(h, x2.shape[0]):
        if ht.size == 0:
            continue
        hb = _block_norms(ht)                                      # ||h_i||, i < S
        E[rs] = U * np.sqrt(hb.size) * ssig.fftconvolve(t[rs], hb[None, :], axes=-1)[:, :t.shape[1]]
    E = np.maximum(E, 0.0)                                         # fftconvolve of non-negative data: clear -1e-20 round-off
    E[_silent_blocks(t, h, x2.shape[0])] = 0.0
    return E.reshape(shape[:-1] + (t.shape[1],))


def _pair_norms(x2):
    """||x_j|| + ||x_{j-1}|| per row and block j."""
    xb = _block_norms(x2)
    t = xb.copy()
    t[:, 1:] += xb[:, :-1]
    return t


def _silent_blocks(t, h, rows):
    """Output blocks whose every input block (b - S ... b) is silent, from the pair norms t."""
    z = np.zeros(t.shape, dtype=bool)
    for ht, rs in _groups(h, rows):
        S = (ht.size + P - 1) // P
        if S == 0:
            z[rs] = True
            continue
        live = (t[rs] > 0).astype(np.int64)
        cnt = np.cumsum(live, axis=-1)
        prev = np.zeros_like(cnt)
        prev[:, S:] = cnt[:, :-S]
        z[rs] = (cnt - prev) == 0                                   # no live block among j in (b - S, b]
    return z


def block_error(got, want):
    """max |got - want| per row and 512-sample block."""
    d = np.abs(np.asarray(got, dtype=np.float64) - np.asarray(want, dtype=np.float64))
    n = d.shape[-1]
    nb = (n + P - 1) // P
    d = np.pad(d, [(0, 0)] * (d.ndim - 1) + [(0, nb * P - n)])
    return d.reshape(d.shape[:-1] + (nb, P)).max(axis=-1)


def ratio(got, want, E):
    """Worst block error over E, per row.  Where E is 0 every input block the output depends on is silent, so the output must be
    exactly 0.0 (inf otherwise; `want` there holds only the float64 transforms' ~1e-16 round-off)."""
    err = block_error(got, want)
    loud = block_error(got, np.zeros_like(got)) > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(E > 0, err / np.where(E > 0, E, 1.0), np.where(loud, np.inf, 0.0))
    return r.max(axis=-1)


# ---- a float32 model of K3's algorithm (CPU only: shows that the contract is sharp) -------------------------------------------
FAULTS = ("drop", "swap", "bin0", "bin256", "bin512", "pack", "overlap", "stale", "delay")


def model(x, h, fault=None, p=None):
    """K3's algorithm in float32 numpy, whole blocks from the stream's first sample.  `fault` plants one bug, in partition `p`
    (default: the middle one) where it concerns one partition:
    drop: partition p left out; swap: partitions p and p + 1 exchanged; bin0 / bin256 / bin512: that bin of H_p zeroed;
    pack: the real and imaginary halves of the packed bin 0 of H_p exchanged (H_p[0] <-> H_p[512]);
    overlap: the overlap taken from the block before the previous one; stale: partition p multiplies the ring slot one
    partition late (X_{b-p-1}); delay: the input delayed by one sample."""
    x = np.asarray(x, dtype=np.float32)
    shape = x.shape
    x = x.reshape(-1, shape[-1])
    ht = trim(h)
    S = (ht.size + P - 1) // P
    if S == 0:
        return np.zeros(shape, dtype=np.float32)
    p = S // 2 if p is None else p
    if fault == "swap":
        p = min(p, S - 2)
    hp = np.zeros(S * P)
    hp[:ht.size] = ht
    H = np.fft.rfft(hp.reshape(S, P), n=N, axis=-1).astype(np.complex64)     # spectra in double, rounded once
    if fault == "drop":
        H[p] = 0
    elif fault == "swap":
        H[[p, p + 1]] = H[[p + 1, p]]
    elif fault in ("bin0", "bin256", "bin512"):
        H[p, int(fault[3:])] = 0
    elif fault == "pack":
        H[p, 0], H[p, N // 2] = H[p, N // 2].real, H[p, 0].real
    if fault == "delay":
        x = np.concatenate([np.zeros((x.shape[0], 1), np.float32), x[:, :-1]], axis=1)
    n = x.shape[1]
    nb = (n + P - 1) // P
    xb = np.pad(x, ((0, 0), (0, nb * P - n))).reshape(x.shape[0], nb, P)
    X = sfft.rfft(xb, n=N, axis=-1)                                           # float32 in, complex64 out
    assert X.dtype == np.complex64
    lag = lambda a, k: np.concatenate([np.zeros_like(a[:, :k]), a[:, :nb - k]], axis=1) if k else a   # a_{b-k}
    acc = np.zeros_like(X)
    for i in list(range(1, S)) + [0]:                                         # older partitions first, then X_b . H_0
        k = i + 1 if (fault == "stale" and i == p) else i
        acc += H[i][None, None, :] * lag(X, min(k, nb))
    y = sfft.irfft(acc, n=N, axis=-1)
    assert y.dtype == np.float32
    out = y[:, :, :P] + lag(y[:, :, P:], 2 if fault == "overlap" else 1)
    return out.reshape(x.shape[0], nb * P)[:, :n].reshape(shape)
