// convolve_kernel.cu — K3: uniformly partitioned FFT convolution, hand-written shared-memory FFT + complex MAC.
// No cuFFT, no tensor cores: this is a streaming frequency-domain delay line, bound by the HBM reads of the input
// spectra (see convolve.h for the algorithmic bytes).
//
// Persistent CTAs (2 per SM; a TMA producer warp, 4 MAC warps, 4 transform warps) walk the channel pairs; a pair shares one
// pass over the IR spectra so that every IR spectrum value fetched from L2 is reused.  Per pair and call:
//   1. append the new samples to the partition's input buffer, zero-pad to 1024 (FFTConvolver.cpp:157-164)
//   2. real FFT 1024 = complex Stockham radix-4 FFT 512 in shared memory + split post-pass  (replaces OouraFFT::fft,
//      AudioFFT.cpp:132-155; float arithmetic instead of the reference's double)
//   3. if the input buffer was empty: Ypre = sum_{i>=1} H_i * X_{cur+i}   (FFTConvolver.cpp:168-177,
//      ComplexMultiplyAccumulate Utilities.cpp:66-117)
//   4. Y = Ypre + X_cur * H_0 (:178-179); inverse real FFT (:182); out = y[fill..] + overlap[fill..] (:185)
//   5. when the partition is complete: overlap = y[512..1024) (:194), the host rotates `cur` (:200)
#include "convolve.h"
#include <cstdio>

namespace eb {

namespace {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cconj(float2 a) { return make_float2(a.x, -a.y); }

// ---- TMA (1-D bulk async copy) + mbarrier primitives: the frequency-domain delay line is streamed HBM -> shared memory
// by cp.async.bulk (SASS: UBLKCP) through a multi-stage ring guarded by full/empty mbarriers and fed by a dedicated
// producer warp, so the MAC loop never waits on a per-thread global load and the stream runs through the FFT phases.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug must end in a trap (the launch fails, the tests say so), never in a hung GPU
__device__ __forceinline__ void mbar_wait_b(uint64_t* bar, uint32_t parity) {
    for (uint32_t spins = 0; !mbar_try(bar, parity); ++spins)
        if (spins > (1u << 24)) __trap();
}

constexpr int CH = CONV_CH_PER_CTA;
constexpr uint32_t ROW_BYTES = CONV_PACKED_BINS * sizeof(float2);
constexpr int NB = CONV_PACKED_BINS;   // 512: bin 0 carries (Re X[0], Re X[512]) — both are purely real
constexpr int N2 = 512;   // complex FFT length

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// =========================================================================================================
// K3, transform/MAC split ("TM"): the same persistent CTA, but the 8 worker warps are two groups with different jobs that
// overlap in time instead of alternating:
//   * T group (4 warps): forward FFT of pair n (-> Xbuf[n&1], and the delay-line slot `cur`), then the inverse FFT, overlap-add
//     and output of pair n-1 (from Ybuf[(n-1)&1]);
//   * M group (4 warps): complex MAC of pair n over the ring the producer warp fills, then Y = acc + X·H_0 -> Ybuf[n&1].
// Xbuf/Ybuf are double buffered and handed over with mbarriers (xfull/xempty, yfull/yempty), so while M streams pair n from HBM,
// T transforms pair n+1 and pair n-1: the HBM stream of a CTA only ever waits for data, not for transforms.
constexpr int TM_GROUP = 128;                       // threads per worker group
constexpr int TM_THREADS = 2 * TM_GROUP + 32;       // T + M + producer warp
constexpr int TM_STAGES = 5;                        // 5 x 12 KB + 44 KB = 104 KB per CTA, two CTAs per SM still fit in 228 KB
constexpr int TM_CTAS_PER_SM = 2;
// The per-channel-IR form streams CH input rows and up to CH IR rows per stage (16 KB): 4 stages x 16 KB + 44 KB = 108 KB per CTA,
// two CTAs per SM still fit in 228 KB (5 stages would not).
constexpr int PC_STAGES = 4;
static_assert(CH == 2, "the unit table holds channel pairs");

template <bool PER_CH> struct ConvForm {
    static constexpr int STAGES = PER_CH ? PC_STAGES : TM_STAGES;
    static constexpr int HROWS = PER_CH ? CH : 1;     // IR rows per ring stage
    static constexpr size_t smem() {
        return (size_t) STAGES * (CH + HROWS) * ROW_BYTES + (size_t) 5 * CH * ROW_BYTES + ROW_BYTES + (2 * STAGES + 8) * sizeof(uint64_t);
    }
};

__device__ __forceinline__ void tgroup_sync() { asm volatile("bar.sync 2, %0;" ::"n"(TM_GROUP) : "memory"); }

// Complex FFT 512 (Stockham autosort, out of place between two shared-memory buffers), 128 threads: four radix-4 stages — one
// butterfly per thread and channel, sub-transform length p = 1, 4, 16, 64 — and a final radix-2 stage (p = 256, two butterflies per
// thread): 5 group barriers instead of the 9 of a pure radix-2 transform.  tw[m] = exp(-2 pi i m / 1024), m < 512.  Result in `b`.
template <bool INVERSE>
__device__ __forceinline__ void fft512_t(float2 (*a)[N2], float2 (*b)[N2], const float2* tw, int t) {
    float2 (*src)[N2] = a;
    float2 (*dst)[N2] = b;
#pragma unroll 1
    for (int p = 1; p < N2 / 2; p <<= 2) {
        const int k = t & (p - 1);
        const int m = k * (N2 / 2 / p);                  // exp(-2 pi i k / (4 p)) = tw[k * 256 / p]
        float2 w1 = tw[m], w2 = tw[2 * m];
        float2 w3 = (3 * m < N2) ? tw[3 * m] : tw[3 * m - N2];
        if (3 * m >= N2) { w3.x = -w3.x; w3.y = -w3.y; }   // exp(-i (pi + x)) = -exp(-i x)
        if (INVERSE) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
        const int j0 = ((t - k) << 2) + k;
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const float2 x0 = src[c][t];
            const float2 a1 = cmul(w1, src[c][t + N2 / 4]);
            const float2 a2 = cmul(w2, src[c][t + N2 / 2]);
            const float2 a3 = cmul(w3, src[c][t + 3 * N2 / 4]);
            const float2 b0 = cadd(x0, a2), b1 = csub(x0, a2), b2 = cadd(a1, a3);
            const float2 d = csub(a1, a3);
            const float2 b3 = INVERSE ? make_float2(-d.y, d.x) : make_float2(d.y, -d.x);   // (a1 - a3) * (+-i)
            dst[c][j0] = cadd(b0, b2);
            dst[c][j0 + p] = cadd(b1, b3);
            dst[c][j0 + 2 * p] = csub(b0, b2);
            dst[c][j0 + 3 * p] = csub(b1, b3);
        }
        tgroup_sync();
        float2 (*tmp)[N2] = src; src = dst; dst = tmp;
    }
    {
        constexpr int ns = N2 / 2;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int bi = t + h * TM_GROUP;                 // butterfly index 0..255
            const int k = bi & (ns - 1);
            float2 w = tw[k * (N2 / ns)];
            if (INVERSE) w.y = -w.y;
            const int j0 = ((bi - k) << 1) + k;
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                const float2 u = src[c][bi];
                const float2 v = cmul(w, src[c][bi + N2 / 2]);
                dst[c][j0] = cadd(u, v);
                dst[c][j0 + ns] = csub(u, v);
            }
        }
        tgroup_sync();
    }
}

// Relayout of a grown input spectra ring (convolve.h convolver_relayout): one CTA of 128 threads per (channel, new slot).
__global__ void convolve_ring_relayout_kernel(float2* __restrict__ dst, const float2* __restrict__ src, int oldR, int newR, int cur) {
    const int ch = blockIdx.x, i = blockIdx.y;
    float2* d = dst + ((size_t) ch * newR + i) * NB;
    if (i < oldR) {
        const int s = (cur + i) % oldR;
        const float2* p = src + ((size_t) ch * oldR + s) * NB;
        for (int k = threadIdx.x; k < NB; k += blockDim.x) d[k] = p[k];
    } else {
        for (int k = threadIdx.x; k < NB; k += blockDim.x) d[k] = make_float2(0.0f, 0.0f);
    }
}

} // namespace

// PER_CH = false: every channel convolves with H (S partitions); units are the channel pairs (2u, 2u + 1).
// PER_CH = true: channel c convolves with chan[c].H (chan[c].S partitions); unit u is the pair units[u] = {c0, c1 (-1: none), max S,
// same IR} and its ring stages carry one IR row (same IR) or two.  A channel past its own S contributes nothing (predicated MAC), so
// a channel's output is bit-identical to the shared form on the same IR.  In both forms the ring has R slots (R >= every S).
template <bool PER_CH>
__global__ void __launch_bounds__(TM_THREADS, TM_CTAS_PER_SM) convolve_chunk_tm_kernel(
    const float* __restrict__ in, int inStride, float* __restrict__ out, int stride, int offset, int n, int fill, int cur, int S, int R, int nv,
    const float2* __restrict__ H, const ConvChannel* __restrict__ chan, const int4* __restrict__ units,
    float2* __restrict__ fdl, float2* __restrict__ ypre,
    float* __restrict__ overlap, float* __restrict__ inbuf, const float2* __restrict__ twg, const ConvEpilogue epi) {
    constexpr int STAGES = ConvForm<PER_CH>::STAGES, HROWS = ConvForm<PER_CH>::HROWS;
    extern __shared__ __align__(128) unsigned char smemRaw[];
    float2 (*stX)[CH][N2] = reinterpret_cast<float2 (*)[CH][N2]>(smemRaw);                                        // [STAGES][CH][512]
    float2 (*stH)[HROWS][N2] = reinterpret_cast<float2 (*)[HROWS][N2]>(smemRaw + (size_t) STAGES * CH * ROW_BYTES);   // [STAGES][HROWS][512]
    float2 (*Xb)[CH][N2] = reinterpret_cast<float2 (*)[CH][N2]>(smemRaw + (size_t) STAGES * (CH + HROWS) * ROW_BYTES);   // [2][CH][512]
    float2 (*Yb)[CH][N2] = Xb + 2;                                                                                 // [2][CH][512]
    float2 (*Sc)[N2] = reinterpret_cast<float2 (*)[N2]>(Yb + 2);                                                   // [CH][512] transform scratch
    float2* tw = reinterpret_cast<float2*>(Sc + CH);                                                               // [512]
    uint64_t* full = reinterpret_cast<uint64_t*>(tw + N2);        // [STAGES]
    uint64_t* empty = full + STAGES;                              // [STAGES]
    uint64_t* xfull = empty + STAGES;                             // [2] T -> M: Xbuf ready
    uint64_t* xempty = xfull + 2;                                 // [2] M -> T: Xbuf consumed
    uint64_t* yfull = xempty + 2;                                 // [2] M -> T: Ybuf ready
    uint64_t* yempty = yfull + 2;                                 // [2] T -> M: Ybuf consumed

    const int tid = threadIdx.x;
    const int numUnits = (nv + CH - 1) / CH;
    // channels of unit u: ch[c] is a valid channel to address (a missing second channel aliases the first), ok[c] whether it is real
    auto unitChannels = [&](int u, int (&ch)[CH], bool (&ok)[CH]) {
        if (PER_CH) {
            const int4 ud = units[u];
            ch[0] = ud.x; ok[0] = true;
            ch[1] = ud.y >= 0 ? ud.y : ud.x; ok[1] = ud.y >= 0;
        } else {
#pragma unroll
            for (int c = 0; c < CH; ++c) { ch[c] = min(u * CH + c, nv - 1); ok[c] = u * CH + c < nv; }
        }
    };
    auto unitS = [&](int u) { return PER_CH ? units[u].z : S; };
    // The producer thread initialises the barriers itself and fills the first ring stages BEFORE the CTA-wide barrier: the delay line
    // is on its way from HBM while the other warps still fetch the twiddle table (cold after an L2 flush).  Its first STAGES
    // stages need no `empty` wait (fresh barriers pass the parity-1 wait), so nothing it touches depends on the other warps yet.
    const bool producerThread = (tid == 2 * TM_GROUP);
    uint32_t pit = 0;                    // producer: stages issued so far
    int pu = blockIdx.x, pi = 1;         // producer: next (unit, partition) to issue
    int puS = 0;                         // producer: partitions of unit pu
    auto skipEmpty = [&]() {             // units whose channels have at most one partition stream nothing
        while (pu < numUnits && (puS = unitS(pu)) <= 1) pu += gridDim.x;
    };
    auto produceOne = [&]() {
        const int stg = pit % STAGES;
        mbar_wait_b(&empty[stg], ((pit / STAGES) & 1) ^ 1);
        int slotIdx = cur + pi;
        if (slotIdx >= R) slotIdx -= R;
        int ch[CH]; bool ok[CH];
        unitChannels(pu, ch, ok);
        if (PER_CH) {
            // one IR row when the unit's channels share the IR, else one per channel; a channel past its own S loads its partner's
            // row (the partner has > pi partitions, since the unit does) and the MAC ignores it
            const int nH = units[pu].w ? 1 : CH;
            mbar_expect_tx(&full[stg], (CH + nH) * ROW_BYTES);
#pragma unroll
            for (int c = 0; c < CH; ++c)
                tma_load_1d(&stX[stg][c][0], fdl + ((size_t) ch[c] * R + slotIdx) * NB, ROW_BYTES, &full[stg]);
            for (int c = 0; c < nH; ++c) {
                const ConvChannel d = chan[ch[c]], e = chan[ch[c ^ 1]];
                const float2* h = (pi < d.S) ? d.H : e.H;
                tma_load_1d(&stH[stg][c][0], h + (size_t) pi * NB, ROW_BYTES, &full[stg]);
            }
        } else {
            mbar_expect_tx(&full[stg], (CH + 1) * ROW_BYTES);
#pragma unroll
            for (int c = 0; c < CH; ++c)
                tma_load_1d(&stX[stg][c][0], fdl + ((size_t) ch[c] * R + slotIdx) * NB, ROW_BYTES, &full[stg]);
            tma_load_1d(&stH[stg][0][0], H + (size_t) pi * NB, ROW_BYTES, &full[stg]);
        }
        ++pit;
        if (++pi >= puS) { pi = 1; pu += gridDim.x; skipEmpty(); }
    };
    const bool streams = fill == 0 && (PER_CH || S > 1);
    if (producerThread) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TM_GROUP / 32); }
        for (int i = 0; i < 2; ++i) { mbar_init(&xfull[i], 1); mbar_init(&xempty[i], TM_GROUP / 32); mbar_init(&yfull[i], TM_GROUP / 32); mbar_init(&yempty[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async();
        if (streams) {
            skipEmpty();
            for (int k = 0; k < STAGES && pu < numUnits; ++k) produceOne();
        }
    }
    for (int i = tid; i < N2; i += TM_THREADS) tw[i] = twg[i];
    __syncthreads();

    if (tid >= 2 * TM_GROUP) {
        // ---------------- producer warp ----------------
        if (producerThread && streams) {
            while (pu < numUnits) produceOne();
        }
        return;
    }

    if (tid >= TM_GROUP) {
        // ---------------- M group: MAC over the ring, then the combine with the new block's spectrum ----------------
        const int t = tid - TM_GROUP;
        uint32_t it = 0;
        int nloc = 0;
        for (int u = blockIdx.x; u < numUnits; u += gridDim.x, ++nloc) {
            const int b = nloc & 1;
            int ch[CH]; bool ok[CH];
            unitChannels(u, ch, ok);
            int cS[CH];                                                    // partitions of each channel's IR
            const float2* cH[CH];
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                if (PER_CH) { const ConvChannel d = chan[ch[c]]; cS[c] = ok[c] ? d.S : 0; cH[c] = d.H; }
                else { cS[c] = S; cH[c] = H; }
            }
            const int uS = unitS(u);
            const bool sameIr = !PER_CH || units[u].w != 0;
            float2 acc[4][CH];
            if (fill == 0) {
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int c = 0; c < CH; ++c) acc[q][c] = make_float2(0.0f, 0.0f);
                for (int i = 1; i < uS; ++i, ++it) {
                    const int stg = it % STAGES;
                    mbar_wait_b(&full[stg], (it / STAGES) & 1);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int k = t + q * TM_GROUP;
                        const float2 h0q = stH[stg][0][k];
#pragma unroll
                        for (int c = 0; c < CH; ++c) {
                            const float2 hq = (PER_CH && c > 0 && !sameIr) ? stH[stg][HROWS - 1][k] : h0q;
                            const float2 x = stX[stg][c][k];
                            if (!PER_CH || i < cS[c])
                                acc[q][c] = (k == 0) ? make_float2(acc[q][c].x + hq.x * x.x, acc[q][c].y + hq.y * x.y) : cadd(acc[q][c], cmul(hq, x));
                        }
                    }
                    __syncwarp();
                    if ((t & 31) == 0) mbar_arrive(&empty[stg]);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int c = 0; c < CH; ++c) if (ok[c]) ypre[(size_t) ch[c] * NB + t + q * TM_GROUP] = acc[q][c];
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int c = 0; c < CH; ++c) acc[q][c] = ypre[(size_t) ch[c] * NB + t + q * TM_GROUP];
            }
            mbar_wait_b(&xfull[b], (nloc >> 1) & 1);                       // the forward transform of this pair is in Xbuf[b]
            mbar_wait_b(&yempty[b], ((nloc >> 1) & 1) ^ 1);                // the inverse transform of pair n-2 has left Ybuf[b]
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int k = t + q * TM_GROUP;
                // the newest partition against each channel's own H_0 (an IR trimmed to nothing: zero)
                float2 h0s[CH];
#pragma unroll
                for (int c = 0; c < CH; ++c) {
                    if (!PER_CH) h0s[c] = (c == 0) ? __ldg(H + k) : h0s[0];
                    else if (cS[c] == 0) h0s[c] = make_float2(0.0f, 0.0f);
                    else if (c > 0 && sameIr) h0s[c] = h0s[0];
                    else h0s[c] = __ldg(cH[c] + k);
                }
#pragma unroll
                for (int c = 0; c < CH; ++c) {
                    const float2 h0 = h0s[c];
                    const float2 x = Xb[b][c][k];
                    Yb[b][c][k] = (k == 0) ? make_float2(acc[q][c].x + x.x * h0.x, acc[q][c].y + x.y * h0.y) : cadd(acc[q][c], cmul(x, h0));
                }
            }
            __syncwarp();
            if ((t & 31) == 0) { mbar_arrive(&yfull[b]); mbar_arrive(&xempty[b]); }
        }
        return;
    }

    // ---------------- T group: forward transform of pair n, inverse transform + output of pair n-1 ----------------
    const int t = tid;
    const bool wholeBlock = (fill == 0) && (n == CONV_BLOCK) && (((inStride | offset) & 1) == 0);
    const float scale = 1.0f / 512.0f;

    auto forward = [&](int u, int nloc) {
        const int b = nloc & 1;
        int chs[CH]; bool oks[CH];
        unitChannels(u, chs, oks);
        if (t == 0) mbar_wait_b(&xempty[b], ((nloc >> 1) & 1) ^ 1);       // M is done with what Xbuf[b] held (pair n-2)
        tgroup_sync();
        if (wholeBlock) {
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                const int ch = chs[c];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int k = t + h * TM_GROUP;
                    float2 z = make_float2(0.0f, 0.0f);
                    if (oks[c]) z = __ldg(reinterpret_cast<const float2*>(in + (size_t) ch * inStride + offset) + k);
                    Sc[c][k] = z;
                    Sc[c][k + 256] = make_float2(0.0f, 0.0f);
                }
            }
        } else {
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                const int ch = chs[c];
                if (oks[c]) {
                    float* ib = inbuf + (size_t) ch * CONV_BLOCK;
                    for (int i = t; i < n; i += TM_GROUP) ib[fill + i] = in[(size_t) ch * inStride + offset + i];
                }
            }
            tgroup_sync();
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                const int ch = chs[c];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int k = t + h * TM_GROUP;
                    float2 z = make_float2(0.0f, 0.0f);
                    if (oks[c]) z = reinterpret_cast<const float2*>(inbuf + (size_t) ch * CONV_BLOCK)[k];
                    Sc[c][k] = z;
                    Sc[c][k + 256] = make_float2(0.0f, 0.0f);
                }
            }
        }
        tgroup_sync();
        fft512_t<false>(Sc, Xb[b], tw, t);                                 // Z = FFT512(z) in Xbuf[b]
        // split in place: bins k and 512-k are produced together from Z[k], Z[512-k]; bin 512 is packed into bin 0
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const bool ok = oks[c];
            float2* slot = fdl + ((size_t) chs[c] * R + cur) * NB;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int k = t + h * TM_GROUP;                            // 0..255
                if (k == 0) {
                    const float2 z0 = Xb[b][c][0], zh = Xb[b][c][256];
                    // k = 0: E0 = Re z0, O0 = Im z0 -> packed (E0 + O0, E0 - O0);  k = 256: X = conj(z[256]) (tw[256] = -i)
                    const float2 x0 = make_float2(z0.x + z0.y, z0.x - z0.y);
                    const float2 eh = make_float2(zh.x, 0.0f), dh = make_float2(0.0f, 2.0f * zh.y);
                    const float2 oh = make_float2(0.5f * dh.y, -0.5f * dh.x);
                    const float2 xh = cadd(eh, cmul(tw[256], oh));
                    Xb[b][c][0] = x0; Xb[b][c][256] = xh;
                    if (ok) { slot[0] = x0; slot[256] = xh; }
                } else {
                    const int kn = N2 - k;
                    const float2 zk = Xb[b][c][k], zq = Xb[b][c][kn];
                    const float2 zn = cconj(zq);
                    const float2 e = make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y + zn.y));
                    const float2 d = csub(zk, zn);
                    const float2 o = make_float2(0.5f * d.y, -0.5f * d.x);
                    const float2 xk = cadd(e, cmul(tw[k], o));
                    // partner bin: Z[kn], conj(Z[k])
                    const float2 zn2 = cconj(zk);
                    const float2 e2 = make_float2(0.5f * (zq.x + zn2.x), 0.5f * (zq.y + zn2.y));
                    const float2 d2 = csub(zq, zn2);
                    const float2 o2 = make_float2(0.5f * d2.y, -0.5f * d2.x);
                    const float2 xn = cadd(e2, cmul(tw[kn], o2));
                    Xb[b][c][k] = xk; Xb[b][c][kn] = xn;
                    if (ok) { slot[k] = xk; slot[kn] = xn; }
                }
            }
        }
        tgroup_sync();
        if (t == 0) mbar_arrive(&xfull[b]);
    };

    auto inverse = [&](int u, int nloc) {
        const int b = nloc & 1;
        int chs[CH]; bool oks[CH];
        unitChannels(u, chs, oks);
        // overlap of the previous partition for this chunk: fetched before waiting, used after the inverse FFT
        float ovv[CH][4];
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const float* ov = overlap + (size_t) chs[c] * CONV_BLOCK;
#pragma unroll
            for (int q = 0; q < 4; ++q) { const int i = t + q * TM_GROUP; ovv[c][q] = (i < n) ? ov[fill + i] : 0.0f; }
        }
        if (t == 0) mbar_wait_b(&yfull[b], (nloc >> 1) & 1);
        tgroup_sync();
        // inverse split in place on Ybuf[b]: Zi[k] = E[k] + i*O[k] from Y[k], conj(Y[512-k])
#pragma unroll
        for (int c = 0; c < CH; ++c) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int k = t + h * TM_GROUP;
                if (k == 0) {
                    const float2 y0 = Yb[b][c][0], yh = Yb[b][c][256];
                    Yb[b][c][0] = make_float2(0.5f * (y0.x + y0.y), 0.5f * (y0.x - y0.y));      // packed (Y0, Y512)
                    const float2 yn = cconj(yh);
                    const float2 e = make_float2(0.5f * (yh.x + yn.x), 0.5f * (yh.y + yn.y));
                    const float2 d = make_float2(0.5f * (yh.x - yn.x), 0.5f * (yh.y - yn.y));
                    const float2 o = cmul(d, cconj(tw[256]));
                    Yb[b][c][256] = make_float2(e.x - o.y, e.y + o.x);
                } else {
                    const int kn = N2 - k;
                    const float2 yk = Yb[b][c][k], yq = Yb[b][c][kn];
                    const float2 yn = cconj(yq);
                    const float2 e = make_float2(0.5f * (yk.x + yn.x), 0.5f * (yk.y + yn.y));
                    const float2 d = make_float2(0.5f * (yk.x - yn.x), 0.5f * (yk.y - yn.y));
                    const float2 o = cmul(d, cconj(tw[k]));
                    const float2 yn2 = cconj(yk);
                    const float2 e2 = make_float2(0.5f * (yq.x + yn2.x), 0.5f * (yq.y + yn2.y));
                    const float2 d2 = make_float2(0.5f * (yq.x - yn2.x), 0.5f * (yq.y - yn2.y));
                    const float2 o2 = cmul(d2, cconj(tw[kn]));
                    Yb[b][c][k] = make_float2(e.x - o.y, e.y + o.x);
                    Yb[b][c][kn] = make_float2(e2.x - o2.y, e2.y + o2.x);
                }
            }
        }
        tgroup_sync();
        fft512_t<true>(Yb[b], Sc, tw, t);                                   // result in Sc: z[j] * 512
        if (t == 0) mbar_arrive(&yempty[b]);                                // Ybuf[b] may be overwritten (pair n+2)
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const int ch = chs[c];
            if (!oks[c]) continue;
            const float* y = reinterpret_cast<const float*>(&Sc[c][0]);
            if (!epi.active) {
                float* o = out + (size_t) ch * stride + offset;
#pragma unroll
                for (int q = 0; q < 4; ++q) { const int i = t + q * TM_GROUP; if (i < n) o[i] = y[fill + i] * scale + ovv[c][q]; }
            } else {
                // root + mix epilogue (ConvEpilogue): the same arithmetic as K1's OP_ROOT, sample index = position in the block
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int i = t + q * TM_GROUP;
                    if (i >= n) continue;
                    const float v = y[fill + i] * scale + ovv[c][q];
                    float r = 0.0f;
                    if (epi.running) {
                        if (epi.gain0 == epi.target) r = v * epi.target;
                        else {
                            const float gr = epi.gain0 + epi.step * (float) (offset + i);
                            r = v * ((gr < 0.0f) ? 0.0f : ((1.0f < gr) ? 1.0f : gr));
                        }
                        r = 0.0f + r;                                   // K1 accumulates into a zeroed output row
                    }
                    for (int oc = 0; oc < epi.nOut; ++oc) {
                        const float w = (oc == epi.channel) ? r : 0.0f;
                        if (epi.mixPartial) epi.mixPartial[((size_t) (epi.tileBase + ch) * epi.nOut + oc) * epi.blockSize + offset + i] = w;
                        if (epi.outVoice) epi.outVoice[((size_t) (epi.voice0 + ch) * epi.nOut + oc) * epi.outStride + epi.outOffset + offset + i] = w;
                    }
                }
            }
        }
        if (fill + n == CONV_BLOCK) {
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                const int ch = chs[c];
                if (!oks[c]) continue;
                const float* y = reinterpret_cast<const float*>(&Sc[c][0]);
                float* ov = overlap + (size_t) ch * CONV_BLOCK;
                float* ib = inbuf + (size_t) ch * CONV_BLOCK;
                for (int i = t; i < CONV_BLOCK; i += TM_GROUP) { ov[i] = y[CONV_BLOCK + i] * scale; if (!wholeBlock) ib[i] = 0.0f; }
            }
        }
        tgroup_sync();                                                      // Sc is reused by the next transform
    };

    int nloc = 0, prevU = -1;
    for (int u = blockIdx.x; u < numUnits; u += gridDim.x, ++nloc) {
        forward(u, nloc);
        if (prevU >= 0) inverse(prevU, nloc - 1);
        prevU = u;
    }
    if (prevU >= 0) inverse(prevU, nloc - 1);
}

cudaError_t convolver_process_chunk(ConvolverState& st, const float* in, int inStride, float* out, int stride, int offset, int n, cudaStream_t stream,
                                    const ConvEpilogue& epi) {
    if (st.planOnly) return cudaErrorNotSupported;
    if (st.maxS == 0) {   // empty (fully trimmed) IR on every channel: silence (FFTConvolver.cpp:149-153)
        if (epi.active) {
            cudaError_t e = cudaSuccess;
            if (epi.mixPartial) e = cudaMemset2DAsync(epi.mixPartial + (size_t) epi.tileBase * epi.nOut * epi.blockSize + offset, sizeof(float) * epi.blockSize, 0, sizeof(float) * n, (size_t) st.nv * epi.nOut, stream);
            if (e == cudaSuccess && epi.outVoice) e = cudaMemset2DAsync(epi.outVoice + (size_t) epi.voice0 * epi.nOut * epi.outStride + epi.outOffset + offset, sizeof(float) * epi.outStride, 0, sizeof(float) * n, (size_t) st.nv * epi.nOut, stream);
            return e;
        }
        return cudaMemset2DAsync(out + offset, sizeof(float) * stride, 0, sizeof(float) * n, st.nv, stream);
    }
    const int units = (st.nv + CONV_CH_PER_CTA - 1) / CONV_CH_PER_CTA;
    static int smCount = 0;
    const bool perCh = st.perChannel();
    const size_t smem = perCh ? ConvForm<true>::smem() : ConvForm<false>::smem();
    if (smCount == 0) {
        cudaError_t e = cudaFuncSetAttribute(convolve_chunk_tm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) ConvForm<false>::smem());
        if (e == cudaSuccess) e = cudaFuncSetAttribute(convolve_chunk_tm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) ConvForm<true>::smem());
        if (e != cudaSuccess) return e;
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&smCount, cudaDevAttrMultiProcessorCount, dev);
        if (smCount <= 0) smCount = 132;
    }
    const int persistent = smCount * TM_CTAS_PER_SM;                   // a multiple of the SM count: one resident wave
    // Every CTA walks the same number of channel pairs: 512 pairs on 264 resident CTAs (H100: 132 SMs x 2) would leave 16 CTAs idle for
    // the second half of the kernel (248 CTAs hold two pairs, 16 hold one); 256 CTAs with two pairs each keep the HBM stream full until the end.
    int grid = units < persistent ? units : persistent;
    if (units > persistent) {
        const int rounds = (units + persistent - 1) / persistent;
        grid = (units + rounds - 1) / rounds;
    }
    if (perCh)
        convolve_chunk_tm_kernel<true><<<grid, TM_THREADS, smem, stream>>>(in, inStride, out, stride, offset, n, st.fill, st.cur, 0, st.partitions, st.nv,
                                                                          nullptr, st.dChan, st.dUnits, st.dFdl, st.dYpre, st.dOverlap, st.dInBuf, st.dTw, epi);
    else   // one IR for every channel (its S may be below the ring's R after reassignments)
        convolve_chunk_tm_kernel<false><<<grid, TM_THREADS, smem, stream>>>(in, inStride, out, stride, offset, n, st.fill, st.cur, st.maxS, st.partitions, st.nv,
                                                                           st.irs[0]->dH, nullptr, nullptr, st.dFdl, st.dYpre, st.dOverlap, st.dInBuf, st.dTw, epi);
    st.fill += n;
    if (st.fill == CONV_BLOCK) {
        st.fill = 0;
        st.cur = (st.cur > 0) ? st.cur - 1 : st.partitions - 1;   // FFTConvolver.cpp:200
    }
    return cudaGetLastError();
}

cudaError_t convolver_relayout(float2* dst, const float2* src, int nv, int oldR, int newR, int cur, cudaStream_t stream) {
    if (nv == 0 || newR == 0) return cudaSuccess;
    convolve_ring_relayout_kernel<<<dim3(nv, newR), 128, 0, stream>>>(dst, src, oldR, newR, cur);
    return cudaGetLastError();
}

} // namespace eb
