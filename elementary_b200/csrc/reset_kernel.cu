// reset_kernel.cu — K6, voice reset (kernels.h ResetPlan, DESIGN.md section 4): chosen voices of any voice groups restart as fresh
// instances in one launch, between two blocks, without a host round trip.
//
// The host groups the sorted voice list into runs, one per (voice group, voice tile).  grid.x = run, grid.y = slice: the blocks of
// one run split its work evenly.  A run's work is
//   * its voices' cells of the group's state rows: each row item gets its creation bits, zero (a double pair), or the same voice's
//     cell of a shadow row (the last `rand.seed` / `once.arm` set for the voice);
//   * the run's lanes of every tile-structured buffer [tile][pos][L] of the group (delay rings, tap buffers, scope / fft / capture
//     rings): consecutive threads take consecutive reset lanes of one position, then the next position, so that the stores of a
//     position land in the same 128-byte lines however few lanes of the tile are reset;
//   * its voices' voice-major convolver regions (float4 stores).
#include "kernels.h"

namespace eb {

namespace {
constexpr int RESET_THREADS = 256;

// [lo, hi) of `total` items for slice s of S
__device__ __forceinline__ void sliceRange(long long total, int s, int S, long long& lo, long long& hi) {
    lo = total * s / S;
    hi = total * (s + 1) / S;
}
}

__global__ void __launch_bounds__(RESET_THREADS) reset_voices_kernel(const __grid_constant__ ResetLaunch a) {
    const int run = blockIdx.x, s = blockIdx.y, S = gridDim.y;
    const ResetGroup& g = a.groups[a.runGroup[run]];
    const int b = a.runStart[run], m = a.runStart[run + 1] - b;   // m distinct voices, ascending, all in one tile
    __shared__ int lanes[32];                                      // group-relative voice of each reset lane, in lane order
    if (threadIdx.x < m) lanes[threadIdx.x] = a.voices[b + threadIdx.x] - g.v0;
    __syncthreads();
    const int tile = lanes[0] / g.L;

    long long lo, hi;
    // state rows: item-major, voice-minor
    sliceRange((long long) g.nRows * m, s, S, lo, hi);
    for (long long i = lo + threadIdx.x; i < hi; i += RESET_THREADS) {
        const ResetRow r = a.rows[g.row0 + (int) (i / m)];
        const int u = lanes[(int) (i % m)];
        uint32_t* rows = reinterpret_cast<uint32_t*>(g.rows);
        if (r.kind == RESET_ROW_DOUBLE) {
            rows[(size_t) r.row * g.Vpad + 2 * u] = 0u;
            rows[(size_t) r.row * g.Vpad + 2 * u + 1] = 0u;
        } else {
            rows[(size_t) r.row * g.Vpad + u] = (r.kind == RESET_ROW_SHADOW) ? rows[(size_t) r.value * g.Vpad + u] : r.value;
        }
    }
    // tile buffers: position-major over the concatenated positions of the group's buffers, reset lanes minor
    sliceRange(g.tilePositions * m, s, S, lo, hi);
    for (int k = 0; k < g.nBufs && lo < hi; ++k) {
        const ResetBuf buf = a.bufs[g.buf0 + k];
        const long long b0 = buf.pos0 * m, b1 = (buf.pos0 + buf.positions) * m;
        const long long e0 = lo > b0 ? lo : b0, e1 = hi < b1 ? hi : b1;
        float* base = buf.base + (size_t) tile * (size_t) buf.positions * g.L;
        for (long long i = e0 + threadIdx.x; i < e1; i += RESET_THREADS) {
            const long long j = i - b0;
            base[(size_t) (j / m) * g.L + lanes[(int) (j % m)] % g.L] = 0.0f;
        }
    }
    // convolver regions: voice-major [voice][floats], float4 stores
    sliceRange(g.convQuads * m, s, S, lo, hi);
    for (int k = 0; k < g.nConvs && lo < hi; ++k) {
        const ResetConv c = a.convs[g.conv0 + k];
        const long long b0 = c.quad0 * m, b1 = (c.quad0 + c.quads) * m;
        const long long e0 = lo > b0 ? lo : b0, e1 = hi < b1 ? hi : b1;
        for (long long i = e0 + threadIdx.x; i < e1; i += RESET_THREADS) {
            const long long j = i - b0;
            reinterpret_cast<float4*>(c.base)[(size_t) lanes[(int) (j / c.quads)] * c.quads + (size_t) (j % c.quads)] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}

cudaError_t launch_reset_voices(const ResetLaunch& a, int nRuns, int slices, cudaStream_t stream) {
    if (nRuns <= 0) return cudaSuccess;
    reset_voices_kernel<<<dim3((unsigned) nRuns, (unsigned) slices), RESET_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

} // namespace eb
