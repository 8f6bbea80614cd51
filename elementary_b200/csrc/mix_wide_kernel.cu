// mix_wide_kernel.cu — the mix bus past MAX_OUT_CHANNELS output channels (DESIGN.md section 4, K2w).
//
// With nOut <= MAX_OUT_CHANNELS every tile writes a dense [nOut][blockSize] partial and K2 (render_kernel.cu) reduces
// [tile][nOut][blockSize].  Past that the partial rows are COMPACT: a voice group writes one row per tile for each channel its roots
// aim at, and nothing for the others, so a channel is the sum over its own row list R_c (CSR, built by the host).  K2w applies K2's
// summation tree to each list: G_c = min(16, ceil(|R_c| / 256)) groups of roundup(ceil(|R_c| / G_c), 32) rows; in a group, lane j
// sums items j, j + 32, ... with four interleaved accumulators, then the group sum is 0 + lane 0 + ... + lane 31; with G_c > 1 the
// mix is 0 + s_0 + ... + s_(G_c - 1).  A channel without rows is +0.0.
//
// The work is sized to the rows, per segment (one tile group of one channel) and 32-sample chunk, lane = sample.  A segment of fewer
// than WIDE_BIG_ROWS rows gets one WARP, which walks the 32 row lanes of the tree itself, eight at a time with their four
// accumulators in registers (32 independent loads in flight): a channel of one row costs one coalesced 128-byte load per chunk
// instead of a 1024-thread CTA.  A larger segment gets a CTA of 32 warps, one row lane each (K2's shape), whose lane sums meet in
// shared memory and are added in lane order — the same tree either way.
// A channel of several groups finishes like K2: each group leaves its sum in scratch, the warp that arrives last at the
// (channel, chunk) ticket adds them in group order — the order is a function of |R_c| only, never of which warp finishes last.
#include "kernels.h"

namespace eb {

__device__ __forceinline__ void wide_st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// HostDeliver arrival of one warp that has just written its part of the final mix bus (kernels.h HostDeliver): the warp that
// arrives last raises the host flag.
__device__ __forceinline__ void wide_deliver_arrive(const HostDeliver& hd, unsigned int nFinal, int lane) {
    __threadfence_system();
    __syncwarp();
    if (lane == 0) {
        const unsigned int d = atomicAdd(hd.done, 1u);
        if (d == nFinal - 1) {
            *hd.done = 0;                                     // ready for the next block of audio
            __threadfence_system();
            wide_st_release_sys(hd.flag, hd.seq);
        }
    }
}

constexpr int WIDE_WARPS = 4;      // small segments: warps per CTA, one work item each
constexpr int WIDE_LANE_BLOCK = 8; // small segments: row lanes of the tree a thread works on at once
constexpr int WIDE_BIG_WARPS = 32; // large segments (kernels.h WIDE_BIG_ROWS rows or more): one CTA per work item, one row lane
constexpr int WIDE_BIG_LANES = 32 / WIDE_BIG_WARPS;   // per warp — K2's shape, 32 samples x 32 row lanes

// Row lanes j0 .. j0 + B - 1 of the tree over the segment's rows r[0 .. n): sums[q] = (a0 + a1) + (a2 + a3) of lane j0 + q, item k of
// lane j (row r[j + 32 k]) going to a[k mod 4] while four items remain and to a0 after that.  A lane without items gives +0.0.
template <int B>
__device__ __forceinline__ void wide_lane_sums(const float* __restrict__ col, const int* __restrict__ r, int n, int j0, int blockSize, float (&sums)[B]) {
    float a[B][4];
#pragma unroll
    for (int q = 0; q < B; ++q) a[q][0] = a[q][1] = a[q][2] = a[q][3] = 0.0f;
    const int mMax = (n - j0 + 31) / 32;                          // items of row lane j0, the fullest of the block
    for (int k = 0; k + 3 < mMax; k += 4) {                       // rounds of four items, all B lanes' loads in flight together
#pragma unroll
        for (int q = 0; q < B; ++q) {
            const int j = j0 + q;
            if (k + 3 < (n - j + 31) / 32) {
                const int* rj = r + j + 32 * k;
                a[q][0] += col[(size_t) __ldg(rj) * blockSize];
                a[q][1] += col[(size_t) __ldg(rj + 32) * blockSize];
                a[q][2] += col[(size_t) __ldg(rj + 64) * blockSize];
                a[q][3] += col[(size_t) __ldg(rj + 96) * blockSize];
            }
        }
    }
#pragma unroll
    for (int q = 0; q < B; ++q) {                                 // the rest of each lane's items go to a0
        const int j = j0 + q;
        const int mj = j < n ? (n - j + 31) / 32 : 0;
        for (int k = mj / 4 * 4; k < mj; ++k) a[q][0] += col[(size_t) __ldg(r + j + 32 * k) * blockSize];
        sums[q] = (a[q][0] + a[q][1]) + (a[q][2] + a[q][3]);
    }
}

// One warp with the group sum v of its segment and 32-sample chunk: the mix itself (G_c = 1), or the group's scratch row and, from the
// warp that arrives last at the (channel, chunk) ticket, 0 + s_0 + ... + s_(G-1) in group order.  Then the host-delivery arrival.
__device__ __forceinline__ void wide_finish(const WideSeg& sg, float v, int chunk, int chunksPerBlock, int s, bool live, int lane,
                                            float* __restrict__ out, float* __restrict__ scratch, unsigned int* __restrict__ tickets,
                                            int blockSize, int outStride, unsigned int nFinal, const HostDeliver& hd) {
    const size_t o = (size_t) sg.channel * outStride + s, oh = (size_t) sg.channel * blockSize + s;
    if (sg.groups == 1) {
        if (live) { out[o] = v; if (hd.out) hd.out[oh] = v; }
        if (hd.out) wide_deliver_arrive(hd, nFinal, lane);
        return;
    }
    if (live) scratch[(size_t) (sg.scratch + sg.group) * blockSize + s] = v;
    __threadfence();
    __syncwarp();
    unsigned int last = 0;
    if (lane == 0) {
        unsigned int* t = tickets + (size_t) sg.scratch * chunksPerBlock + chunk;
        last = atomicAdd(t, 1u) == (unsigned int) sg.groups - 1;
        if (last) *t = 0;                                         // ready for the next block of audio
    }
    last = __shfl_sync(0xFFFFFFFFu, last, 0);
    if (!last) return;
    __threadfence();
    if (live) {
        float w = 0.0f;
        for (int k = 0; k < sg.groups; ++k) w += __ldcg(scratch + (size_t) (sg.scratch + k) * blockSize + s);
        out[o] = w;
        if (hd.out) hd.out[oh] = w;
    }
    if (hd.out) wide_deliver_arrive(hd, nFinal, lane);
}

// Segments of fewer than WIDE_BIG_ROWS rows: one warp per (segment, chunk), walking the row lanes eight at a time.
__global__ void __launch_bounds__(32 * WIDE_WARPS) mix_reduce_wide_kernel(const float* __restrict__ partial, const int* __restrict__ rows,
                                                                          const WideSeg* __restrict__ segs, int nItems, int chunks, int chunksPerBlock,
                                                                          float* __restrict__ out, float* __restrict__ scratch,
                                                                          unsigned int* __restrict__ tickets, int blockSize, int outStride, int numSamples,
                                                                          unsigned int nFinal, const HostDeliver hd) {
    const int item = blockIdx.x * WIDE_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (item >= nItems) return;                                   // whole warps leave
    const int chunk = item % chunks;
    const WideSeg sg = segs[item / chunks];
    const int s = chunk * 32 + lane;
    const bool live = s < numSamples;
    const float* const col = partial + (live ? s : 0);            // lanes past numSamples read sample 0 and discard it
    const int n = sg.rowCount;
    float v = 0.0f;
    const int nl = min(32, n);                                    // lanes of the tree that have items
    for (int jb = 0; jb < nl; jb += WIDE_LANE_BLOCK) {
        float sums[WIDE_LANE_BLOCK];
        wide_lane_sums<WIDE_LANE_BLOCK>(col, rows + sg.rowBegin, n, jb, blockSize, sums);
        // lanes in order; a lane without items adds +0.0, which changes no sum that starts from +0.0
#pragma unroll
        for (int q = 0; q < WIDE_LANE_BLOCK; ++q)
            if (jb + q < nl) v += sums[q];
    }
    wide_finish(sg, v, chunk, chunksPerBlock, s, live, lane, out, scratch, tickets, blockSize, outStride, nFinal, hd);
}

// Segments of WIDE_BIG_ROWS rows or more: one CTA per (segment, chunk); warp w forms the sums of row lanes w * WIDE_BIG_LANES ...
// into shared memory, then warp 0 adds the 32 lanes in order — the same tree, and the same loads per thread as K2.
__global__ void __launch_bounds__(32 * WIDE_BIG_WARPS) mix_reduce_wide_big_kernel(const float* __restrict__ partial, const int* __restrict__ rows,
                                                                                  const WideSeg* __restrict__ segs, int chunks, int chunksPerBlock,
                                                                                  float* __restrict__ out, float* __restrict__ scratch,
                                                                                  unsigned int* __restrict__ tickets, int blockSize, int outStride, int numSamples,
                                                                                  unsigned int nFinal, const HostDeliver hd) {
    __shared__ float laneSum[32][33];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunk = blockIdx.x % chunks;
    const WideSeg sg = segs[blockIdx.x / chunks];
    const int s = chunk * 32 + lane;
    const bool live = s < numSamples;
    const float* const col = partial + (live ? s : 0);
    float sums[WIDE_BIG_LANES];
    wide_lane_sums<WIDE_BIG_LANES>(col, rows + sg.rowBegin, sg.rowCount, warp * WIDE_BIG_LANES, blockSize, sums);
#pragma unroll
    for (int q = 0; q < WIDE_BIG_LANES; ++q) laneSum[warp * WIDE_BIG_LANES + q][lane] = sums[q];
    __syncthreads();
    if (warp != 0) return;
    float v = 0.0f;
    for (int j = 0; j < 32; ++j) v += laneSum[j][lane];           // every lane has items (>= 32 rows): 0 + lane 0 + ... + lane 31
    wide_finish(sg, v, chunk, chunksPerBlock, s, live, lane, out, scratch, tickets, blockSize, outStride, nFinal, hd);
}

// Per-voice outputs of the wide path: the compact rows [row][blockSize] go to out[dstRow[row]] ([voice][nOut][blockSize]); the
// other channels of the destination were zeroed before.
__global__ void __launch_bounds__(128) voice_out_scatter_kernel(const float* __restrict__ compact, const int* __restrict__ dstRow, int nRows,
                                                                float* __restrict__ out, int blockSize, int numSamples) {
    for (int row = blockIdx.x; row < nRows; row += gridDim.x) {
        const float* src = compact + (size_t) row * blockSize;
        float* dst = out + (size_t) __ldg(dstRow + row) * blockSize;
        for (int s = threadIdx.x; s < numSamples; s += blockDim.x) dst[s] = src[s];
    }
}

cudaError_t launch_mix_reduce_wide(const float* partial, const int* rows, const WideSeg* segs, int nSmall, int nBig, int nOut, float* out,
                                   int outStride, float* scratch, unsigned int* tickets, int blockSize, int numSamples, cudaStream_t stream, HostDeliver hd) {
    const int chunks = numSamples > 0 ? (numSamples + 31) / 32 : 1;
    const int chunksPerBlock = (blockSize + 31) / 32;
    const unsigned int nFinal = (unsigned int) (nOut * chunks);   // (channel, chunk) pairs: the host-delivery arrivals of both launches
    if (nSmall > 0) {
        const int nItems = nSmall * chunks;
        mix_reduce_wide_kernel<<<(nItems + WIDE_WARPS - 1) / WIDE_WARPS, 32 * WIDE_WARPS, 0, stream>>>(
            partial, rows, segs, nItems, chunks, chunksPerBlock, out, scratch, tickets, blockSize, outStride, numSamples, nFinal, hd);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    if (nBig > 0) {
        mix_reduce_wide_big_kernel<<<nBig * chunks, 32 * WIDE_BIG_WARPS, 0, stream>>>(
            partial, rows, segs + nSmall, chunks, chunksPerBlock, out, scratch, tickets, blockSize, outStride, numSamples, nFinal, hd);
        return cudaGetLastError();
    }
    return cudaSuccess;
}

cudaError_t launch_voice_out_scatter(const float* compact, const int* dstRow, int nRows, float* out, int blockSize, int numSamples, cudaStream_t stream) {
    if (nRows <= 0 || numSamples <= 0) return cudaSuccess;
    voice_out_scatter_kernel<<<std::min(nRows, 65535), 128, 0, stream>>>(compact, dstRow, nRows, out, blockSize, numSamples);
    return cudaGetLastError();
}

} // namespace eb
