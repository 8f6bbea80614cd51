// kernels.h — host-callable launchers of the device kernels (render_kernel.cu, convolve_kernel.cu).
#pragma once
#include "program.h"
#ifndef __CUDACC_RTC__   // host-callable launchers: not part of a run-time compiled specialisation of K1
#include <cuda_runtime.h>

namespace eb {

// K1: fused render-sequence kernel, one launch per voice group per block.
int render_niter_for(int tileWidth, int niterOverride);   // elements per lane per sample tile (E = 32*NITER = L*T)
size_t render_smem_bytes(int nSlots, int nOut, int nStateRows, int nParams, int warpsPerCta, int tileWidth, int niterOverride);
int render_delay_buf_floats(int nDelayBuf, int tileWidth, int niterOverride);   // per warp, a multiple of 4
struct SpecKernel;   // spec_host.h: K1 compiled at run time against one program (nullptr = the built-in interpreter)
cudaError_t launch_render_block(const LaunchParams& P, int warpsPerCta, int niterOverride, cudaStream_t stream, const SpecKernel* spec = nullptr);

// K1 for many voice groups of one tile geometry in one launch (descs / tileStart are device pointers).  outOffset / inOffset: the
// column of every output / input row the block starts at (an offline chunk holds several blocks per row; 0 otherwise).
cudaError_t launch_render_groups(const LaunchParams* descs, const int* tileStart, int nGroups, int totalTiles, int tileWidth,
                                 int maxSlots, int nOut, int maxStateRows, int maxParams, int warpsPerCta, long long sampleTime, int outOffset, int inOffset, cudaStream_t stream,
                                 int niterOverride = 0);

// K1 for many ONE-VOICE graphs whose programs were cut into pipeline stages (LaunchParams::pipeW): one CTA of `stages` warps per graph.
cudaError_t launch_render_groups_pipe(const LaunchParams* descs, const int* tileStart, int nGroups, int totalTiles, int stages,
                                      int maxSlots, int nOut, int maxStateRows, int maxParams, long long sampleTime, int outOffset, int inOffset, cudaStream_t stream,
                                      int niterOverride = 0);

// K2: deterministic reduction of per-tile partial mixes into the mix bus, channel c at out + c * outStride (blockSize for the mix bus
// of one block; an offline chunk's column otherwise; a host-delivery copy always has pitch blockSize).
// scratch: [MIX_REDUCE_MAX_GROUPS][nOut][blockSize] floats, tickets: [nOut * ceil(blockSize/32)] zeroed counters (both may be null:
// single-pass reduction).
constexpr int MIX_REDUCE_MAX_GROUPS = 16;
// Host delivery of the finished mix bus: the kernel that writes the FINAL mix (K2 on one GPU, K4 across GPUs) also stores it into a
// mapped pinned host buffer and, once every CTA has done so (`done` counter), raises `flag = seq` there — Runtime::process polls that
// word instead of paying a D2H copy launch + stream synchronize per block.  out == nullptr: no host delivery.
struct HostDeliver {
    float* out = nullptr;            // device alias of the mapped host buffer [nOut][blockSize]
    uint32_t* flag = nullptr;        // device alias of the host sequence word
    unsigned int* done = nullptr;    // device counter, zero between launches
    uint32_t seq = 0;
};
cudaError_t launch_mix_reduce(const float* partial, float* out, int outStride, float* scratch, unsigned int* tickets, int nTiles, int nOut,
                              int blockSize, int numSamples, cudaStream_t stream, HostDeliver hd = HostDeliver{});

// K2w (mix_wide_kernel.cu): the mix bus for nOut > MAX_OUT_CHANNELS from COMPACT partial rows [row][blockSize].  Channel c sums its row
// list rows[rowPtr_c ...] with K2's tree into out + c * outStride (pitch as for K2); a segment is one tile group of one channel.  Every channel in [0, nOut) has at least one
// segment (a channel without rows has one empty segment, which writes +0.0).
constexpr int MAX_WIDE_OUT_CHANNELS = 4096;   // output channels of the compact mix bus; a call with more returns -2
struct WideSeg {
    int channel;
    int rowBegin, rowCount;   // the group's rows: rows[rowBegin .. rowBegin + rowCount)
    int groups, group;        // G_c and this segment's index in it
    int scratch;              // G_c > 1: first of the channel's G_c scratch rows [blockSize] and ticket rows [ceil(blockSize / 32)]; else -1
};
// segs: the nSmall segments of fewer than WIDE_BIG_ROWS rows (a warp each), then the nBig larger ones (a CTA of 32 warps each).
constexpr int WIDE_BIG_ROWS = 128;
cudaError_t launch_mix_reduce_wide(const float* partial, const int* rows, const WideSeg* segs, int nSmall, int nBig, int nOut, float* out,
                                   int outStride, float* scratch, unsigned int* tickets, int blockSize, int numSamples, cudaStream_t stream,
                                   HostDeliver hd = HostDeliver{});
// Per-voice outputs of the wide path: compact row r [blockSize] -> row dstRow[r] of out ([voice][nOut][blockSize]), numSamples samples.
cudaError_t launch_voice_out_scatter(const float* compact, const int* dstRow, int nRows, float* out, int blockSize, int numSamples, cudaStream_t stream);

// K4: the one collective of the path (SURVEY.md §8e) as our own kernel over NVLink/NVSwitch peer memory: K2 leaves this rank's
// partial mix bus in PeerMix::own; world-1 CTAs each push it into one peer's buffer as (sample, epoch) pairs, then every CTA waits for the
// pairs of all sources to arrive in its OWN buffer and sums a share of the samples in rank order — one launch, deterministic, no NCCL
// call on the data path, one NVLink one-way latency between "my partial is ready" and "the peer can use it".  count = 0 makes it a
// cross-GPU stream barrier (flags).
constexpr int MAX_PEERS = 8;
struct PeerMix {
    uint2* slot[MAX_PEERS];       // slot[p]: rank p's exchange buffer [2 parities][MAX_PEERS sources][stride] of (sample bits, epoch) pairs
                                  // (peer-mapped for p != rank): every 8-byte store carries its own arrival flag, so the data needs no
                                  // fence and no separate flag store behind it (the "LL" form NCCL uses for small messages)
    uint32_t* flag[MAX_PEERS];    // flag[p]: rank p's flags [2][MAX_PEERS] — used by the pure barrier (count = 0) only
    float* own;                   // this rank's partial mix bus [stride] (local; K2 leaves it here)
    int rank, world, stride;
};
cudaError_t launch_mix_exchange(const PeerMix& pm, float* mix, int count, uint32_t epoch, int* status, cudaStream_t stream, HostDeliver hd = HostDeliver{});

// K5 (event_log_kernel.cu): the per-block event log of an offline render with events.  After a block renders, one launch copies what a
// poll after that block would read into the chunk's event log and applies the poll's side effects, so that the device state evolves as
// under a process() + processQueuedEvents() loop.  One item per polled event node, voices [b, b + n) of its group:
//   EVLOG_ROWS     meter / snapshot: log [3][n] words of state rows 0..2 (the readouts, the push count); zero the push count
//   EVLOG_CAPTURE  capture: log [3][n] words of state rows 2..4 (write position, read position, relay-ready flag), then [n][lim] floats:
//                  the ring's samples [r, w) of each voice (at most lim); set the read position to w and clear the flag
//   EVLOG_WINDOW   scope / fft: log [tile t0..t1)[channel < nch][size][L] floats, the ring window at read position r (no side effect)
//   EVLOG_READOUT  meter / snapshot as arrays (Engine::pollReadouts): fresh[i] = 1 where voice b + i's queue holds a readout (push count
//                  mod 32 != 0), and then outA[i] = the bits of state row aRow, outB[i] (if not null) those of row 1; zero the push
//                  count.  drain == 0 (the node is not under an active root): fresh[i] = 0 only, the rows are not read
enum EventLogKind : int { EVLOG_ROWS = 0, EVLOG_CAPTURE = 1, EVLOG_WINDOW = 2, EVLOG_READOUT = 3 };
struct EventLogItem {
    uint32_t* rows;           // the node's first state row (row j of voice v: rows[j * Vpad + v])
    const float* ring;        // capture: [tile][ringFloats][L]; scope / fft: [tile][ringCh][SCOPE_RING][L]
    uint32_t* log;            // where this item's record starts
    int kind, b, n, Vpad, L;
    uint32_t cap, lim, ringFloats;   // capture: ring capacity (a power of two), samples logged per voice at most, ring + scratch floats per lane
    uint32_t r, size;         // window: read position, window length
    int ringCh, nch, t0, t1;  // window: channels of the ring, channels logged, tiles
    uint32_t* outA;           // readout: destinations of voices [b, b + n), compacted (outB may be null)
    uint32_t* outB;
    uint8_t* fresh;
    int aRow, drain;          // readout: the state row `a` reads (meter 0 = min, snapshot 1 = value); drain the queue
};
constexpr int EVENT_LOG_BATCH = 32;   // items per launch (the batch travels as one kernel parameter)
struct EventLogBatch { int n; EventLogItem item[EVENT_LOG_BATCH]; };
cudaError_t launch_event_log(const EventLogBatch& batch, cudaStream_t stream);

// K6 (reset_kernel.cu): voices restart as fresh instances (Engine::resetVoices).  The reset plan of a voice group lists what a voice
// owns: cells of state rows, lanes of tile-structured buffers [tile][pos][L] and voice-major convolver regions.  One launch covers the
// runs of a call — the sorted voices of one voice tile each, voices[runStart[r] .. runStart[r + 1]) in group runGroup[r].
enum ResetRowKind : uint32_t { RESET_ROW_BITS = 0, RESET_ROW_DOUBLE = 1, RESET_ROW_SHADOW = 2 };
struct ResetRow { int row; uint32_t kind; uint32_t value; };   // BITS: the creation bits; DOUBLE: a double pair row, zeroed; SHADOW: value = shadow row
struct ResetBuf { float* base; long long positions, pos0; };  // [tile][positions][L] floats; pos0: positions of the group's earlier buffers
struct ResetConv { float* base; long long quads, quad0; };    // [voice][quads] float4; quad0: quads of the group's earlier regions
struct ResetGroup {
    float* rows;
    int v0, Vpad, L;
    int row0, nRows, buf0, nBufs, conv0, nConvs;              // the group's entries of the plan arrays
    long long tilePositions, convQuads;                       // sums over its buffers / regions
};
struct ResetLaunch {
    const ResetGroup* groups; const ResetRow* rows; const ResetBuf* bufs; const ResetConv* convs;
    const int* voices; const int* runStart; const int* runGroup;
};
cudaError_t launch_reset_voices(const ResetLaunch& a, int nRuns, int slices, cudaStream_t stream);

// A/B builds (-DEB_OPPROF): cycles / dispatches per opcode of the interpreter; zeros in the product library.
cudaError_t debug_opprof_read(unsigned long long* out128, bool reset);

} // namespace eb
#endif   // __CUDACC_RTC__
