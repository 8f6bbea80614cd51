// event_log_kernel.cu — K5, the per-block event log of an offline render with events (kernels.h EventLogItem, DESIGN.md section 4).
//
// An offline render enqueues its blocks back to back, so nobody can poll the event queues between two blocks.  After every block this
// kernel does on the device what a poll between the blocks would have done: it copies what the poll would read into the chunk's event
// log (the host turns it into events after the chunk's copy, with the same code as a live poll) and applies the poll's side effects —
// meter / snapshot queues drained, capture read positions moved to the write position and relay flags cleared — so that the render of
// the next block sees the state a process() + processQueuedEvents() loop leaves behind.  Scope / fft windows are only read: their read
// positions are the same for every voice of a group and live on the host.
//
// The same kernel serves the array poll (Engine::pollReadouts, EVLOG_READOUT items): meter / snapshot readouts written straight into
// caller arrays, with the live poll's side effect.
//
// grid.y = item; grid.x strides over the item's work: a voice per thread (rows, readouts), a voice per warp (capture), a float per
// thread (window).
#include <algorithm>

#include "kernels.h"

namespace eb {

// EVLOG_READOUT (kernels.h); out of line, so that the other item kinds keep their register allocation
__device__ __noinline__ void readout_item(const EventLogItem& it, long long tid, long long nth) {
    for (long long i = tid; i < it.n; i += nth) {
        uint8_t f = 0;
        if (it.drain) {
            uint32_t* row = it.rows + it.b + i;
            f = row[2 * it.Vpad] % 32u != 0u;     // the 32-slot queue arithmetic of the live poll (events_host.cpp emitPoll)
            if (f) {
                it.outA[i] = row[it.aRow * it.Vpad];
                if (it.outB) it.outB[i] = row[it.Vpad];
            }
            row[2 * it.Vpad] = 0u;
        }
        it.fresh[i] = f;
    }
}

__global__ void __launch_bounds__(256) event_log_kernel(const __grid_constant__ EventLogBatch batch) {
    const EventLogItem& it = batch.item[blockIdx.y];
    const long long tid = (long long) blockIdx.x * blockDim.x + threadIdx.x, nth = (long long) gridDim.x * blockDim.x;
    const int n = it.n;
    if (it.kind == EVLOG_ROWS) {
        for (long long i = tid; i < n; i += nth) {
            uint32_t* row = it.rows + it.b + i;
            it.log[i] = row[0];
            it.log[n + i] = row[it.Vpad];
            it.log[2 * n + i] = row[2 * it.Vpad];
            row[2 * it.Vpad] = 0u;
        }
    } else if (it.kind == EVLOG_CAPTURE) {
        const int lane = threadIdx.x & 31;
        const uint32_t mask = it.cap - 1;
        float* const samples = reinterpret_cast<float*>(it.log + 3 * (size_t) n);
        for (long long i = tid >> 5; i < n; i += nth >> 5) {
            const int v = it.b + (int) i;
            const uint32_t w = it.rows[2 * (size_t) it.Vpad + v], r = it.rows[3 * (size_t) it.Vpad + v], ready = it.rows[4 * (size_t) it.Vpad + v];
            const uint32_t avail = (w > r) ? (w - r) : ((it.cap - (r - w)) & mask);
            const uint32_t cnt = avail < it.lim ? avail : it.lim;
            const float* col = it.ring + (size_t) (v / it.L) * it.ringFloats * it.L + (v % it.L);
            float* dst = samples + (size_t) i * it.lim;
            for (uint32_t k = lane; k < cnt; k += 32) dst[k] = col[(size_t) ((r + k) & mask) * it.L];
            __syncwarp();   // every lane has read the positions before lane 0 moves them
            if (lane == 0) {
                it.log[i] = w; it.log[n + i] = r; it.log[2 * n + i] = ready;
                it.rows[3 * (size_t) it.Vpad + v] = w;
                it.rows[4 * (size_t) it.Vpad + v] = 0u;
            }
        }
    } else if (it.kind == EVLOG_READOUT) {
        readout_item(it, tid, nth);
    } else {
        const long long per = (long long) it.size * it.L, total = (long long) (it.t1 - it.t0) * it.nch * per;
        float* const dst = reinterpret_cast<float*>(it.log);
        for (long long j = tid; j < total; j += nth) {
            const long long q = j / per, rem = j - q * per;
            const int tile = it.t0 + (int) (q / it.nch), ch = (int) (q % it.nch);
            const uint32_t pos = (it.r + (uint32_t) (rem / it.L)) & (SCOPE_RING - 1);
            dst[j] = it.ring[((size_t) (tile * it.ringCh + ch) * SCOPE_RING + pos) * it.L + rem % it.L];
        }
    }
}

cudaError_t launch_event_log(const EventLogBatch& batch, cudaStream_t stream) {
    if (batch.n <= 0) return cudaSuccess;
    long long work = 1;
    for (int k = 0; k < batch.n; ++k) {
        const EventLogItem& it = batch.item[k];
        const long long w = (it.kind == EVLOG_ROWS || it.kind == EVLOG_READOUT) ? it.n : it.kind == EVLOG_CAPTURE ? 32LL * it.n
                                                                                      : (long long) (it.t1 - it.t0) * it.nch * it.size * it.L;
        work = w > work ? w : work;
    }
    const unsigned gx = (unsigned) std::min<long long>((work + 255) / 256, 1024);
    event_log_kernel<<<dim3(gx, (unsigned) batch.n), 256, 0, stream>>>(batch);
    return cudaGetLastError();
}

} // namespace eb
