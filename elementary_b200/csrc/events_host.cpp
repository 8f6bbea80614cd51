// events_host.cpp — the parts of eb::Engine that talk to the outside between blocks: the cross-GPU exchange plumbing
// (CUDA IPC mapping of the K4 buffers) and Runtime::processQueuedEvents (read-back of the per-voice analysis records
// the kernel leaves in HBM, turned into the reference's event objects).  See graph_host.h.
#include "graph_host.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <set>
#include <string>
#include <vector>

namespace eb {

// ---------------------------------------------------------------------------------------------------------
// K4 plumbing: exchange buffers mapped across the ranks of one box with CUDA IPC (one process per GPU)
int Engine::peerExport(void* handleOut64) {
    Lock lk(mu_);
    if (planOnly_) return fail(rc::CudaError, "plan-only runtime has no device memory to export");
    dsetdev();
    if (!dExchange_) {
        const size_t stride = (size_t) MAX_OUT_CHANNELS * blockSize_;
        exchangeFlagOffset_ = sizeof(uint2) * 2 * MAX_PEERS * stride;                       // (sample, epoch) pairs: [2][MAX_PEERS][stride]
        exchangeOwnOffset_ = exchangeFlagOffset_ + sizeof(uint32_t) * 2 * MAX_PEERS + 64;    // then the flags, then this rank's own partial mix
        exchangeOwnOffset_ = (exchangeOwnOffset_ + 255) & ~(size_t) 255;
        exchangeBytes_ = exchangeOwnOffset_ + sizeof(float) * stride;
        if (!cuda(cudaMalloc(&dExchange_, exchangeBytes_), "cudaMalloc exchange buffer")) return rc::CudaError;
        if (!cuda(cudaMemset(dExchange_, 0, exchangeBytes_), "memset exchange buffer")) return rc::CudaError;
        if (!cuda(cudaMalloc((void**) &dPeerStatus_, sizeof(int)), "cudaMalloc peer status")) return rc::CudaError;
        if (!cuda(cudaMemset(dPeerStatus_, 0, sizeof(int)), "memset peer status")) return rc::CudaError;
    }
    cudaIpcMemHandle_t h;
    if (!cuda(cudaIpcGetMemHandle(&h, dExchange_), "cudaIpcGetMemHandle")) return rc::CudaError;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    std::memcpy(handleOut64, &h, 64);
    return rc::Ok;
}

int Engine::peerAttach(int rank, int world, const void* handles) {
    Lock lk(mu_);
    if (planOnly_) return fail(rc::CudaError, "plan-only runtime cannot attach peers");
    if (world < 1 || world > MAX_PEERS || rank < 0 || rank >= world || !dExchange_) return fail(rc::BadArgument, "peerAttach: bad rank/world, or peerExport was not called");
    dsetdev();
    peer_ = PeerMix{};
    peer_.rank = rank; peer_.world = world; peer_.stride = MAX_OUT_CHANNELS * blockSize_;
    for (int p = 0; p < world; ++p) {
        void* base = dExchange_;
        if (p != rank) {
            cudaIpcMemHandle_t h;
            std::memcpy(&h, static_cast<const char*>(handles) + (size_t) p * 64, 64);
            if (!cuda(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle (is peer access available between the GPUs?)")) return rc::CudaError;
            peerMapped_.push_back(base);
        }
        peer_.slot[p] = static_cast<uint2*>(base);
        peer_.flag[p] = reinterpret_cast<uint32_t*>(static_cast<char*>(base) + exchangeFlagOffset_);
        if (p == rank) peer_.own = reinterpret_cast<float*>(static_cast<char*>(base) + exchangeOwnOffset_);
    }
    peerAttached_ = true;
    peerEpoch_ = 0;
    return rc::Ok;
}

int Engine::peerStatus() {
    Lock lk(mu_);
    if (!dPeerStatus_) return 0;
    int st = 0;
    cudaStreamSynchronize(stream_);
    cudaMemcpy(&st, dPeerStatus_, sizeof(int), cudaMemcpyDeviceToHost);
    return st;
}

// ---------------------------------------------------------------------------------------------------------
// Runtime::processQueuedEvents (Runtime.h:438-446) -> GraphRenderSequence::processQueuedEvents (:296-304) ->
// RootRenderSequence::processQueuedEvents (:189-198): for every root sub-sequence whose root has active == true, every
// node's processEvents() in render order.  Here the per-voice records the kernel left in HBM are read back and
// turned into the same event objects, one per voice, as JSON text with the reference's keys plus "voice".
static std::string jsonString(const std::string& s) {
    std::string o = "\"";
    for (unsigned char ch : s) {
        if (ch == '"' || ch == '\\') { o += '\\'; o += (char) ch; }
        else if (ch < 0x20) { char b[8]; std::snprintf(b, sizeof b, "\\u%04x", ch); o += b; }
        else o += (char) ch;
    }
    return o + "\"";
}
static std::string jsonNumber(float f) {
    if (!std::isfinite(f)) return "null";                 // nlohmann::json dumps non-finite numbers as null (JSON.h:175-179)
    char b[40];
    std::snprintf(b, sizeof b, "%.9g", (double) f);
    return b;
}
static std::string sourceOf(const Node& n) {              // getPropertyWithDefault("name", js::Value()) — undefined serialises as null
    auto it = n.props.find("name");
    if (it == n.props.end() || !it->second.isString()) return "null";
    return jsonString(it->second.asString());
}
static void appendFloatArray(std::string& o, const float* d, size_t n) {
    o += '[';
    for (size_t i = 0; i < n; ++i) { if (i) o += ", "; o += jsonNumber(d[i]); }
    o += ']';
}

// AudioFFT::fft semantics (wasm/FFTConvolver/AudioFFT.cpp:132-155): n real float samples -> n/2+1 bins, the transform itself in
// double (the reference runs Ooura's rdft in double), Im of bins 0 and n/2 exactly zero.
static void realFftFloatIO(const std::vector<float>& x, std::vector<float>& re, std::vector<float>& im) {
    const size_t n = x.size();
    std::vector<double> ar(x.begin(), x.end()), ai(n, 0.0);
    for (size_t i = 1, j = 0; i < n; ++i) {
        size_t bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) { std::swap(ar[i], ar[j]); std::swap(ai[i], ai[j]); }
    }
    for (size_t len = 2; len <= n; len <<= 1) {
        const double ang = -2.0 * M_PI / (double) len;
        for (size_t k = 0; k < len / 2; ++k) {
            const double wr = std::cos(ang * (double) k), wi = std::sin(ang * (double) k);
            for (size_t i = k; i < n; i += len) {
                const size_t j = i + len / 2;
                const double xr = ar[j] * wr - ai[j] * wi, xi = ar[j] * wi + ai[j] * wr;
                ar[j] = ar[i] - xr; ai[j] = ai[i] - xi;
                ar[i] += xr; ai[i] += xi;
            }
        }
    }
    for (size_t k = 0; k <= n / 2; ++k) { re[k] = (float) ar[k]; im[k] = (float) ai[k]; }
    im[0] = 0.0f; im[n / 2] = 0.0f;
}

static double numProp(const Node& n, const char* k, double d) {
    auto it = n.props.find(k);
    return (it != n.props.end() && it->second.isNumber()) ? it->second.asNumber() : d;
}
// scope / fft: the window a poll reads (Analyzers.h:203-251 `size`, wasm/FFT.h:49-62) and the ring channels it holds
static void windowShape(const Node& n, uint32_t& size, int& nch) {
    if (n.kind == NodeKind::Scope) {
        size = (uint32_t) (size_t) numProp(n, "size", 512);
        nch = (int) std::min((size_t) numProp(n, "channels", 1), (size_t) SCOPE_CHANNELS);
    } else { size = (uint32_t) n.window.size(); nch = 1; }
}
static int ringChannels(const Node& n) { return n.kind == NodeKind::Scope ? SCOPE_CHANNELS : 1; }

// Where a poll reads the device state it reports, in the layouts of kernels.h EventLogItem.  null: a CUDA error (lastError_ is set).
struct Engine::PollSource {
    virtual ~PollSource() = default;
    virtual const uint32_t* rows(const PollItem& it, int first) = 0;   // state rows first .. first + 2 of voices [b, e): [3][e - b] words
    virtual const float* capture(const PollItem& it, int vi, uint32_t r, uint32_t avail) = 0;   // ring samples [r, r + avail) of voice b + vi
    virtual const float* window(const PollItem& it, int tile, int ch) = 0;   // [size][L] floats of ring channel ch of `tile` from it.r
};

// A live poll: device memory, read after the render stream was synchronised.
struct Engine::DeviceSource : Engine::PollSource {
    Engine& E;
    bool hideReady = false;   // report no relay flags (the backlog an offline render with events reads first)
    std::vector<uint32_t> rowBuf;
    std::vector<float> col, win[SCOPE_CHANNELS];
    explicit DeviceSource(Engine& e) : E(e) {}
    const uint32_t* rows(const PollItem& it, int first) override {
        const Group& g = *it.g;
        const size_t n = (size_t) (it.e - it.b);
        rowBuf.resize(3 * n);
        if (!E.cuda(cudaMemcpy2D(rowBuf.data(), sizeof(uint32_t) * n, g.dRows + (size_t) (it.n->stateRow + first) * g.Vpad + it.b, sizeof(uint32_t) * g.Vpad,
                                 sizeof(uint32_t) * n, 3, cudaMemcpyDeviceToHost), "read event rows")) return nullptr;
        if (hideReady) std::fill(rowBuf.begin() + 2 * n, rowBuf.end(), 0u);
        return rowBuf.data();
    }
    const float* capture(const PollItem& it, int vi, uint32_t r, uint32_t avail) override {
        const Node& n = *it.n;
        const int L = it.g->tileWidth, v = it.b + vi;
        const uint32_t cap = (uint32_t) (n.size - CAPTURE_SCRATCH);
        const float* base = n.ring + (size_t) (v / L) * (size_t) n.size * L + (v % L);
        col.resize(avail);
        const uint32_t first = std::min(avail, cap - r);
        if (!E.cuda(cudaMemcpy2D(col.data(), sizeof(float), base + (size_t) r * L, sizeof(float) * L, sizeof(float), first, cudaMemcpyDeviceToHost), "read capture ring")) return nullptr;
        if (first < avail && !E.cuda(cudaMemcpy2D(col.data() + first, sizeof(float), base, sizeof(float) * L, sizeof(float), avail - first, cudaMemcpyDeviceToHost), "read capture ring (wrap)")) return nullptr;
        return col.data();
    }
    const float* window(const PollItem& it, int tile, int ch) override {
        // one contiguous [pos][L] slab per (tile, channel), a wrapped read in two pieces
        const int L = it.g->tileWidth;
        const size_t size = it.size, first = std::min(size, (size_t) SCOPE_RING - it.r);
        const float* base = it.n->ring + ((size_t) tile * ringChannels(*it.n) + ch) * SCOPE_RING * L;
        std::vector<float>& slab = win[ch];
        slab.resize(size * L);
        if (!E.cuda(cudaMemcpy(slab.data(), base + (size_t) it.r * L, sizeof(float) * first * L, cudaMemcpyDeviceToHost), "read scope ring")) return nullptr;
        if (first < size && !E.cuda(cudaMemcpy(slab.data() + first * L, base, sizeof(float) * (size - first) * L, cudaMemcpyDeviceToHost), "read scope ring (wrap)")) return nullptr;
        return slab.data();
    }
};

// An offline block's poll: the records K5 left in the chunk's event log (copied to pinned host memory).
struct Engine::LogSource : Engine::PollSource {
    Engine& E;
    const uint32_t* log;
    uint32_t lim;             // capture samples per voice in a record
    LogSource(Engine& e, const uint32_t* l, uint32_t lm) : E(e), log(l), lim(lm) {}
    const uint32_t* rows(const PollItem& it, int) override { return log + it.logOff; }
    const float* capture(const PollItem& it, int vi, uint32_t, uint32_t avail) override {
        if (avail > lim) { E.fail(rc::InvariantViolation, "offline event log: more capture samples in one block than a record holds"); return nullptr; }
        return reinterpret_cast<const float*>(log + it.logOff + 3 * (size_t) (it.e - it.b)) + (size_t) vi * lim;
    }
    const float* window(const PollItem& it, int tile, int ch) override {
        const int L = it.g->tileWidth;
        return reinterpret_cast<const float*>(log + it.logOff) + ((size_t) (tile - it.b / L) * it.nch + ch) * it.size * L;
    }
};

// The walk of a poll (see above): every event node, in render order, of every root sub-sequence whose root has active == true, of the
// sequence process() last used (queued: the one the next process() will use).
template <class F> int Engine::forEachPolled(int vb, int ve, bool queued, F&& f) {
    if (vb < 0) vb = 0;
    if (ve < 0 || ve > numVoices_) ve = numVoices_;
    for (auto& gp : groups_) {
        Group& g = *gp;
        Program* const p = (queued && g.pending) ? g.pending.get() : g.active.get();
        if (!p || p->evNodes.empty()) continue;                         // `if (auto ptr = rtRenderSeq)`
        const int b = std::max(vb, g.v0) - g.v0, e = std::min(ve, g.v0 + g.nv) - g.v0;   // group-relative voice range
        if (b >= e) continue;                                           // the poll does not touch this voice group at all
        for (size_t ri = 0; ri < p->rootIds.size(); ++ri) {
            auto rit = g.nodes.find(p->rootIds[ri]);
            if (rit == g.nodes.end()) continue;
            auto ap = rit->second.props.find("active");                                     // GraphRenderSequence.h:192
            if (ap == rit->second.props.end() || !ap->second.isBool() || !ap->second.asBool()) continue;
            for (auto& ev : p->evNodes) {
                if (ev.root != (int) ri) continue;
                auto nit = g.nodes.find(ev.node);
                if (nit == g.nodes.end()) continue;
                const int r = f(g, nit->second, b, e);
                if (r != rc::Ok) return r;
            }
        }
    }
    return rc::Ok;
}

// The decisions of a poll that are the same for every voice of a group, taken on the host mirrors (which advance like the device rings,
// graph_host.cpp walkGroups): whether a scope / fft window is read, where, and the read position after it; the metro flag.
int Engine::planPoll(int vb, int ve, std::vector<PollItem>& items) {
    return forEachPolled(vb, ve, false, [&](Group& g, Node& n, int b, int e) -> int {
        PollItem it; it.g = &g; it.n = &n; it.b = b; it.e = e;
        switch (n.kind) {
        case NodeKind::Meter: case NodeKind::Snapshot: break;
        case NodeKind::Capture: if (!n.ring) return rc::CudaError; break;
        case NodeKind::Scope: case NodeKind::Fft: {   // Analyzers.h:203-251 (FloatType == float branch), wasm/FFT.h:90-131
            windowShape(n, it.size, it.nch);
            const uint32_t mask = SCOPE_RING - 1, r = n.scopeR, w = n.scopeW;
            const size_t full = (w > r) ? (w - r) : (((uint32_t) SCOPE_RING - (r - w)) & mask);
            // scope: ringBuffer.read once more than `size` samples wait; fft: one windowed transform once `size` samples wait
            const bool fire = n.kind == NodeKind::Scope ? full > it.size : (it.size != 0 && full >= it.size);
            if (!fire || !n.ring) return rc::Ok;
            it.fire = true; it.r = r;
            n.scopeR = (r + it.size) & mask;
        } break;
        case NodeKind::Metro:                         // wasm/Metro.h:58-66
            if (!n.metroFlag) return rc::Ok;
            it.fire = true;
            if (b == 0 && e == g.nv) n.metroFlag = false;      // the flag is one per group: cleared when every voice was served
            break;
        default: return rc::Ok;
        }
        items.push_back(it);
        return rc::Ok;
    });
}

size_t Engine::pollRecordWords(const PollItem& it) const {
    const size_t n = (size_t) (it.e - it.b);
    const int L = it.g->tileWidth;
    switch (it.n->kind) {
    case NodeKind::Meter: case NodeKind::Snapshot: return 3 * n;
    case NodeKind::Capture: return n * (3 + (size_t) blockSize_ + CAPTURE_SCRATCH);
    case NodeKind::Scope: case NodeKind::Fft: return it.fire ? (size_t) ((it.e + L - 1) / L - it.b / L) * it.nch * it.size * L : 0;
    default: return 0;
    }
}

// The events of one planned item, one per voice that has something to report: JSON text with the reference's keys plus "voice".
int Engine::emitPoll(const PollItem& it, PollSource& src, EventFn cb, void* user) {
    Group& g = *it.g;
    Node& n = *it.n;
    const int b = it.b, e = it.e, nv = e - b, L = g.tileWidth;
    const std::string source = sourceOf(n);
    auto asFloat = [](uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; };
    switch (n.kind) {
    case NodeKind::Meter: {            // Analyzers.h:42-60: the latest readout, if the queue shows any
        const uint32_t* rows = src.rows(it, 0);
        if (!rows) return rc::CudaError;
        for (int i = 0; i < nv && cb; ++i) {
            // SingleWriterSingleReaderQueue(32).size() == pushes mod 32 (:77-83,:86-98): a queue that was
            // pushed exactly 32 times since it was drained reads as empty
            if (rows[(size_t) 2 * nv + i] % 32u == 0) continue;
            std::string js = "{\"max\": " + jsonNumber(asFloat(rows[(size_t) nv + i])) + ", \"min\": " + jsonNumber(asFloat(rows[i])) +
                             ", \"source\": " + source + ", \"voice\": " + std::to_string(g.v0 + b + i) + "}";
            cb("meter", js.c_str(), g.v0 + b + i, user);
        }
    } break;
    case NodeKind::Snapshot: {         // Analyzers.h:108-127
        const uint32_t* rows = src.rows(it, 0);
        if (!rows) return rc::CudaError;
        for (int i = 0; i < nv && cb; ++i) {
            if (rows[(size_t) 2 * nv + i] % 32u == 0) continue;
            std::string js = "{\"data\": " + jsonNumber(asFloat(rows[(size_t) nv + i])) + ", \"source\": " + source +
                             ", \"voice\": " + std::to_string(g.v0 + b + i) + "}";
            cb("snapshot", js.c_str(), g.v0 + b + i, user);
        }
    } break;
    case NodeKind::Scope: {            // ringBuffer.read(...) of `size` samples per channel, de-interleaved per voice
        const size_t size = it.size, channels = (size_t) numProp(n, "channels", 1);
        const int t0 = b / L, t1 = (e + L - 1) / L;
        std::vector<float> one(size);
        for (int tile = t0; tile < t1 && cb; ++tile) {
            std::vector<const float*> tileData((size_t) it.nch);
            for (int ch = 0; ch < it.nch; ++ch)
                if (!(tileData[ch] = src.window(it, tile, ch))) return rc::CudaError;
            for (int vl = 0; vl < L; ++vl) {
                const int v = tile * L + vl;
                if (v < b || v >= e) continue;
                std::string js = "{\"data\": [";
                for (size_t ch = 0; ch < channels; ++ch) {
                    if (ch) js += ", ";
                    std::fill(one.begin(), one.end(), 0.0f);   // channels beyond the ring's 4 stay zero like a fresh Float32Array
                    if (ch < tileData.size()) for (size_t i = 0; i < size; ++i) one[i] = tileData[ch][i * L + vl];
                    appendFloatArray(js, one.data(), size);
                }
                js += "], \"source\": " + source + ", \"voice\": " + std::to_string(g.v0 + v) + "}";
                cb("scope", js.c_str(), g.v0 + v, user);
            }
        }
    } break;
    case NodeKind::Fft: {              // wasm/FFT.h:90-131: the window, then the transform on the host
        const size_t size = it.size;
        std::vector<float> x(size), re(size / 2 + 1), im(size / 2 + 1);
        const int t0 = b / L, t1 = (e + L - 1) / L;
        for (int tile = t0; tile < t1 && cb; ++tile) {
            const float* slab = src.window(it, tile, 0);
            if (!slab) return rc::CudaError;
            for (int vl = 0; vl < L; ++vl) {
                const int v = tile * L + vl;
                if (v < b || v >= e) continue;
                for (size_t i = 0; i < size; ++i) x[i] = slab[i * L + vl] * n.window[i];
                realFftFloatIO(x, re, im);
                std::string js = "{\"data\": {\"imag\": ";
                appendFloatArray(js, im.data(), im.size());
                js += ", \"real\": ";
                appendFloatArray(js, re.data(), re.size());
                js += "}, \"source\": " + source + ", \"voice\": " + std::to_string(g.v0 + v) + "}";
                cb("fft", js.c_str(), g.v0 + v, user);
            }
        }
    } break;
    case NodeKind::Capture: {          // Capture.h:60-93: drain the ring into the relay; on relayReady.exchange(false), report and clear it
        const uint32_t* rows = src.rows(it, 2);     // write position, read position, relay-ready flag
        if (!rows) return rc::CudaError;
        const std::vector<uint32_t> hdr(rows, rows + 3 * (size_t) nv);
        const uint32_t cap = (uint32_t) (n.size - CAPTURE_SCRATCH), mask = cap - 1;
        if (n.relay.size() < (size_t) g.nv) n.relay.resize((size_t) g.nv);
        for (int i = 0; i < nv; ++i) {
            const int v = b + i;
            const uint32_t w = hdr[i], r = hdr[(size_t) nv + i];
            const uint32_t avail = (w > r) ? (w - r) : ((cap - (r - w)) & mask);
            if (avail > 0) {
                const float* col = src.capture(it, i, r, avail);
                if (!col) return rc::CudaError;
                n.relay[v].insert(n.relay[v].end(), col, col + avail);
            }
            if (hdr[(size_t) 2 * nv + i]) {
                if (cb) {
                    std::string js = "{\"data\": ";
                    appendFloatArray(js, n.relay[v].data(), n.relay[v].size());
                    js += ", \"source\": " + source + ", \"voice\": " + std::to_string(g.v0 + v) + "}";
                    cb("capture", js.c_str(), g.v0 + v, user);
                }
                n.relay[v].clear();
            }
        }
    } break;
    case NodeKind::Metro: {
        for (int v = b; v < e && cb; ++v) {
            std::string js = "{\"source\": " + source + ", \"voice\": " + std::to_string(g.v0 + v) + "}";
            cb("metro", js.c_str(), g.v0 + v, user);
        }
    } break;
    default: break;
    }
    return rc::Ok;
}

// A live poll's capture side effect on the device: the read position moves to the write position (and the relay flag is cleared).
int Engine::captureConsumed(const PollItem& it, bool clearReady) {
    Group& g = *it.g;
    float* const row = g.dRows + (size_t) it.n->stateRow * g.Vpad + it.b;
    const size_t bytes = sizeof(float) * (size_t) (it.e - it.b);
    if (!cuda(cudaMemcpyAsync(row + (size_t) 3 * g.Vpad, row + (size_t) 2 * g.Vpad, bytes, cudaMemcpyDeviceToDevice, stream_), "write capture positions")) return rc::CudaError;
    if (clearReady && !cuda(cudaMemsetAsync(row + (size_t) 4 * g.Vpad, 0, bytes, stream_), "clear capture relay flags")) return rc::CudaError;
    return rc::Ok;
}

int Engine::processQueuedEvents(int vb, int ve, EventFn cb, void* user) {
    Lock lk(mu_);
    if (planOnly_) return rc::Ok;
    dsetdev();
    std::vector<PollItem> items;
    int r = planPoll(vb, ve, items);
    if (r != rc::Ok || items.empty()) return r;
    if (!cuda(cudaStreamSynchronize(stream_), "sync before events")) return rc::CudaError;
    DeviceSource src(*this);
    for (const PollItem& it : items) {
        if ((r = emitPoll(it, src, cb, user)) != rc::Ok) return r;
        // the poll's side effects on the device (K5 applies the same ones after every block of an offline render with events)
        const Node& n = *it.n;
        if (n.kind == NodeKind::Meter || n.kind == NodeKind::Snapshot) {
            if (!cuda(cudaMemsetAsync(it.g->dRows + (size_t) (n.stateRow + 2) * it.g->Vpad + it.b, 0, sizeof(float) * (it.e - it.b), stream_), "reset readout queue")) return rc::CudaError;
        } else if (n.kind == NodeKind::Capture && (r = captureConsumed(it, true)) != rc::Ok) return r;
    }
    return rc::Ok;
}

// ---------------------------------------------------------------------------------------------------------
// The event log of an offline render with events (Engine::processOfflineEvents, graph_host.cpp offlineLoop).

// Before the first block: the bound on one block's records, and the capture samples that already wait in the rings — read once into the
// relays, as a poll would, without reporting anything, so that a block's record never holds more than that block's samples.
int Engine::eventLogBegin(EventLog& log) {
    log.blockWords = 0;
    std::vector<PollItem> backlog;
    int r = forEachPolled(log.vb, log.ve, true, [&](Group& g, Node& n, int b, int e) -> int {
        PollItem it; it.g = &g; it.n = &n; it.b = b; it.e = e;
        if (n.kind == NodeKind::Scope || n.kind == NodeKind::Fft) {
            windowShape(n, it.size, it.nch);
            it.fire = n.ring && it.size <= (uint32_t) SCOPE_RING;   // a larger window never fills
        }
        if (n.kind == NodeKind::Capture && n.ring) backlog.push_back(it);
        log.blockWords += pollRecordWords(it);
        return rc::Ok;
    });
    if (r != rc::Ok || backlog.empty()) return r;
    if (!cuda(cudaStreamSynchronize(stream_), "sync before reading capture rings")) return rc::CudaError;
    DeviceSource src(*this);
    src.hideReady = true;
    for (const PollItem& it : backlog)
        if ((r = emitPoll(it, src, nullptr, nullptr)) != rc::Ok || (r = captureConsumed(it, false)) != rc::Ok) return r;
    return rc::Ok;
}

// After block inChunk of the chunk in `slot` was enqueued: plan its poll, give every item a record in the chunk's log, and launch K5.
int Engine::eventLogBlock(EventLog& log, int slot, size_t inChunk) {
    if (inChunk == 0) { log.blocks[slot].clear(); log.used[slot] = 0; }
    log.blocks[slot].emplace_back();
    std::vector<PollItem>& items = log.blocks[slot].back();
    int r = planPoll(log.vb, log.ve, items);
    if (r != rc::Ok) return r;
    uint32_t* const base = reinterpret_cast<uint32_t*>(offLog_.dev[slot]);
    EventLogBatch batch;
    batch.n = 0;
    auto flush = [&]() -> bool { return flushEventLog(batch) == rc::Ok; };
    for (PollItem& it : items) {
        it.logOff = log.used[slot];
        const size_t words = pollRecordWords(it);
        if (words == 0) continue;                       // metro: nothing on the device
        log.used[slot] += words;
        if (log.used[slot] > offLog_.devFloats[slot]) return fail(rc::InvariantViolation, "offline event log: a block's records passed their bound");
        const Group& g = *it.g;
        const Node& n = *it.n;
        EventLogItem& d = batch.item[batch.n++];
        d = EventLogItem{};
        d.rows = reinterpret_cast<uint32_t*>(g.dRows + (size_t) n.stateRow * g.Vpad);
        d.ring = n.ring; d.log = base + it.logOff;
        d.b = it.b; d.n = it.e - it.b; d.Vpad = g.Vpad; d.L = g.tileWidth;
        if (n.kind == NodeKind::Meter || n.kind == NodeKind::Snapshot) d.kind = EVLOG_ROWS;
        else if (n.kind == NodeKind::Capture) {
            d.kind = EVLOG_CAPTURE;
            d.cap = (uint32_t) (n.size - CAPTURE_SCRATCH); d.lim = (uint32_t) (blockSize_ + CAPTURE_SCRATCH); d.ringFloats = (uint32_t) n.size;
        } else {
            d.kind = EVLOG_WINDOW;
            d.r = it.r; d.size = it.size; d.ringCh = ringChannels(n); d.nch = it.nch;
            d.t0 = it.b / g.tileWidth; d.t1 = (it.e + g.tileWidth - 1) / g.tileWidth;
        }
        if (batch.n == EVENT_LOG_BATCH && !flush()) return rc::CudaError;
    }
    return flush() ? rc::Ok : rc::CudaError;
}

// One K5 launch of the items gathered in `batch`, which is emptied.
int Engine::flushEventLog(EventLogBatch& batch) {
    if (batch.n == 0) return rc::Ok;
    if (!cuda(launch_event_log(batch, stream_), "event log kernel launch")) return rc::CudaError;
    ++launches_;
    batch.n = 0;
    return rc::Ok;
}

// After the chunk in `slot` was scattered (its log is in pinned memory): its blocks' events, in block order, through the live formatter.
int Engine::eventLogReplay(EventLog& log, int slot, size_t firstBlock) {
    LogSource src(*this, reinterpret_cast<const uint32_t*>(offLog_.pinned[slot]), (uint32_t) (blockSize_ + CAPTURE_SCRATCH));
    struct Relay { BlockEventFn cb; void* user; size_t block; } relay{log.cb, log.user, firstBlock};
    const EventFn toBlock = [](const char* type, const char* json, int, void* u) {
        const Relay* rl = static_cast<const Relay*>(u);
        rl->cb(rl->block, type, json, rl->user);
    };
    for (const std::vector<PollItem>& items : log.blocks[slot]) {
        for (const PollItem& it : items) {
            const int r = emitPoll(it, src, toBlock, &relay);
            if (r != rc::Ok) return r;
        }
        ++relay.block;
    }
    return rc::Ok;
}

// ---------------------------------------------------------------------------------------------------------
// Array polls: the readouts of one meter / snapshot node for a range of voices, written by K5 (EVLOG_READOUT) into dense arrays instead
// of one JSON event per voice.  The rules are those of processQueuedEvents: the voice groups where that poll reaches the node (the
// sequence process() last used, an active root; forEachPolled) report and drain their queues, the others report nothing and keep them.

// The (group, node) pairs a poll of voices [vb, ve) reaches: one walk, shared by every node a call or an offline block polls.
int Engine::readoutPolled(int vb, int ve, PolledSet& out) {
    out.clear();
    return forEachPolled(vb, ve, false, [&](Group& g, Node& n, int, int) -> int {
        out.insert({&g, n.id});
        return rc::Ok;
    });
}

int Engine::readoutEnqueue(int32_t nodeId, const std::vector<VoiceTarget>& targets, const PolledSet& polled, uint32_t* a, uint32_t* b,
                           uint8_t* fresh, EventLogBatch& batch) {
    for (const VoiceTarget& t : targets) {
        EventLogItem& d = batch.item[batch.n++];
        d = EventLogItem{};
        d.kind = EVLOG_READOUT;
        d.b = t.b; d.n = t.e - t.b; d.Vpad = t.g.Vpad; d.L = t.g.tileWidth;
        d.drain = polled.count({&t.g, nodeId}) ? 1 : 0;
        if (d.drain) d.rows = reinterpret_cast<uint32_t*>(t.g.dRows + (size_t) t.n.stateRow * t.g.Vpad);
        d.aRow = t.n.kind == NodeKind::Meter ? 0 : 1;   // meter: rows min, max; snapshot: row 1 is the latched value (emitPoll)
        d.outA = a + t.at;
        d.outB = (b && t.n.kind == NodeKind::Meter) ? b + t.at : nullptr;
        d.fresh = fresh + t.at;
        if (batch.n == EVENT_LOG_BATCH) {
            const int r = flushEventLog(batch);
            if (r != rc::Ok) return r;
        }
    }
    return rc::Ok;
}

// A record of readoutWords(count) words (a, b, fresh bytes) into the caller's arrays: fresh everywhere, a and b where fresh.  b is null
// for a snapshot, whose record carries no b (the caller's b is never written).
static void readoutCopy(const uint32_t* rec, int count, float* a, float* b, uint8_t* fresh) {
    const uint8_t* f = reinterpret_cast<const uint8_t*>(rec + 2 * (size_t) count);
    for (int i = 0; i < count; ++i) {
        fresh[i] = f[i];
        if (!f[i]) continue;
        std::memcpy(a + i, rec + i, 4);
        if (b) std::memcpy(b + i, rec + count + i, 4);
    }
}

int Engine::pollReadouts(int32_t nodeId, int vb, int count, float* a, float* b, uint8_t* fresh, bool device) {
    Lock lk(mu_);
    if (count > 0 && (!a || !fresh)) return fail(rc::BadArgument, "pollReadouts: a or fresh is NULL");
    std::vector<VoiceTarget> targets;
    int r = readoutTargets(nodeId, vb, count, targets);
    if (r != rc::Ok || count == 0) return r;
    if (planOnly_) return fail(rc::CudaError, "plan-only runtime (no CUDA device): there are no readouts to poll");
    dsetdev();
    PolledSet polled;
    if ((r = readoutPolled(vb, vb + count, polled)) != rc::Ok) return r;
    EventLogBatch batch;
    batch.n = 0;
    if (device) {
        if ((r = readoutEnqueue(nodeId, targets, polled, reinterpret_cast<uint32_t*>(a), reinterpret_cast<uint32_t*>(b), fresh, batch)) != rc::Ok) return r;
        return flushEventLog(batch);
    }
    // host arrays: K5 fills a device staging record, which comes down in one copy
    const size_t words = readoutWords(count);
    if (!grow(dReadout_, readoutCap_, words, "cudaMalloc readout staging") ||
        !grow(hReadout_, readoutPinned_, words, "cudaMallocHost readout staging", false, 1, true)) return rc::CudaError;
    if ((r = readoutEnqueue(nodeId, targets, polled, dReadout_, dReadout_ + count, reinterpret_cast<uint8_t*>(dReadout_ + 2 * (size_t) count), batch)) != rc::Ok ||
        (r = flushEventLog(batch)) != rc::Ok) return r;
    if (!cuda(cudaMemcpyAsync(hReadout_, dReadout_, words * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream_), "D2H readouts") ||
        !cuda(cudaStreamSynchronize(stream_), "sync after readouts")) return rc::CudaError;
    readoutCopy(hReadout_, count, a, targets.front().n.kind == NodeKind::Meter ? b : nullptr, fresh);
    return rc::Ok;
}

// After block inChunk of the chunk in `slot` was enqueued: every listed node's poll into the block's records in the chunk's log.
int Engine::readoutBlock(ReadoutLog& ro, int slot, size_t inChunk) {
    const size_t w = readoutWords(ro.count);
    uint32_t* const rec = reinterpret_cast<uint32_t*>(offLog_.dev[slot]) + inChunk * ro.blockWords();
    int r = readoutPolled(ro.vb, ro.vb + ro.count, ro.polled);     // the active program may change at any block: one walk per block
    if (r != rc::Ok) return r;
    EventLogBatch batch;
    batch.n = 0;
    for (size_t j = 0; j < ro.nodes.size(); ++j) {
        uint32_t* const base = rec + j * w;
        r = readoutEnqueue(ro.nodes[j], ro.targets[j], ro.polled, base, base + ro.count, reinterpret_cast<uint8_t*>(base + 2 * (size_t) ro.count), batch);
        if (r != rc::Ok) return r;
    }
    return flushEventLog(batch);
}

void Engine::readoutScatter(const ReadoutLog& ro, const uint32_t* rec, size_t block) {
    const size_t w = readoutWords(ro.count);
    for (size_t j = 0; j < ro.nodes.size(); ++j) {
        const size_t at = (j * ro.numBlocks + block) * (size_t) ro.count;
        const bool meter = ro.targets[j].front().n.kind == NodeKind::Meter;   // every group has the same kind (readoutTargets)
        readoutCopy(rec + j * w, ro.count, ro.a + at, ro.b && meter ? ro.b + at : nullptr, ro.fresh + at);
    }
}

} // namespace eb
