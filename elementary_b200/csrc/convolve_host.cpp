// convolve_host.cpp — host side of K3: impulse-response partitioning, the IR spectra bank and device state of the convolver.
#include "convolve.h"

#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdlib>
#include <cstring>

namespace eb {

namespace {

void freeDev(void* p, bool plan) { if (!p) return; if (plan) std::free(p); else cudaFree(p); }

bool allocDev(void** p, size_t bytes, bool plan, cudaStream_t stream, std::string& err) {
    if (plan) { *p = std::calloc(1, bytes ? bytes : 1); if (!*p) { err = "out of host memory"; return false; } return true; }
    cudaError_t e = cudaMalloc(p, bytes ? bytes : 1);
    if (e != cudaSuccess) { err = std::string("cudaMalloc convolver: ") + cudaGetErrorString(e); return false; }
    e = cudaMemsetAsync(*p, 0, bytes, stream);
    if (e != cudaSuccess) { err = std::string("cudaMemset convolver: ") + cudaGetErrorString(e); return false; }
    return true;
}

bool zeroDev(void* p, size_t bytes, bool plan, cudaStream_t stream, std::string& err) {
    if (!p || !bytes) return true;
    if (plan) { std::memset(p, 0, bytes); return true; }
    if (cudaMemsetAsync(p, 0, bytes, stream) != cudaSuccess) { err = "convolver reset failed"; return false; }
    return true;
}

// host -> device from a pageable temporary: cudaMemcpyAsync returns once the source is staged (CUDA runtime API, "API
// synchronization behavior"), and the copy is ordered behind every kernel already queued on the stream that reads the old contents
bool uploadDev(void* dst, const void* src, size_t bytes, bool plan, cudaStream_t stream, std::string& err) {
    if (!bytes) return true;
    if (plan) { std::memcpy(dst, src, bytes); return true; }
    if (cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream) != cudaSuccess) { err = "convolver table upload failed"; return false; }
    return true;
}

// In-place iterative radix-2 FFT in double (host, init time only): spectra of the IR partitions are computed in
// double like the reference's OouraFFT (AudioFFT.cpp:132-155) and rounded to float once.
void fftDouble(std::vector<std::complex<double>>& a) {
    const size_t n = a.size();
    for (size_t i = 1, j = 0; i < n; ++i) {
        size_t bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) std::swap(a[i], a[j]);
    }
    for (size_t len = 2; len <= n; len <<= 1) {
        const double ang = -2.0 * M_PI / (double) len;
        for (size_t i = 0; i < n; i += len)
            for (size_t k = 0; k < len / 2; ++k) {
                const std::complex<double> w(std::cos(ang * (double) k), std::sin(ang * (double) k));
                const std::complex<double> u = a[i + k], v = a[i + k + len / 2] * w;
                a[i + k] = u + v;
                a[i + k + len / 2] = u - v;
            }
    }
}

bool computeSpectra(IrSpectra& s, const float* ir, size_t irLen, bool planOnly, cudaStream_t stream, std::string& err) {
    s.planOnly = planOnly;
    // FFTConvolver.cpp:94-98 / TwoStageFFTConvolver.cpp:93-97: trailing taps below 1e-6 are dropped
    while (irLen > 0 && std::fabs(ir[irLen - 1]) < 0.000001f) --irLen;
    s.partitions = (int) ((irLen + CONV_BLOCK - 1) / CONV_BLOCK);
    if (s.partitions == 0) return true;
    const int S = s.partitions;
    std::vector<float2> H((size_t) S * CONV_PACKED_BINS);
    std::vector<std::complex<double>> buf(CONV_FFT);
    for (int i = 0; i < S; ++i) {
        for (int k = 0; k < CONV_FFT; ++k) {
            const size_t idx = (size_t) i * CONV_BLOCK + k;
            buf[k] = (k < CONV_BLOCK && idx < irLen) ? std::complex<double>((double) ir[idx], 0.0) : std::complex<double>(0.0, 0.0);
        }
        fftDouble(buf);
        for (int b = 1; b < CONV_PACKED_BINS; ++b) H[(size_t) i * CONV_PACKED_BINS + b] = make_float2((float) buf[b].real(), (float) buf[b].imag());
        H[(size_t) i * CONV_PACKED_BINS] = make_float2((float) buf[0].real(), (float) buf[CONV_BLOCK].real());   // packed (H[0], H[512])
    }
    if (!allocDev((void**) &s.dH, H.size() * sizeof(float2), planOnly, stream, err)) return false;
    if (planOnly) { std::memcpy(s.dH, H.data(), H.size() * sizeof(float2)); return true; }
    cudaError_t e = cudaMemcpyAsync(s.dH, H.data(), H.size() * sizeof(float2), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);   // H is a pageable temporary
    if (e != cudaSuccess) { err = std::string("convolver upload: ") + cudaGetErrorString(e); return false; }
    return true;
}

void reclaim(ConvolverState& st, bool wait) {
    for (auto it = st.retired.begin(); it != st.retired.end();) {
        if (it->first && !wait && cudaEventQuery(it->first) == cudaErrorNotReady) { ++it; continue; }
        if (it->first) { cudaEventSynchronize(it->first); cudaEventDestroy(it->first); }
        freeDev(it->second, st.planOnly);
        it = st.retired.erase(it);
    }
}

// The per-channel state besides the ring exists once some channel has a non-empty IR.
bool ensureChannelBuffers(ConvolverState& st, cudaStream_t stream, std::string& err) {
    if (st.dYpre || st.nv == 0) return true;
    const size_t nv = (size_t) st.nv;
    return allocDev((void**) &st.dYpre, nv * CONV_PACKED_BINS * sizeof(float2), st.planOnly, stream, err) &&
           allocDev((void**) &st.dOverlap, nv * CONV_BLOCK * sizeof(float), st.planOnly, stream, err) &&
           allocDev((void**) &st.dInBuf, nv * CONV_BLOCK * sizeof(float), st.planOnly, stream, err);
}

// irs / maxS from chIr; in the per-channel form also the descriptors and the unit table: channels ordered by IR (first use), so that
// consecutive channels — the two of a unit — share one IR wherever the assignment allows
bool rebuildTables(ConvolverState& st, cudaStream_t stream, std::string& err) {
    st.irs.clear();
    st.maxS = 0;
    std::map<const IrSpectra*, int> order;
    std::vector<int> chOrder((size_t) st.nv);
    for (int c = 0; c < st.nv; ++c) {
        const IrSpectra* s = st.chIr[(size_t) c].get();
        auto ins = order.emplace(s, (int) st.irs.size());
        if (ins.second) { st.irs.push_back(st.chIr[(size_t) c]); st.maxS = std::max(st.maxS, s->partitions); }
        chOrder[(size_t) c] = ins.first->second;
    }
    if (!st.perChannel()) return true;
    std::vector<ConvChannel> desc((size_t) st.nv);
    for (int c = 0; c < st.nv; ++c) desc[(size_t) c] = ConvChannel{st.chIr[(size_t) c]->dH, st.chIr[(size_t) c]->partitions, 0};
    std::vector<int> byIr((size_t) st.nv);
    for (int c = 0; c < st.nv; ++c) byIr[(size_t) c] = c;
    std::stable_sort(byIr.begin(), byIr.end(), [&](int a, int b) { return chOrder[(size_t) a] < chOrder[(size_t) b]; });
    const int units = (st.nv + CONV_CH_PER_CTA - 1) / CONV_CH_PER_CTA;
    std::vector<int4> ut((size_t) units);
    for (int u = 0; u < units; ++u) {
        const int a = byIr[(size_t) 2 * u], b = 2 * u + 1 < st.nv ? byIr[(size_t) 2 * u + 1] : -1;
        const int Sa = desc[(size_t) a].S, Sb = b >= 0 ? desc[(size_t) b].S : 0;
        ut[(size_t) u] = make_int4(a, b, std::max(Sa, Sb), (b < 0 || st.chIr[(size_t) a] == st.chIr[(size_t) b]) ? 1 : 0);
    }
    if (!st.dChan && !allocDev((void**) &st.dChan, (size_t) st.nv * sizeof(ConvChannel), st.planOnly, stream, err)) return false;
    if (!st.dUnits && !allocDev((void**) &st.dUnits, (size_t) units * sizeof(int4), st.planOnly, stream, err)) return false;
    return uploadDev(st.dChan, desc.data(), desc.size() * sizeof(ConvChannel), st.planOnly, stream, err) &&
           uploadDev(st.dUnits, ut.data(), ut.size() * sizeof(int4), st.planOnly, stream, err);
}

} // namespace

IrSpectra::~IrSpectra() { freeDev(dH, planOnly); }

std::shared_ptr<IrSpectra> IrBank::acquire(const void* key, const std::weak_ptr<const void>& owner, const float* ir, size_t irLen,
                                           bool planOnly, cudaStream_t stream, std::string& err) {
    for (auto it = entries_.begin(); it != entries_.end();) {   // entries nobody uses any more
        if (it->second.spectra.expired()) it = entries_.erase(it); else ++it;
    }
    auto it = entries_.find(key);
    if (it != entries_.end() && !it->second.owner.expired() &&
        !it->second.owner.owner_before(owner) && !owner.owner_before(it->second.owner)) {
        if (auto sp = it->second.spectra.lock()) return sp;
    }
    auto sp = std::make_shared<IrSpectra>();
    if (!computeSpectra(*sp, ir, irLen, planOnly, stream, err)) return nullptr;
    entries_[key] = Entry{owner, sp};
    return sp;
}

size_t IrBank::live() const {
    size_t n = 0;
    for (auto& kv : entries_) if (!kv.second.spectra.expired()) ++n;
    return n;
}

ConvolverState::~ConvolverState() {
    reclaim(*this, true);
    freeDev(dFdl, planOnly); freeDev(dYpre, planOnly); freeDev(dOverlap, planOnly); freeDev(dInBuf, planOnly); freeDev(dTw, planOnly);
    freeDev(dChan, planOnly); freeDev(dUnits, planOnly);
}

bool convolver_init(ConvolverState& st, IrBank& bank, const void* key, const std::weak_ptr<const void>& owner, const float* ir, size_t irLen,
                    int nv, bool planOnly, cudaStream_t stream, std::string& err) {
    st.planOnly = planOnly;
    st.nv = nv;
    st.cur = 0;
    st.fill = 0;
    auto h = bank.acquire(key, owner, ir, irLen, planOnly, stream, err);
    if (!h) return false;
    st.chIr.assign((size_t) nv, h);
    st.partitions = h->partitions;
    std::vector<float2> tw(512);
    for (int m = 0; m < 512; ++m) {
        const double a = -2.0 * M_PI * (double) m / 1024.0;
        tw[m] = make_float2((float) std::cos(a), (float) std::sin(a));
    }
    if (!allocDev((void**) &st.dTw, tw.size() * sizeof(float2), planOnly, stream, err)) return false;
    if (st.partitions > 0) {
        if (!allocDev((void**) &st.dFdl, (size_t) nv * st.partitions * CONV_PACKED_BINS * sizeof(float2), planOnly, stream, err)) return false;
        if (!ensureChannelBuffers(st, stream, err)) return false;
    }
    if (!rebuildTables(st, stream, err)) return false;
    if (planOnly) { std::memcpy(st.dTw, tw.data(), tw.size() * sizeof(float2)); return true; }
    cudaError_t e = cudaMemcpyAsync(st.dTw, tw.data(), tw.size() * sizeof(float2), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);   // tw is a pageable temporary
    if (e != cudaSuccess) { err = std::string("convolver upload: ") + cudaGetErrorString(e); return false; }
    return true;
}

bool convolver_assign(ConvolverState& st, int c0, int n, const std::vector<std::shared_ptr<IrSpectra>>& h, cudaStream_t stream, std::string& err) {
    reclaim(st, false);
    int R = st.partitions;
    for (auto& s : h) R = std::max(R, s->partitions);
    if (R > st.partitions) {   // grow the ring: newest spectra first in the new layout (cur = 0), the new slots zero
        float2* ring = nullptr;
        const size_t bytes = (size_t) st.nv * R * CONV_PACKED_BINS * sizeof(float2);
        if (st.planOnly) {
            ring = static_cast<float2*>(std::calloc(1, bytes ? bytes : 1));
            if (!ring) { err = "out of host memory"; return false; }
            for (int c = 0; c < st.nv && st.dFdl; ++c)
                for (int i = 0; i < st.partitions; ++i)
                    std::memcpy(ring + ((size_t) c * R + i) * CONV_PACKED_BINS,
                                st.dFdl + ((size_t) c * st.partitions + (st.cur + i) % st.partitions) * CONV_PACKED_BINS, CONV_PACKED_BINS * sizeof(float2));
        } else {
            if (cudaMalloc((void**) &ring, bytes) != cudaSuccess) { err = "cudaMalloc convolver ring"; return false; }
            if (convolver_relayout(ring, st.dFdl, st.nv, st.dFdl ? st.partitions : 0, R, st.cur, stream) != cudaSuccess) {
                cudaFree(ring); err = "convolver ring re-layout failed"; return false;
            }
        }
        if (st.dFdl) {   // kernels queued before this point still read the old ring
            cudaEvent_t ev = nullptr;
            if (!st.planOnly && (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(ev, stream) != cudaSuccess)) {
                cudaFree(ring); err = "convolver ring event failed"; return false;
            }
            st.retired.push_back({ev, st.dFdl});
        }
        st.dFdl = ring;
        st.partitions = R;
        st.cur = 0;
    }
    if (R > 0 && !ensureChannelBuffers(st, stream, err)) return false;
    for (int i = 0; i < n; ++i) st.chIr[(size_t) (c0 + i)] = h[(size_t) i];
    // the addressed channels restart: empty delay line, partial sums, overlap and input buffer
    for (const ConvRegion& r : convolver_channel_regions(st))
        if (!zeroDev(static_cast<char*>(r.base) + (size_t) c0 * r.bytesPerChannel, (size_t) n * r.bytesPerChannel, st.planOnly, stream, err)) return false;
    return rebuildTables(st, stream, err);
}

std::vector<ConvRegion> convolver_channel_regions(const ConvolverState& st) {
    std::vector<ConvRegion> out;
    if (st.dFdl) out.push_back({st.dFdl, (size_t) st.partitions * CONV_PACKED_BINS * sizeof(float2)});
    if (st.dYpre) {
        out.push_back({st.dYpre, CONV_PACKED_BINS * sizeof(float2)});
        out.push_back({st.dOverlap, CONV_BLOCK * sizeof(float)});
        out.push_back({st.dInBuf, CONV_BLOCK * sizeof(float)});
    }
    return out;
}

bool convolver_clone_range(const ConvolverState& src, int c0, int n, ConvolverState& dst, cudaStream_t stream, std::string& err) {
    dst.planOnly = src.planOnly;
    dst.nv = n; dst.partitions = src.partitions; dst.cur = src.cur; dst.fill = src.fill;
    dst.chIr.assign(src.chIr.begin() + c0, src.chIr.begin() + c0 + n);
    const size_t S = (size_t) src.partitions;
    struct Part { void** d; const void* s; size_t bytes; };
    const Part parts[] = {
        {(void**) &dst.dTw, src.dTw, 512 * sizeof(float2)},
        {(void**) &dst.dFdl, src.dFdl ? src.dFdl + (size_t) c0 * S * CONV_PACKED_BINS : nullptr, (size_t) n * S * CONV_PACKED_BINS * sizeof(float2)},
        {(void**) &dst.dYpre, src.dYpre ? src.dYpre + (size_t) c0 * CONV_PACKED_BINS : nullptr, (size_t) n * CONV_PACKED_BINS * sizeof(float2)},
        {(void**) &dst.dOverlap, src.dOverlap ? src.dOverlap + (size_t) c0 * CONV_BLOCK : nullptr, (size_t) n * CONV_BLOCK * sizeof(float)},
        {(void**) &dst.dInBuf, src.dInBuf ? src.dInBuf + (size_t) c0 * CONV_BLOCK : nullptr, (size_t) n * CONV_BLOCK * sizeof(float)},
    };
    for (const Part& p : parts) {
        if (!p.s) continue;
        if (!allocDev(p.d, p.bytes, src.planOnly, stream, err)) return false;
        if (src.planOnly) std::memcpy(*p.d, p.s, p.bytes);
        else if (cudaMemcpyAsync(*p.d, p.s, p.bytes, cudaMemcpyDeviceToDevice, stream) != cudaSuccess) { err = "convolver clone copy failed"; return false; }
    }
    return rebuildTables(dst, stream, err);
}

bool convolver_truncate(ConvolverState& st, int n, cudaStream_t stream, std::string& err) {
    st.nv = n;
    st.chIr.resize((size_t) n);
    return rebuildTables(st, stream, err);
}

} // namespace eb
