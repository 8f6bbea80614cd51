// graph_host.cpp — see graph_host.h.  Reference behaviour mirrored here is cited inline as file:line of
// /root/reference (runtime/elem/...).
#include "graph_host.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstring>
#include <functional>
#include <list>
#include <sstream>
#include <thread>
#include <unordered_set>

#include "convolve.h"
#include "kernels.h"
#include "spec_host.h"

namespace eb {

static inline void cpuRelax() {
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#elif defined(__aarch64__)
    asm volatile("yield" ::: "memory");
#endif
}

// ---------------------------------------------------------------------------------------------------------
// GainFade mirror (helpers/GainFade.h)
static double msToStep(double sr, double ms) { return ms > 1e-6 ? 1.0 / (sr * ms / 1000.0) : 1.0; }   // :10-12

void GainFade::init(double sr) {            // GainFade(sr, 20, 20, 0.0, 1.0)  Core.h:80, GainFade.h:18-24
    current = 0.0f; target = 1.0f; step = 0.0f; inStep = 0.0f; outStep = 0.0f;
    setFadeInMs(sr, 20.0);
    setFadeOutMs(sr, 20.0);
}
void GainFade::setFadeInMs(double sr, double ms) { inStep = (float) msToStep(sr, ms); updateStep(); }              // :74-77
void GainFade::setFadeOutMs(double sr, double ms) { outStep = (float) ((double) -1.0f * msToStep(sr, ms)); updateStep(); }   // :79-82
bool GainFade::settled() const { return std::fabs(target - current) <= 1e-6f; }                                     // :102-104
void GainFade::advance(int n) {                                                                                  // :56-72
    if (current == target) return;
    float v = current + step * (float) n;
    current = v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
}


// ---------------------------------------------------------------------------------------------------------
// Device-memory shims.  In "plan-only" mode (device == -1; used by the CPU test-suite to exercise the host
// logic: instruction interpreter, return codes, gc, compilation) they fall back to host memory so that the
// graph compiler can run without a GPU.  Plan-only engines can NOT render: every process call fails loudly.
static void rawFree(void* p, bool plan) { if (!p) return; if (plan) std::free(p); else cudaFree(p); }

cudaError_t Engine::dmalloc(void** p, size_t bytes) {
    if (planOnly_) { *p = std::calloc(1, bytes ? bytes : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
    return cudaMalloc(p, bytes);
}
void Engine::dfree(void* p) { rawFree(p, planOnly_); }
cudaError_t Engine::dmemset(void* p, int v, size_t bytes) {
    if (planOnly_) { std::memset(p, v, bytes); return cudaSuccess; }
    return cudaMemsetAsync(p, v, bytes, stream_);
}
cudaError_t Engine::dmemcpy(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind) {
    if (planOnly_) { std::memmove(dst, src, bytes); return cudaSuccess; }
    return cudaMemcpyAsync(dst, src, bytes, kind, stream_);
}
cudaError_t Engine::dmemcpySync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind) {
    if (planOnly_) { std::memmove(dst, src, bytes); return cudaSuccess; }
    cudaError_t e = cudaMemcpyAsync(dst, src, bytes, kind, stream_);
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(stream_);
}
cudaError_t Engine::dzeroBlock(float* p, int pitch, size_t rows) {
    if (planOnly_) { for (size_t r = 0; r < rows; ++r) std::memset(p + r * pitch, 0, sizeof(float) * blockSize_); return cudaSuccess; }
    return cudaMemset2DAsync(p, sizeof(float) * pitch, 0, sizeof(float) * blockSize_, rows, stream_);
}
template <typename T> bool Engine::grow(T*& p, size_t& cap, size_t n, const char* what, bool zero, size_t slack, bool pinned) {
    if (n <= cap) return true;
    dsync();
    if (pinned) { if (p) cudaFreeHost(p); }
    else dfree(p);
    p = nullptr; cap = 0;
    const size_t bytes = sizeof(T) * n * slack;
    if (!cuda(pinned ? cudaMallocHost((void**) &p, bytes) : dmalloc((void**) &p, bytes), what)) { p = nullptr; return false; }
    if (zero && !cuda(pinned ? (std::memset(p, 0, bytes), cudaSuccess) : dmemset(p, 0, bytes), what)) return false;
    cap = n * slack;
    return true;
}
template bool Engine::grow<uint32_t>(uint32_t*&, size_t&, size_t, const char*, bool, size_t, bool);   // events_host.cpp: readout staging
void Engine::dsync() { if (!planOnly_ && stream_) cudaStreamSynchronize(stream_); }
void Engine::dsetdev() { if (!planOnly_) cudaSetDevice(device_); }
void Engine::setStream(cudaStream_t s) {
    Lock lk(mu_);
    if (planOnly_) return;
    if (ownStream_ && stream_) { cudaStreamSynchronize(stream_); cudaStreamDestroy(stream_); }
    stream_ = s; ownStream_ = false;
}

// ---------------------------------------------------------------------------------------------------------
Program::~Program() {
    if (dCode) rawFree(dCode, planOnly);      // stateMap / paramMap live in the same allocation
    for (float* p : blockBuffers) rawFree(p, planOnly);
}

DeviceArray::~DeviceArray() { if (d) rawFree(d, planOnly); }

struct TypeInfo { NodeKind kind; uint32_t fn; int stateRows; int doubleRows; };   // doubleRows: the leading state rows that are double pairs

// Registered builtin names: DefaultNodeTypes.h:53-143 (+ "convolve", "metro", "time": wasm/Main.cpp:47-61).  Types that
// are out of scope (SURVEY.md §2d: sampleseq, sampleseq2, mc.*) are deliberately absent and yield UnknownNodeType like any
// unregistered name (Runtime.h:304-305).
static const std::unordered_map<std::string, TypeInfo>& typeTable() {
    static const std::unordered_map<std::string, TypeInfo> t = {
        {"in", {NodeKind::In, 0, 0, 0}},
        {"sin", {NodeKind::Unary, F_SIN, 0, 0}}, {"cos", {NodeKind::Unary, F_COS, 0, 0}},
        {"tan", {NodeKind::Unary, F_TAN, 0, 0}}, {"tanh", {NodeKind::Unary, F_TANH, 0, 0}},
        {"asinh", {NodeKind::Unary, F_ASINH, 0, 0}}, {"ln", {NodeKind::Unary, F_LN, 0, 0}},
        {"log", {NodeKind::Unary, F_LOG10, 0, 0}}, {"log2", {NodeKind::Unary, F_LOG2, 0, 0}},
        {"ceil", {NodeKind::Unary, F_CEIL, 0, 0}}, {"floor", {NodeKind::Unary, F_FLOOR, 0, 0}},
        {"round", {NodeKind::Unary, F_ROUND, 0, 0}}, {"sqrt", {NodeKind::Unary, F_SQRT, 0, 0}},
        {"exp", {NodeKind::Unary, F_EXP, 0, 0}}, {"abs", {NodeKind::Unary, F_ABS, 0, 0}},
        {"le", {NodeKind::Binary, F_LE, 0, 0}}, {"leq", {NodeKind::Binary, F_LEQ, 0, 0}},
        {"ge", {NodeKind::Binary, F_GE, 0, 0}}, {"geq", {NodeKind::Binary, F_GEQ, 0, 0}},
        {"pow", {NodeKind::Binary, F_POW, 0, 0}}, {"eq", {NodeKind::Binary, F_EQ, 0, 0}},
        {"and", {NodeKind::Binary, F_AND, 0, 0}}, {"or", {NodeKind::Binary, F_OR, 0, 0}},
        {"add", {NodeKind::Reduce, F_ADD, 0, 0}}, {"sub", {NodeKind::Reduce, F_SUB, 0, 0}},
        {"mul", {NodeKind::Reduce, F_MUL, 0, 0}}, {"div", {NodeKind::Reduce, F_DIV, 0, 0}},
        {"mod", {NodeKind::Reduce, F_MOD, 0, 0}}, {"min", {NodeKind::Reduce, F_MIN, 0, 0}},
        {"max", {NodeKind::Reduce, F_MAX, 0, 0}},
        {"root", {NodeKind::Root, 0, 0, 0}}, {"const", {NodeKind::Const, 0, 0, 0}},
        {"sr", {NodeKind::Sr, 0, 0, 0}},
        {"phasor", {NodeKind::Phasor, 0, 1, 0}}, {"sphasor", {NodeKind::SPhasor, 0, 2, 0}},
        {"counter", {NodeKind::Counter, 0, 1, 0}}, {"accum", {NodeKind::Accum, 0, 2, 0}},
        {"latch", {NodeKind::Latch, 0, 2, 0}}, {"maxhold", {NodeKind::MaxHold, 0, 3, 0}},
        {"rand", {NodeKind::Rand, 0, 1, 0}},
        {"delay", {NodeKind::Delay, 0, 1, 0}}, {"sdelay", {NodeKind::SDelay, 0, 1, 0}},
        {"z", {NodeKind::Z, 0, 1, 0}},
        {"pole", {NodeKind::Pole, 0, 1, 0}}, {"env", {NodeKind::Env, 0, 1, 0}},
        {"biquad", {NodeKind::Biquad, 0, 2, 0}}, {"prewarp", {NodeKind::Prewarp, 0, 0, 0}},
        {"mm1p", {NodeKind::MM1p, 0, 2, 2}}, {"svf", {NodeKind::Svf, 0, 4, 4}},
        {"svfshelf", {NodeKind::SvfShelf, 0, 4, 4}},
        {"tapIn", {NodeKind::TapIn, 0, 0, 0}}, {"tapOut", {NodeKind::TapOut, 0, 0, 0}},
        {"table", {NodeKind::Table, 0, 0, 0}},
        {"blepsaw", {NodeKind::Blep, 0, 2, 0}}, {"blepsquare", {NodeKind::Blep, 1, 2, 0}},
        {"bleptriangle", {NodeKind::Blep, 2, 2, 0}},
        {"convolve", {NodeKind::Convolve, 0, 0, 0}},
        {"once", {NodeKind::Once, 0, 4, 0}}, {"seq", {NodeKind::Seq, 0, 6, 0}},
        {"seq2", {NodeKind::Seq2, 0, 3, 0}}, {"sparseq", {NodeKind::SparSeq, 0, 13, 0}},
        {"sparseq2", {NodeKind::SparSeq2, 0, 3, 0}},
        {"time", {NodeKind::Time, 0, 0, 0}}, {"metro", {NodeKind::Metro, 0, 0, 0}},
        {"meter", {NodeKind::Meter, 0, 3, 0}}, {"snapshot", {NodeKind::Snapshot, 0, 3, 0}},
        {"scope", {NodeKind::Scope, 0, 0, 0}}, {"capture", {NodeKind::Capture, 0, 5, 0}},
        {"fft", {NodeKind::Fft, 0, 0, 0}},
        {"sample", {NodeKind::Sample, 0, 10, 4}},   // two reader positions (double), gains, change.lastIn, currentReader
    };
    return t;
}

// Per-voice parameter rows after Node::paramRow, as the render kernel reads them: sample (ctl_sample, render_kernel.cu) and the seq
// family with its voices' own sequences (ctl_seq_src).  Both begin with the array a voice reads (VoiceArray): its device address, low
// and high word, and a length word — a sample's numSamples + 1 (0: no buffer), a sequence's count.
constexpr int ARRAY_ROWS = 3;
constexpr int SAMPLE_START_OFFSET = 3, SAMPLE_STOP_OFFSET = 4, SAMPLE_PARAM_ROWS = 5;
constexpr int SEQ_GEN = 3, SEQ_PARAM_ROWS = 4;
// sample state rows (ctl_sample): the two readers' positions (double row pairs), then their target gains and gains, interleaved
constexpr int SAMPLE_POS0 = 0, SAMPLE_POS1 = 2, SAMPLE_TARGET_GAIN0 = 4, SAMPLE_TARGET_GAIN1 = 6, SAMPLE_GAINS_END = 8;

struct VoiceArray { std::shared_ptr<const void> hold; uint64_t ptr = 0; uint32_t len = 0; };
// What a per-voice call on voices [vb, vb + count) touches in one voice group: the node, its voices [b, e) there (group-relative), and
// `at`, the index of voice b in the call's per-voice arrays.  snapshot() reports the value set for voice last(), the highest addressed.
static bool voiceRangeOk(int vb, int count, int numVoices) { return vb >= 0 && count >= 0 && vb <= numVoices - count; }   // cannot overflow
static VoiceArray seqArray(const std::shared_ptr<DeviceArray>& a) {
    return a ? VoiceArray{a, (uint64_t) (uintptr_t) a->d, (uint32_t) a->count} : VoiceArray{};
}

// The props a per-voice call may set without cutting the voice group — setPropertyPerVoice, and JSON batches made of nothing else
// (isValueOnlyBatch): the row a value goes to (n.*base + row, and with `shadow` the node's shadow row) and its row bits.  once.arm is
// JSON-only, a bool (no bits): it can arm but never disarm, which a table of per-voice values cannot express.
struct PerVoiceProp {
    NodeKind kind; const char* key;
    using NodeRow = int Node::*;
    NodeRow base; int row; bool shadow;
    bool (*bits)(double v, uint32_t& out);   // false: the value is invalid (InvalidPropertyValue)
};
static bool floatBits(double v, uint32_t& out) { const float f = (float) v; std::memcpy(&out, &f, 4); return true; }
static bool seedBits(double v, uint32_t& out) { out = static_cast<uint32_t>(v); return true; }
static bool offsetBits(double v, uint32_t& out) { out = (uint32_t) static_cast<int>(v); return static_cast<int>(v) >= 0; }   // Sample.h:56,69
static const PerVoiceProp* perVoiceProp(NodeKind kind, const std::string& key) {
    static const PerVoiceProp props[] = {
        {NodeKind::Const, "value", &Node::paramRow, 0, false, floatBits},
        {NodeKind::Rand, "seed", &Node::stateRow, 0, true, seedBits},
        {NodeKind::Once, "arm", &Node::stateRow, 0, true, nullptr},
        {NodeKind::Sample, "startOffset", &Node::paramRow, SAMPLE_START_OFFSET, false, offsetBits},
        {NodeKind::Sample, "stopOffset", &Node::paramRow, SAMPLE_STOP_OFFSET, false, offsetBits},
    };
    for (const auto& p : props)
        if (p.kind == kind && key == p.key) return &p;
    return nullptr;
}

// Fresh state, the one definition of what a node holds right after creation: createNode writes it, compile writes a delay's again
// when its ring is (re)allocated, and resetVoices restores it.  State row k of a node of this kind starts as freshRowBits(kind, k);
// row shadowedRow(kind) (-1: none) is a prop the reference sets per instance (rand.seed, once.arm), restored from the node's shadow
// row, which holds the value last set for each voice.  Rings, tap buffers and convolver state start at zero.
static uint32_t freshRowBits(NodeKind kind, int k) {
    if (kind == NodeKind::SparSeq && (k == 2 || k == 5 || k == 6)) return 0xFFFFFFFFu;   // SparSeq.h:353,342-345: edgeCount = -1, loopPoints = {-1, -1}
    return 0u;                                                                          // everything else, a delay's write index included
}
static int shadowedRow(NodeKind kind) { return (kind == NodeKind::Rand || kind == NodeKind::Once) ? 0 : -1; }

static int bitceil(int n) {   // helpers/BitUtils.h:9
    if ((n & (n - 1)) == 0) return n;
    int o = 1;
    while (o < n) o <<= 1;
    return o;
}

// ---------------------------------------------------------------------------------------------------------
Engine::Engine(double sampleRate, int blockSize, int numVoices, int device)
    : sr_(sampleRate), blockSize_(blockSize), numVoices_(numVoices), device_(device) {
    if (numVoices_ < 1) numVoices_ = 1;
    planOnly_ = device_ < 0;
    if (!planOnly_) {
        cuda(cudaSetDevice(device_), "cudaSetDevice");
        cuda(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking), "cudaStreamCreate");
        int sms = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device_) == cudaSuccess && sms > 0) smCount_ = sms;
        else cudaGetLastError();
    }
    auto g = std::make_unique<Group>();
    g->v0 = 0; g->nv = numVoices_; g->Vpad = (numVoices_ + 31) / 32 * 32;
    groups_.push_back(std::move(g));
    grow(dMix_, mixFloats_, (size_t) MAX_OUT_CHANNELS * blockSize_, "cudaMalloc mix", true);
    if (!planOnly_) {
        const size_t tick = (size_t) MAX_OUT_CHANNELS * ((blockSize_ + 31) / 32);
        cuda(cudaMalloc((void**) &dMixScratch_, sizeof(float) * MIX_REDUCE_MAX_GROUPS * MAX_OUT_CHANNELS * blockSize_), "cudaMalloc mix scratch");
        cuda(cudaMalloc((void**) &dMixTickets_, sizeof(unsigned int) * tick), "cudaMalloc mix tickets");
        if (dMixTickets_) cuda(cudaMemsetAsync(dMixTickets_, 0, sizeof(unsigned int) * tick, stream_), "memset mix tickets");
        // the fast hand-over of the mix bus (HostDeliver) needs both; a failure here only disables it
        if (cudaMalloc((void**) &dDeliverDone_, sizeof(unsigned int)) == cudaSuccess) { cudaMemsetAsync(dDeliverDone_, 0, sizeof(unsigned int), stream_); allocMixHost(); }
        else { dDeliverDone_ = nullptr; cudaGetLastError(); }
    }
}

// The mapped pinned copy of the mix bus, mixFloats_ floats, and the sequence word behind it (HostDeliver).  A failure only disables the
// fast hand-over: hMixHost_ stays null.
void Engine::allocMixHost() {
    if (hMixHost_) cudaFreeHost(hMixHost_);
    hMixHost_ = nullptr; hMixFlag_ = nullptr; dMixHostAlias_ = nullptr; dMixFlagAlias_ = nullptr;
    const size_t bytes = sizeof(float) * mixFloats_ + 64;
    void* d = nullptr;
    if (cudaHostAlloc((void**) &hMixHost_, bytes, cudaHostAllocMapped) != cudaSuccess) { hMixHost_ = nullptr; cudaGetLastError(); return; }
    if (cudaHostGetDevicePointer(&d, hMixHost_, 0) != cudaSuccess) { cudaFreeHost(hMixHost_); hMixHost_ = nullptr; cudaGetLastError(); return; }
    std::memset(hMixHost_, 0, bytes);
    hMixFlag_ = reinterpret_cast<volatile uint32_t*>(hMixHost_ + mixFloats_);
    dMixHostAlias_ = static_cast<float*>(d);
    dMixFlagAlias_ = reinterpret_cast<uint32_t*>(dMixHostAlias_ + mixFloats_);
}

static void freeGroupStorage(Group& g, bool plan) {
    for (auto& kv : g.nodes) {
        if (kv.second.ring) rawFree(kv.second.ring, plan);
        if (kv.second.tapPrivate) rawFree(kv.second.tapPrivate, plan);
    }
    for (auto& kv : g.tapShared) if (kv.second) rawFree(kv.second, plan);
    if (g.dRows) rawFree(g.dRows, plan);
}

Engine::~Engine() {
    dsetdev();
    dsync();
    retireArrays({});
    for (auto& g : groups_) freeGroupStorage(*g, planOnly_);
    groups_.clear();
    for (auto& kv : resources_) if (kv.second->dChannel0) dfree(kv.second->dChannel0);
    for (void* m : peerMapped_) cudaIpcCloseMemHandle(m);
    if (dExchange_) cudaFree(dExchange_);
    if (dPeerStatus_) cudaFree(dPeerStatus_);
    if (dMix_) dfree(dMix_);
    if (dMixScratch_) cudaFree(dMixScratch_);
    if (dMixTickets_) cudaFree(dMixTickets_);
    if (dPartial_) dfree(dPartial_);
    if (dOutVoice_) dfree(dOutVoice_);
    if (dInVoice_) dfree(dInVoice_);
    if (dInShared_) dfree(dInShared_);
    if (hPinned_ && !planOnly_) cudaFreeHost(hPinned_);
    if (hMixHost_) cudaFreeHost(hMixHost_);
    for (OfflineBuf* b : {&offOut_, &offIn_, &offMix_, &offLog_})
        for (int i = 0; i < 2; ++i) { if (b->dev[i]) cudaFree(b->dev[i]); if (b->pinned[i]) cudaFreeHost(b->pinned[i]); }
    if (dDeliverDone_) cudaFree(dDeliverDone_);
    if (dResetPlan_) dfree(dResetPlan_);
    if (dResetCall_) dfree(dResetCall_);
    if (dReadout_) dfree(dReadout_);
    if (hReadout_) cudaFreeHost(hReadout_);
    if (wide_.dRows) dfree(wide_.dRows);
    if (wide_.dSegs) dfree(wide_.dSegs);
    if (wide_.dDst) dfree(wide_.dDst);
    if (dWideScratch_) dfree(dWideScratch_);
    if (dWideTickets_) dfree(dWideTickets_);
    if (dOutCompact_) dfree(dOutCompact_);
    for (auto& kv : batch_) { if (kv.second.dDescs) dfree(kv.second.dDescs); if (kv.second.dTileStart) dfree(kv.second.dTileStart); }
    for (auto& l : timed_)
        for (auto& ev : l) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    for (auto& ev : eventPool_) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    if (ownStream_ && stream_) cudaStreamDestroy(stream_);
}

bool Engine::cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    lastError_ = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

int Engine::setOption(const char* key, double value) {
    Lock lk(mu_);
    steadyValid_ = false;
    const std::string k(key);
    if (k == "tile_width") { opt_.tileWidth = (int) value; }
    else if (k == "warps_per_cta") { opt_.warpsPerCta = (int) value; }
    else if (k == "target_tiles") { opt_.targetTiles = (int) value; opt_.targetTilesSet = true; }
    else if (k == "niter") { opt_.niter = (int) value; }
    else if (k == "batch_groups") { opt_.batchGroups = value != 0; }
    else if (k == "fuse_chains") { opt_.fuseChains = value != 0; }
    else if (k == "specialize") { opt_.specialize = (int) value; }
    else if (k == "specialize_max_words") { opt_.specializeMaxWords = (int) value; }
    else if (k == "specialize_strict") { opt_.specializeStrict = value != 0; }
    else if (k == "spec_minblocks") { opt_.specMinBlocks = (int) value; }
    else if (k == "spec_opprof") { opt_.specOpprof = value != 0; }
    else if (k == "time_kernels") { timeKernels_ = value != 0 && !planOnly_; }
    else if (k == "fuse_conv_root") { opt_.fuseConvRoot = value != 0; }
    else if (k == "pipeline_stages") { opt_.pipelineStages = std::max(0, std::min((int) value, (int) MAX_PIPE)); }
    else if (k == "host_deliver") { hostDeliver_ = value != 0; }
    else if (k == "process_allreduce") { processAllReduce_ = value != 0; }
    else if (k == "plan_dry_run") { planDryRun_ = value != 0 && planOnly_; }
    else return rc::BadArgument;
    return rc::Ok;
}

std::string Engine::describe() const {
    Lock lk(mu_);
    std::ostringstream os;
    os << "{\"voices\":" << numVoices_ << ",\"steady\":" << (steadyValid_ ? "true" : "false") << ",\"groups\":[";
    bool first = true;
    for (auto& g : groups_) {
        if (!first) os << ",";
        first = false;
        os << "{\"v0\":" << g->v0 << ",\"nv\":" << g->nv << ",\"tile_width\":" << g->tileWidth << ",\"nodes\":" << g->nodes.size();
        if (g->pending || g->active) {
            auto& p = g->pending ? g->pending : g->active;
            os << ",\"slots\":" << p->nSlots << ",\"state_rows\":" << p->nStateRows << ",\"params\":" << p->paramMap.size() << ",\"ops\":" << p->nOps << ",\"code_words\":" << p->code.size()
               << ",\"roots\":" << p->rootIds.size() << ",\"pipeline_stages\":" << p->pipeW;
            // the group's mix channels for any nOut past MAX_OUT_CHANNELS are the ones below nOut (DESIGN.md section 3), of the program
            // the last block rendered (a queued program takes over at the next block; before the first block, the queued one's)
            os << ",\"mix_channels\":[";
            const std::vector<int> mc = mixChannels(*g, g->active ? *g->active : *p, (size_t) 1 << 30);
            for (size_t i = 0; i < mc.size(); ++i) os << (i ? "," : "") << mc[i];
            os << "]";
            if (p->specJob) {
                const int st = p->specJob->state.load(std::memory_order_acquire);
                os << ",\"spec_state\":" << st << ",\"spec_cubin_bytes\":" << (st > 0 ? p->specJob->kernel.cubin.size() : 0);
                if (st == 2) os << ",\"spec_regs\":" << p->specJob->kernel.numRegs << ",\"spec_local_bytes\":" << p->specJob->kernel.localBytes;
                if (st < 0) {   // the compiler / loader log, JSON-escaped
                    os << ",\"spec_log\":\"";
                    for (char c : p->specJob->log) {
                        if (c == '"' || c == '\\') os << '\\' << c;
                        else if (c == '\n') os << "\\n";
                        else if ((unsigned char) c >= 0x20) os << c;
                    }
                    os << "\"";
                }
            }
        }
        // K3 state per convolver: distinct IRs in use and the kernel form that runs (silent: every IR trimmed to nothing)
        std::map<int32_t, const ConvolverState*> convs;
        for (auto& kv : g->nodes) if (kv.second.kind == NodeKind::Convolve && kv.second.conv) convs[kv.first] = kv.second.conv.get();
        if (!convs.empty()) {
            os << ",\"convolvers\":[";
            bool firstConv = true;
            for (auto& kv : convs) {
                const ConvolverState& cs = *kv.second;
                os << (firstConv ? "" : ",") << "{\"node\":" << kv.first << ",\"irs\":" << cs.irs.size() << ",\"partitions\":" << cs.partitions
                   << ",\"form\":\"" << (cs.maxS == 0 ? "silent" : (cs.perChannel() ? "per_channel" : "shared")) << "\"}";
                firstConv = false;
            }
            os << "]";
        }
        os << "}";
    }
    os << "],\"ir_bank\":" << irBank_.live() << "}";
    return os.str();
}

std::string Engine::snapshot(int voice) const {
    Lock lk(mu_);
    std::string o = "{";
    for (auto& g : groups_) {
        if (voice < g->v0 || voice >= g->v0 + g->nv) continue;
        std::map<int32_t, const Node*> sorted;
        for (auto& kv : g->nodes) sorted[kv.first] = &kv.second;
        bool first = true;
        for (auto& kv : sorted) {
            char key[24];
            std::snprintf(key, sizeof key, "\"0x%08x\":", (unsigned) kv.first);    // nodeIdToHex, Types.h:16-27
            if (!first) o += ',';
            first = false;
            o += key;
            Value props = Value::object();
            for (auto& p : kv.second->props) props.asObject()[p.first] = p.second;
            writeJson(o, props);
        }
        break;
    }
    return o + "}";
}

long Engine::specializeDryRun(int voice, std::string& log) {
    Lock lk(mu_);
    for (auto& g : groups_) {
        if (voice < g->v0 || voice >= g->v0 + g->nv) continue;
        auto& p = g->pending ? g->pending : g->active;
        if (!p) { log = "no compiled program for this voice"; return -1; }
        if (p->stages.size() > 1) { log = "multi-stage programs (convolve) are not specialised"; return -1; }
        SpecKernel k;
        if (!specialise_compile(p->code, g->tileWidth, opt_.niter, customSource(), k, log, opt_.specMinBlocks, opt_.specOpprof)) return -1;
        return (long) k.cubin.size();
    }
    log = "voice out of range";
    return -1;
}

bool Engine::specOpprofRead(unsigned long long* out128, bool reset) {
    Lock lk(mu_);
    std::set<const SpecJob*> seen;
    for (auto& g : groups_) {
        const auto& p = g->active;
        if (!p || !p->specJob || !p->specJob->opprof || p->specJob->state.load(std::memory_order_acquire) != 2) continue;
        if (!seen.insert(p->specJob.get()).second) continue;
        if (!specialise_opprof_read(p->specJob->kernel, out128, reset)) return false;
    }
    return true;
}

std::vector<uint32_t> Engine::programWords(int voice) const {
    Lock lk(mu_);
    for (auto& g : groups_) {
        if (voice < g->v0 || voice >= g->v0 + g->nv) continue;
        auto& p = g->pending ? g->pending : g->active;
        if (p) return p->code;
    }
    return {};
}

// ---------------------------------------------------------------------------------------------------------
// storage
int Engine::allocRows(Group& g, int count, bool evenAlign, int& row) {
    int start = g.rowsUsed;
    if (evenAlign && (start & 1)) ++start;
    const int need = start + count;
    if (need > g.rowsCap) {
        int cap = std::max(64, g.rowsCap * 2);
        while (cap < need) cap *= 2;
        float* nb = nullptr;
        if (!cuda(dmalloc((void**) &nb, sizeof(float) * (size_t) cap * g.Vpad), "cudaMalloc rows")) return rc::CudaError;
        if (!cuda(dmemset(nb, 0, sizeof(float) * (size_t) cap * g.Vpad), "memset rows")) return rc::CudaError;
        if (g.dRows) {
            if (!cuda(dmemcpy(nb, g.dRows, sizeof(float) * (size_t) g.rowsUsed * g.Vpad, cudaMemcpyDeviceToDevice), "copy rows")) return rc::CudaError;
            dsync();
            dfree(g.dRows);
        }
        g.dRows = nb;
        g.rowsCap = cap;
    }
    row = start;
    g.rowsUsed = need;
    return rc::Ok;
}

int Engine::fillRowBits(Group& g, int row, int vb, int ve, uint32_t bits) {
    if (row < 0) return rc::Ok;
    const int n = ve - vb;
    if (n <= 0) return rc::Ok;
    uint32_t* p = reinterpret_cast<uint32_t*>(g.dRows + (size_t) row * g.Vpad + vb);
    if (bits == 0) return cuda(dmemset(p, 0, sizeof(float) * n), "memset row") ? rc::Ok : rc::CudaError;
    // cudaMemcpyAsync from PAGEABLE host memory returns once the source has been copied to the driver's staging buffer (CUDA runtime
    // API, "API synchronization behavior"): tmp may die right after the call, no stream synchronisation needed — a graph with fifty
    // consts used to cost fifty of them (config 5 set-up: 1250 graphs).
    std::vector<uint32_t> tmp((size_t) n, bits);
    if (!cuda(dmemcpy(p, tmp.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice), "fill row")) return rc::CudaError;
    return rc::Ok;
}

int Engine::fillRow(Group& g, int row, int vb, int ve, float value) {
    uint32_t bits;
    std::memcpy(&bits, &value, 4);
    return fillRowBits(g, row, vb, ve, bits);
}

// Rows row .. row + rows - 1 of group voices [vb, vb + cnt) <- words[k * cnt + i] (32-bit words, row-major).  The source is pageable:
// staged before the call returns (fillRowBits), so it may die right after.
int Engine::writeColumns(Group& g, int row, int rows, int vb, int cnt, const void* words, const char* what) {
    for (int k = 0; k < rows; ++k)
        if (!cuda(dmemcpy(g.dRows + (size_t) (row + k) * g.Vpad + vb, static_cast<const uint32_t*>(words) + (size_t) k * cnt,
                          sizeof(uint32_t) * cnt, cudaMemcpyHostToDevice), what)) return rc::CudaError;
    return rc::Ok;
}

// Voice vb + i (group-relative, i < ve - vb) of node n reads arrs[index[i]] (index null: arrs[0]) from its next block on: the array's
// address and length go to the node's first ARRAY_ROWS parameter rows — a seq-family node's generation *gen to the next (SEQ_GEN) —
// and the voice holds the array.  The arrays the voices held before are retired (retireArrays).
int Engine::assignVoiceArrays(Group& g, Node& n, const std::vector<VoiceArray>& arrs, const int32_t* index, int vb, int ve, const uint32_t* gen) {
    const int cnt = ve - vb, rows = gen ? SEQ_PARAM_ROWS : ARRAY_ROWS;
    if (cnt <= 0) return rc::Ok;
    std::vector<uint32_t> words((size_t) rows * cnt);
    for (int i = 0; i < cnt; ++i) {
        const VoiceArray& a = arrs[index ? (size_t) index[i] : 0];
        words[(size_t) i] = (uint32_t) a.ptr;
        words[(size_t) cnt + i] = (uint32_t) (a.ptr >> 32);
        words[(size_t) 2 * cnt + i] = a.len;
        if (gen) words[(size_t) SEQ_GEN * cnt + i] = *gen;
    }
    const int r = writeColumns(g, n.paramRow, rows, vb, cnt, words.data(), "per-voice array rows");
    if (r != rc::Ok) return r;
    if (n.voiceArrays.size() < (size_t) g.nv) n.voiceArrays.resize((size_t) g.nv);
    std::vector<std::shared_ptr<const void>> old(n.voiceArrays.begin() + vb, n.voiceArrays.begin() + ve);
    for (int i = 0; i < cnt; ++i) n.voiceArrays[(size_t) (vb + i)] = arrs[index ? (size_t) index[i] : 0].hold;
    retireArrays(std::move(old));
    steadyValid_ = false;
    return rc::Ok;
}

int Engine::ensureResourceOnDevice(Resource& r) {
    if (r.dChannel0 || r.numSamples == 0) return rc::Ok;
    const size_t padded = (r.numSamples + 3) / 4 * 4;
    if (!cuda(dmalloc((void**) &r.dChannel0, sizeof(float) * padded), "cudaMalloc resource")) return rc::CudaError;
    if (!cuda(dmemset(r.dChannel0, 0, sizeof(float) * padded), "memset resource")) return rc::CudaError;
    if (!cuda(dmemcpySync(r.dChannel0, r.channels[0].data(), sizeof(float) * r.numSamples, cudaMemcpyHostToDevice), "upload resource")) return rc::CudaError;
    return rc::Ok;
}

int Engine::uploadArray(std::shared_ptr<DeviceArray>& out, const void* data, size_t bytes, size_t count) {
    auto a = std::make_shared<DeviceArray>();
    a->planOnly = planOnly_; a->bytes = bytes; a->count = count;
    if (!cuda(dmalloc(&a->d, std::max<size_t>(bytes, 16)), "cudaMalloc sequence data")) return rc::CudaError;
    if (bytes && !cuda(dmemcpySync(a->d, data, bytes, cudaMemcpyHostToDevice), "upload sequence data")) return rc::CudaError;
    out = a;   // programs compiled against the previous array keep it alive until they are released
    return rc::Ok;
}

// A `seq` value as the device array a node of the seq family reads (ctl_seq / ctl_seq2 / ctl_sparseq / ctl_sparseq2): seq and seq2
// float[n]; sparseq int32 tickTime[n] then float value[n]; sparseq2 double time[n] then float value[n].  The keyed forms are sorted
// and keep the FIRST value of a duplicated key, like std::map::insert in the reference (SparSeq.h:111, SparSeq2.h:50).
static int seqBlob(NodeKind kind, const Value& val, std::vector<char>& blob, size_t& count) {
    if (!val.isArray()) return rc::InvalidPropertyType;
    if (kind == NodeKind::Seq || kind == NodeKind::Seq2) {   // Core.h:447-466, Seq2.h:60-84
        std::vector<float> data;
        for (auto& e : val.asArray()) {
            if (!e.isNumber()) return rc::InvalidInstructionFormat;   // the reference throws bad_variant_access here
            data.push_back((float) e.asNumber());
        }
        blob.assign(reinterpret_cast<const char*>(data.data()), reinterpret_cast<const char*>(data.data() + data.size()));
        count = data.size();
        return rc::Ok;
    }
    const bool sparseq = kind == NodeKind::SparSeq;
    std::map<double, float> m;   // sparseq: the int32 tick time, exact in a double
    for (auto& e : val.asArray()) {
        if (!e.isObject()) return rc::InvalidInstructionFormat;
        auto& o = e.asObject();
        auto v = o.find("value"), t = o.find(sparseq ? "tickTime" : "time");
        if (v == o.end() || t == o.end() || !v->second.isNumber() || !t->second.isNumber()) return rc::InvalidInstructionFormat;
        m.insert({sparseq ? (double) static_cast<int32_t>(t->second.asNumber()) : t->second.asNumber(), (float) v->second.asNumber()});
    }
    const size_t kb = sparseq ? 4 : 8;
    blob.assign(m.size() * (kb + 4), 0);
    size_t i = 0;
    for (auto& kv : m) {
        if (sparseq) { const int32_t t = (int32_t) kv.first; std::memcpy(blob.data() + 4 * i, &t, 4); }
        else std::memcpy(blob.data() + 8 * i, &kv.first, 8);
        std::memcpy(blob.data() + kb * m.size() + 4 * i, &kv.second, 4);
        ++i;
    }
    count = m.size();
    return rc::Ok;
}

static bool isSeqFamily(NodeKind k) { return k == NodeKind::Seq || k == NodeKind::Seq2 || k == NodeKind::SparSeq || k == NodeKind::SparSeq2; }

// Whether some voice of the group has a non-empty sequence: seq, seq2 and sparseq2 render zeros without touching their state otherwise
static bool anySeq(const Node& n) {
    if (n.paramRow < 0) return n.seqData && n.seqData->count > 0;
    return std::any_of(n.voiceArrays.begin(), n.voiceArrays.end(),
                       [](const std::shared_ptr<const void>& a) { return a && static_cast<const DeviceArray*>(a.get())->count > 0; });
}

// Arrays voices stopped reading.  No program pins them and no later block reads them, but blocks already enqueued may: each is released
// (freed when nothing else holds it) once the stream has passed an event recorded now.  Stream-ordered deferral, no drain.
void Engine::retireArrays(std::vector<std::shared_ptr<const void>>&& arrs) {
    while (!retiredArrays_.empty() && cudaEventQuery(retiredArrays_.front().first) == cudaSuccess) {
        cudaEventDestroy(retiredArrays_.front().first);
        retiredArrays_.pop_front();
    }
    std::sort(arrs.begin(), arrs.end());
    arrs.erase(std::unique(arrs.begin(), arrs.end()), arrs.end());
    if (!arrs.empty() && !arrs.front()) arrs.erase(arrs.begin());
    if (planOnly_ || arrs.empty()) return;
    cudaEvent_t ev = nullptr;
    if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(ev, stream_) != cudaSuccess) {
        if (ev) cudaEventDestroy(ev);
        dsync();   // no event: wait for the blocks instead
        return;
    }
    retiredArrays_.emplace_back(ev, std::move(arrs));
}

int Engine::setSeqPerVoice(int32_t nodeId, const char* const* seqs, int numSeqs, const int32_t* index, int vb, int count) {
    // Each distinct text is parsed once, outside the lock, like applyInstructions' batch
    std::vector<Value> vals((size_t) std::max(0, numSeqs));
    std::vector<char> parsed(vals.size(), 0);
    for (size_t k = 0; k < vals.size(); ++k) {
        if (!seqs[k]) continue;
        try { vals[k] = parseJson(seqs[k], std::strlen(seqs[k])); parsed[k] = 1; } catch (const std::exception&) {}
    }
    Lock lk(mu_);
    dsetdev();
    if (numSeqs < 0) return fail(rc::BadArgument, "voice range out of bounds");
    for (int i = 0; i < count; ++i)
        if (index[i] < 0 || index[i] >= numSeqs) return fail(rc::BadArgument, "sequence index out of range");
    // every check before any change: a failed call changes nothing
    std::vector<VoiceTarget> targets;
    int r = voiceTargets(nodeId, vb, count, isSeqFamily, "node is not a seq, seq2, sparseq or sparseq2", targets);
    if (r != rc::Ok) return r;
    std::vector<NodeKind> kinds;   // of the node in the groups of the range (cuts keep a node's kind, so normally one)
    for (auto& t : targets)
        if (std::find(kinds.begin(), kinds.end(), t.n.kind) == kinds.end()) kinds.push_back(t.n.kind);
    std::vector<std::vector<char>> blobs(kinds.size() * vals.size());
    std::vector<size_t> counts(blobs.size(), 0);
    for (size_t k = 0; k < vals.size(); ++k) {
        if (!parsed[k]) return fail(rc::InvalidInstructionFormat, "sequence " + std::to_string(k) + " is not valid JSON");
        for (size_t j = 0; j < kinds.size(); ++j) {
            if ((r = seqBlob(kinds[j], vals[k], blobs[j * vals.size() + k], counts[j * vals.size() + k])) != rc::Ok)
                return fail(r, "sequence " + std::to_string(k) + " is not a valid seq value for this node");
        }
    }
    // one device array per distinct sequence (and node kind) that some voice takes
    std::vector<std::vector<VoiceArray>> arrs(kinds.size(), std::vector<VoiceArray>(vals.size()));
    for (size_t j = 0; j < kinds.size(); ++j)
        for (int i = 0; i < count; ++i) {
            const size_t k = (size_t) index[i], b = j * vals.size() + k;
            if (arrs[j][k].hold) continue;
            std::shared_ptr<DeviceArray> a;
            if ((r = uploadArray(a, blobs[b].data(), blobs[b].size(), counts[b])) != rc::Ok) return r;
            arrs[j][k] = seqArray(a);
        }
    for (auto& t : targets) {
        if (t.n.paramRow < 0) {   // its first per-voice sequence: the rows, every voice on the group's sequence; the next compile sets mode bit 3
            if ((r = allocRows(t.g, SEQ_PARAM_ROWS, false, t.n.paramRow)) != rc::Ok ||
                (r = assignVoiceArrays(t.g, t.n, {seqArray(t.n.seqData)}, nullptr, 0, t.g.nv, &t.n.seqGen)) != rc::Ok) return r;
            t.g.codeDirty = true;
        }
        ++t.n.seqGen;   // one counter per node, shared with JSON `seq`: a voice's generation changes exactly when it receives a sequence
        const size_t j = (size_t) (std::find(kinds.begin(), kinds.end(), t.n.kind) - kinds.begin());
        const bool had = anySeq(t.n);
        if ((r = assignVoiceArrays(t.g, t.n, arrs[j], index + t.at, t.b, t.e, &t.n.seqGen)) != rc::Ok) return r;
        if (anySeq(t.n) != had) t.g.codeDirty = true;   // the op is emitted while some voice has a sequence
        t.n.props["seq"] = vals[(size_t) index[t.last()]];
    }
    return rc::Ok;
}

int Engine::addSharedResource(const char* name, const float* const* chans, size_t nCh, size_t nSamples) {
    Lock lk(mu_);
    // insert-only: SharedResource.h:44-46 (emplace fails on an existing key)
    if (resources_.count(name)) return 0;
    auto r = std::make_shared<Resource>();
    r->name = name;
    r->numSamples = nSamples;
    for (size_t c = 0; c < nCh; ++c) r->channels.emplace_back(chans[c], chans[c] + nSamples);   // copied in: AudioBufferResource.h:13-24
    if (nCh == 0) r->numSamples = 0;
    resources_[name] = r;
    return 1;
}

void Engine::pruneSharedResources() {
    Lock lk(mu_);   // SharedResource.h:93-101: drop entries nobody else references
    dsync();
    retireArrays({});   // the stream is drained: releases every retired array, the sample buffers voices stopped playing among them
    for (auto it = resources_.begin(); it != resources_.end();) {
        if (it->second.use_count() == 1) {
            if (it->second->dChannel0) dfree(it->second->dChannel0);
            it = resources_.erase(it);
        } else ++it;
    }
}

std::vector<std::string> Engine::listSharedResources() const {
    Lock lk(mu_);
    std::vector<std::string> out;
    for (auto& kv : resources_) out.push_back(kv.first);
    return out;
}

// ---------------------------------------------------------------------------------------------------------
// instruction interpreter
static bool toInt32(const Value& v, int32_t& out) {
    if (!v.isNumber()) return false;
    out = static_cast<int32_t>(v.asNumber());   // Runtime.h:299
    return true;
}

// builtin or registered: kind, fn (registered types: their index), state rows
static bool lookupType(const std::string& name, const std::vector<std::pair<std::string, int>>& custom, TypeInfo& out) {
    auto it = typeTable().find(name);
    if (it != typeTable().end()) { out = it->second; return true; }
    for (size_t i = 0; i < custom.size(); ++i)
        if (custom[i].first == name) { out = TypeInfo{NodeKind::Custom, (uint32_t) i, custom[i].second, false}; return true; }
    return false;
}

int Engine::registerNodeType(const char* type, int numInputs, int numState, const char* body) {
    Lock lk(mu_);
    if (!type || !body || numInputs < 0 || numInputs > 8 || numState < 0 || numState > 8) return fail(rc::BadArgument, "registerNodeType: 0..8 inputs, 0..8 state floats");
    if (hasNodeType(type)) return rc::NodeTypeAlreadyExists;     // Runtime.h:482-483
    customTypes_.push_back(CustomType{type, body, numInputs, numState});
    return rc::Ok;
}

bool Engine::hasNodeType(const char* type) const {
    Lock lk(mu_);
    if (typeTable().count(type)) return true;
    for (auto& c : customTypes_) if (c.name == type) return true;
    return false;
}

std::string Engine::customSource() const {
    if (customTypes_.empty()) return std::string();
    std::ostringstream os;
    os << "#define EB_CUSTOM_NODES 1\nnamespace eb {\n";
    for (size_t i = 0; i < customTypes_.size(); ++i)
        os << "// registered node type \"" << customTypes_[i].name << "\"\n__device__ __forceinline__ float eb_custom_" << i
           << "(float* s, const float* in, const float sr) {\n" << customTypes_[i].body << "\n}\n";
    os << "template <int ID> __device__ __forceinline__ float eb_custom_call(float* s, const float* in, const float sr) {\n";
    for (size_t i = 0; i < customTypes_.size(); ++i) os << "    if constexpr (ID == " << i << ") return eb_custom_" << i << "(s, in, sr);\n";
    os << "    return 0.0f;\n}\n}\n";
    return os.str();
}

int Engine::createNode(Group& g, const Value& a1, const Value& a2) {   // Runtime.h:294-313
    int32_t id;
    if (!toInt32(a1, id) || !a2.isString()) return rc::InvalidInstructionFormat;
    std::vector<std::pair<std::string, int>> custom;
    for (auto& c : customTypes_) custom.push_back({c.name, c.nState});
    TypeInfo ti;
    if (!lookupType(a2.asString(), custom, ti)) return rc::UnknownNodeType;
    struct { TypeInfo second; } holder{ti};
    auto* it = &holder;
    if (g.nodes.count(id)) return rc::NodeAlreadyExists;

    Node n;
    n.id = id;
    n.kind = it->second.kind;
    n.fn = it->second.fn;
    n.typeName = a2.asString();
    if (it->second.stateRows > 0) {
        int r = allocRows(g, it->second.stateRows, it->second.doubleRows > 0, n.stateRow);
        if (r != rc::Ok) return r;
        for (int k = 0; k < it->second.stateRows; ++k)   // new rows are zero
            if (freshRowBits(n.kind, k) != 0u && (r = fillRowBits(g, n.stateRow + k, 0, g.Vpad, freshRowBits(n.kind, k))) != rc::Ok) return r;
    }
    if (shadowedRow(n.kind) >= 0) {   // outside the state rows: no program stages it
        int r = allocRows(g, 1, false, n.shadowRow);
        if (r != rc::Ok) return r;
    }
    switch (n.kind) {
        case NodeKind::Const: {   // Core.h:166 default 1
            int r = allocRows(g, 1, false, n.paramRow);
            if (r != rc::Ok) return r;
            if ((r = fillRow(g, n.paramRow, 0, g.nv, 1.0f)) != rc::Ok) return r;
        } break;
        case NodeKind::Sr: {      // Core.h:173-180
            int r = allocRows(g, 1, false, n.paramRow);
            if (r != rc::Ok) return r;
            if ((r = fillRow(g, n.paramRow, 0, g.nv, (float) sr_)) != rc::Ok) return r;
        } break;
        case NodeKind::Root: n.fade.init(sr_); n.channel = -1; break;          // Core.h:80-82
        case NodeKind::Delay: n.size = blockSize_; n.ringDirty = true; break;  // Delays.h:56
        case NodeKind::SDelay: n.length = blockSize_; n.size = bitceil(blockSize_ + blockSize_); n.ringDirty = true; break;   // Delays.h:183,197-198
        case NodeKind::Metro: n.intervalSamps = static_cast<int64_t>(std::max(2.0, 1000.0 * 0.001 * sr_)); break;   // Metro.h:14-18
        case NodeKind::Scope:   // Analyzers.h:147-153: the constructor sets both props
            n.props["channels"] = Value::number(1); n.props["size"] = Value::number(512);
            n.size = SCOPE_CHANNELS * SCOPE_RING; break;
        case NodeKind::Capture: n.size = bitceil((int) (size_t) sr_) + CAPTURE_SCRATCH; break;   // Capture.h:17
        case NodeKind::Sample: {   // no buffer, offsets 0: new rows are zero
            int r = allocRows(g, SAMPLE_PARAM_ROWS, false, n.paramRow);
            if (r != rc::Ok) return r;
        } break;
        case NodeKind::Fft: {   // wasm/FFT.h:18-26: ring of one channel, default size 1024 set through setProperty
            n.size = SCOPE_RING;
            Node& ref = g.nodes.emplace(id, std::move(n)).first->second;
            return nodeSetProperty(g, ref, "size", Value::number(1024), 0, g.nv);
        }
        default: break;
    }
    g.nodes.emplace(id, std::move(n));
    return rc::Ok;
}

int Engine::appendChild(Group& g, const Value& a1, const Value& a2, const Value& a3) {   // Runtime.h:336-366
    int32_t parent, child, chan;
    if (!toInt32(a1, parent) || !toInt32(a2, child) || !toInt32(a3, chan)) return rc::InvalidInstructionFormat;
    auto p = g.nodes.find(parent);
    if (p == g.nodes.end()) return rc::NodeNotFound;
    if (!g.nodes.count(child)) return rc::NodeNotFound;
    p->second.inlets.push_back(Inlet{child, chan});
    return rc::Ok;
}

int Engine::nodeSetProperty(Group& g, Node& n, const std::string& key, const Value& val, int vb, int ve) {
    // vb/ve are group-relative voice bounds; only per-voice capable props honour a sub-range.
    const PerVoiceProp* pv = perVoiceProp(n.kind, key);
    if (pv && pv->bits) {   // const.value (Core.h:142-152), rand.seed (Noise.h:13-23), sample.startOffset / stopOffset (Sample.h:56,69)
        if (!val.isNumber()) return rc::InvalidPropertyType;
        uint32_t bits;
        if (!pv->bits(val.asNumber(), bits)) return rc::InvalidPropertyValue;
        int r = fillRowBits(g, n.*pv->base + pv->row, vb, ve, bits);
        if (r == rc::Ok && pv->shadow) r = fillRowBits(g, n.shadowRow, vb, ve, bits);
        if (r != rc::Ok) return r;
        n.props[key] = val;
        return rc::Ok;
    }
    if (key == "seq" && isSeqFamily(n.kind)) {   // the whole group: a batch that sets `seq` cuts the group at its voice range first
        std::vector<char> blob;
        size_t count = 0;
        int r = seqBlob(n.kind, val, blob, count);
        if (r == rc::Ok) r = uploadArray(n.seqData, blob.data(), blob.size(), count);
        if (r != rc::Ok) return r;
        ++n.seqGen; g.codeDirty = true;
        // the voices' own rows, if any, all take the new sequence
        if (n.paramRow >= 0 && (r = assignVoiceArrays(g, n, {seqArray(n.seqData)}, nullptr, vb, ve, &n.seqGen)) != rc::Ok) return r;
        n.props[key] = val;
        return rc::Ok;
    }
    switch (n.kind) {
        case NodeKind::Root:        // Core.h:33-64
            if (key == "active") {
                if (!val.isBool()) return rc::InvalidPropertyType;
                if (val.asBool()) n.fade.fadeIn(); else n.fade.fadeOut();
            }
            if (key == "channel") {
                if (!val.isNumber()) return rc::InvalidInstructionFormat;   // reference throws bad_variant_access here
                n.channel = static_cast<int>(val.asNumber());
            }
            if (key == "fadeInMs") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                n.fade.setFadeInMs(sr_, val.asNumber());
            }
            if (key == "fadeOutMs") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                n.fade.setFadeOutMs(sr_, val.asNumber());
            }
            break;
        case NodeKind::In:          // Math.h:95-105
            if (key == "channel") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                n.channel = static_cast<int>(val.asNumber());
                g.codeDirty = true;
            }
            break;
        case NodeKind::Svf:         // filters/SVF.h:30-46
            if (key == "mode") {
                if (!val.isString()) return rc::InvalidPropertyType;
                const std::string& m = val.asString();
                if (m == "lowpass") n.mode = 0; if (m == "bandpass") n.mode = 1; if (m == "highpass") n.mode = 2;
                if (m == "notch") n.mode = 3; if (m == "allpass") n.mode = 4;
                g.codeDirty = true;
            }
            break;
        case NodeKind::SvfShelf:    // filters/SVFShelf.h:30-44
            if (key == "mode") {
                if (!val.isString()) return rc::InvalidPropertyType;
                const std::string& m = val.asString();
                if (m == "lowshelf") n.mode = 0; if (m == "highshelf") n.mode = 1; if (m == "bell" || m == "peak") n.mode = 2;
                g.codeDirty = true;
            }
            break;
        case NodeKind::MM1p:        // filters/MultiMode1p.h:50-65
            if (key == "mode") {
                if (!val.isString()) return rc::InvalidPropertyType;
                const std::string& m = val.asString();
                if (m == "lowpass") n.mode = 0; if (m == "highpass") n.mode = 2; if (m == "allpass") n.mode = 4;
                g.codeDirty = true;
            }
            break;
        case NodeKind::Delay:       // Delays.h:59-76
            if (key == "size") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                n.size = std::max(0, static_cast<int>(val.asNumber()));
                n.ringDirty = true; g.codeDirty = true;
            }
            break;
        case NodeKind::SDelay:      // Delays.h:188-206
            if (key == "size") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                n.length = std::max(0, static_cast<int>(val.asNumber()));
                n.size = bitceil(n.length + blockSize_);
                n.ringDirty = true; g.codeDirty = true;
            }
            break;
        case NodeKind::MaxHold:     // Core.h:292-303
            if (key == "hold") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                const double h = sr_ * 0.001 * val.asNumber();
                n.holdSamples = static_cast<uint32_t>(h); g.codeDirty = true;
            }
            break;
        case NodeKind::TapIn:
        case NodeKind::TapOut:      // Feedback.h:24-38,71-85
            if (key == "name") {
                if (!val.isString()) return rc::InvalidPropertyType;
                n.tapName = val.asString(); g.codeDirty = true;
            }
            break;
        case NodeKind::Table:       // Table.h:20-34
        case NodeKind::Convolve:    // wasm/Convolve.h:35-56
            if (key == "path") {
                if (!val.isString()) return rc::InvalidPropertyType;
                auto it = resources_.find(val.asString());
                if (it == resources_.end()) return rc::InvalidPropertyValue;
                n.resource = it->second;
                n.resourceDirty = true; g.codeDirty = true;
            }
            break;
        case NodeKind::Sample:      // Sample.h:25-76
            if (key == "path") {
                if (!val.isString()) return rc::InvalidPropertyType;
                auto it = resources_.find(val.asString());
                if (it == resources_.end()) return rc::InvalidPropertyValue;
                int r = assignSampleBuffers(g, n, {it->second}, nullptr, vb, ve);
                if (r != rc::Ok) return r;
            }
            if (key == "mode") {
                if (!val.isString()) return rc::InvalidPropertyType;
                const std::string& m = val.asString();
                if (m == "trigger") n.mode = 0; if (m == "gate") n.mode = 1; if (m == "loop") n.mode = 2;
                g.codeDirty = true;
            }
            break;

        case NodeKind::Once:        // Core.h:345-361: the prop can arm but never disarm
            if (key == "arm") {
                if (!val.isBool()) return rc::InvalidPropertyType;
                if (val.asBool()) {
                    int r = fillRow(g, n.stateRow, vb, ve, 1.0f);
                    if (r == rc::Ok) r = fillRow(g, n.shadowRow, vb, ve, 1.0f);
                    if (r != rc::Ok) return r;
                }
            }
            break;
        case NodeKind::Seq:         // Core.h:411-466
        case NodeKind::Seq2:        // Seq2.h:39-84
            if (key == "hold") { if (!val.isBool()) return rc::InvalidPropertyType; n.seqHold = val.asBool(); g.codeDirty = true; }
            if (key == "loop") { if (!val.isBool()) return rc::InvalidPropertyType; n.seqLoop = val.asBool(); g.codeDirty = true; }
            if (key == "offset") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                if (val.asNumber() < 0.0) return rc::InvalidPropertyValue;
                n.seqOffset = static_cast<uint64_t>(val.asNumber()); g.codeDirty = true;
            }
            break;
        case NodeKind::SparSeq:     // SparSeq.h:40-124
            if (key == "offset") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                if (val.asNumber() < 0.0) return rc::InvalidPropertyValue;
                n.seqOffset = static_cast<uint64_t>(val.asNumber()); g.codeDirty = true;
            }
            if (key == "loop") {
                if (val.isNull() || (val.isBool() && !val.asBool())) { n.loopStart = -1; n.loopEnd = -1; }
                else {
                    if (!val.isArray()) return rc::InvalidPropertyType;
                    auto& pts = val.asArray();
                    if (pts.size() < 2 || !pts[0].isNumber() || !pts[1].isNumber()) return rc::InvalidInstructionFormat;
                    n.loopStart = static_cast<int32_t>(pts[0].asNumber()); n.loopEnd = static_cast<int32_t>(pts[1].asNumber());
                }
                ++n.loopGen; g.codeDirty = true;
            }
            if (key == "follow") { if (!val.isBool()) return rc::InvalidPropertyType; n.follow = val.asBool(); g.codeDirty = true; }
            if (key == "interpolate") { if (!val.isNumber()) return rc::InvalidPropertyType; n.interpolate = static_cast<int32_t>(val.asNumber()); g.codeDirty = true; }
            if (key == "tickInterval") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                if (val.asNumber() < 0.0) return rc::InvalidPropertyValue;
                n.tickIntervalSamples = sr_ * val.asNumber(); g.codeDirty = true;
            }
            break;
        case NodeKind::SparSeq2:    // SparSeq2.h:20-56
            if (key == "interpolate") { if (!val.isNumber()) return rc::InvalidPropertyType; n.interpolate = static_cast<int32_t>(val.asNumber()); g.codeDirty = true; }
            break;
        case NodeKind::Scope:       // Analyzers.h:155-179
            if (key == "size") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                if (val.asNumber() < 256 || val.asNumber() > 8192) return rc::InvalidPropertyValue;
            }
            if (key == "channels") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                if (val.asNumber() < 0 || val.asNumber() > 4) return rc::InvalidPropertyValue;
            }
            if (key == "name" && !val.isString()) return rc::InvalidPropertyType;
            break;
        case NodeKind::Fft:         // wasm/FFT.h:32-71
            if (key == "size") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                const int size = static_cast<int>(val.asNumber());
                if (!(size > 0 && (size & (size - 1)) == 0) || size < 256 || size > 8192) return rc::InvalidPropertyValue;
                n.window.resize((size_t) size);
                for (int i = 0; i < size; ++i) {   // Blackman-Harris in the reference's mixed float/double arithmetic (FFT.h:49-62)
                    const float a0 = 0.35875f, a1 = 0.48829f, a2 = 0.14128f, a3 = 0.01168f;
                    const float pi = 3.1415926535897932385f;
                    const float t1 = (float) (a1 * std::cos(2.0 * pi * (i / (double) (size - 1))));
                    const float t2 = (float) (a2 * std::cos(4.0 * pi * (i / (double) (size - 1))));
                    const float t3 = (float) (a3 * std::cos(6.0 * pi * (i / (double) (size - 1))));
                    n.window[(size_t) i] = a0 - t1 + t2 - t3;
                }
            }
            if (key == "name" && !val.isString()) return rc::InvalidPropertyType;
            break;
        case NodeKind::Metro:       // wasm/Metro.h:20-37
            if (key == "interval") {
                if (!val.isNumber()) return rc::InvalidPropertyType;
                if (0 >= val.asNumber()) return rc::InvalidPropertyValue;
                n.intervalSamps = static_cast<int64_t>(std::max(2.0, val.asNumber() * 0.001 * sr_)); g.codeDirty = true;
            }
            break;
        default: break;
    }
    n.props[key] = val;   // GraphNode.h:60-63
    return rc::Ok;
}

int Engine::setProperty(Group& g, const Value& a1, const Value& a2, const Value& v, int vb, int ve) {   // Runtime.h:316-333
    int32_t id;
    if (!toInt32(a1, id) || !a2.isString()) return rc::InvalidInstructionFormat;
    auto it = g.nodes.find(id);
    if (it == g.nodes.end()) return rc::NodeNotFound;
    return nodeSetProperty(g, it->second, a2.asString(), v, vb, ve);
}

int Engine::activateRoots(Group& g, const Value& roots) {   // Runtime.h:369-433
    if (!roots.isArray()) return rc::InvalidInstructionFormat;
    std::set<int32_t> active;
    for (auto& v : roots.asArray()) {
        int32_t id;
        if (!toInt32(v, id)) return rc::InvalidInstructionFormat;
        auto it = g.nodes.find(id);
        if (it == g.nodes.end()) return rc::NodeNotFound;
        if (it->second.kind == NodeKind::Root) {
            nodeSetProperty(g, it->second, "active", Value::boolean(true), 0, g.nv);
            active.insert(id);
        }
    }
    for (int32_t id : g.currentRoots) {
        auto it = g.nodes.find(id);
        if (it == g.nodes.end() || it->second.kind != NodeKind::Root) continue;
        Node& n = it->second;
        if (!active.count(id)) nodeSetProperty(g, n, "active", Value::boolean(false), 0, g.nv);
        if (n.fade.on() || !n.fade.settled()) active.insert(id);   // stillRunning(): Core.h:28-31
    }
    g.currentRoots.swap(active);
    return rc::Ok;
}

int Engine::applyToGroup(Group& g, const std::vector<Value>& batch, int vb, int ve) {   // Runtime.h:170-218
    bool shouldRebuild = false;
    for (auto& next : batch) {
        if (!next.isArray()) return rc::InvalidInstructionFormat;
        auto& ar = next.asArray();
        if (ar.empty() || !ar[0].isNumber()) return rc::InvalidInstructionFormat;
        const int cmd = static_cast<int>(ar[0].asNumber());
        int res = rc::Ok;
        // the reference indexes ar[1..3] unchecked; a short instruction is undefined behaviour there, an
        // InvalidInstructionFormat here.
        auto need = [&](size_t n) { return ar.size() >= n; };
        switch (cmd) {
            case 0: res = need(3) ? createNode(g, ar[1], ar[2]) : rc::InvalidInstructionFormat; break;
            case 3: res = need(4) ? setProperty(g, ar[1], ar[2], ar[3], vb, ve) : rc::InvalidInstructionFormat; break;
            case 2: res = need(4) ? appendChild(g, ar[1], ar[2], ar[3]) : rc::InvalidInstructionFormat; break;
            case 4:
                res = need(2) ? activateRoots(g, ar[1]) : rc::InvalidInstructionFormat;
                shouldRebuild = true;
                break;
            case 5:
                if (shouldRebuild) {
                    std::shared_ptr<Program> p;
                    res = compile(g, g.active ? g.active->nIn : (g.pending ? g.pending->nIn : 0), p);
                    if (res == rc::Ok) {                // rseqQueue.push(buildRenderSequence())
                        if (g.pending) g.superseded.push_back(g.pending);
                        g.pending = p;
                    }
                }
                break;
            default: break;
        }
        if (res != rc::Ok) return res;   // no rollback: Runtime.h:211-214
    }
    return rc::Ok;
}

bool Engine::isValueOnlyBatch(const std::vector<Value>& batch, int vb, int ve) {
    // A batch made only of SET_PROPERTY on per-voice-capable props (perVoiceProp) never changes the structure of a group, so it may
    // address any sub-range of voices without splitting the group.
    for (auto& ins : batch) {
        if (!ins.isArray()) return false;
        auto& ar = ins.asArray();
        if (ar.size() < 4 || !ar[0].isNumber() || static_cast<int>(ar[0].asNumber()) != 3) return false;
        int32_t id;
        if (!toInt32(ar[1], id) || !ar[2].isString() || !(ar[3].isNumber() || ar[3].isBool())) return false;
        for (auto& g : groups_) {
            if (g->v0 >= ve || g->v0 + g->nv <= vb) continue;
            auto it = g->nodes.find(id);
            if (it == g->nodes.end()) return false;
            const PerVoiceProp* p = perVoiceProp(it->second.kind, ar[2].asString());
            if (!p || (p->bits ? !ar[3].isNumber() : !ar[3].isBool())) return false;
        }
    }
    return true;
}

int Engine::splitGroupsAt(int v) {
    if (v <= 0 || v >= numVoices_) return rc::Ok;
    for (size_t i = 0; i < groups_.size(); ++i) {
        Group& g = *groups_[i];
        if (v <= g.v0 || v >= g.v0 + g.nv) continue;
        auto ng = std::make_unique<Group>();
        const int cut = v - g.v0;                       // first voice (group-relative) that moves to the new group
        ng->v0 = v; ng->nv = g.nv - cut; ng->Vpad = (ng->nv + 31) / 32 * 32;
        if (g.nodes.empty() && !g.dRows) {              // nothing to migrate
            g.nv = cut; g.Vpad = (g.nv + 31) / 32 * 32;
            groups_.insert(groups_.begin() + i + 1, std::move(ng));
            return rc::Ok;
        }
        // ---- the group is live: the voices [cut, nv) leave with a copy of the graph and THEIR device state -------
        // (dynamic graph updates at voice scale, SURVEY.md §8f N1: afterwards each half can be re-wired independently,
        // every voice keeping its phases, filter memories, delay lines and taps, like a Runtime of its own would.)
        const int L = g.tileWidth;
        if (L > 0 && cut % L != 0)
            return fail(rc::InvariantViolation, "voice groups can only be cut on a voice-tile boundary (multiple of the group's tile width)");
        dsync();
        ng->tileWidth = L;
        ng->currentRoots = g.currentRoots;
        // rows: column slice of every row; a double state is a row PAIR viewed as double[Vpad], sliced as doubles
        ng->rowsCap = g.rowsCap; ng->rowsUsed = g.rowsUsed;
        if (g.dRows && g.rowsCap > 0) {
            if (!cuda(dmalloc((void**) &ng->dRows, sizeof(float) * (size_t) ng->rowsCap * ng->Vpad), "cudaMalloc rows (split)")) return rc::CudaError;
            if (!cuda(dmemset(ng->dRows, 0, sizeof(float) * (size_t) ng->rowsCap * ng->Vpad), "memset rows (split)")) return rc::CudaError;
            std::vector<char> isDoublePair((size_t) g.rowsUsed + 2, 0);
            for (auto& kv : g.nodes) {
                const Node& n = kv.second;
                if (n.kind == NodeKind::Custom) continue;     // registered types keep float state only
                const auto& ti = typeTable().at(n.typeName);
                if (n.stateRow >= 0) for (int k = 0; k < ti.doubleRows; k += 2) isDoublePair[(size_t) n.stateRow + k] = 1;
            }
            for (int r = 0; r < g.rowsUsed; ++r) {
                if (isDoublePair[(size_t) r]) {
                    const float* src = g.dRows + (size_t) r * g.Vpad + (size_t) 2 * cut;
                    if (!cuda(dmemcpy(ng->dRows + (size_t) r * ng->Vpad, src, sizeof(double) * ng->nv, cudaMemcpyDeviceToDevice), "copy double row (split)")) return rc::CudaError;
                    ++r;   // the pair's second row is part of the same double array
                } else {
                    if (!cuda(dmemcpy(ng->dRows + (size_t) r * ng->Vpad, g.dRows + (size_t) r * g.Vpad + cut, sizeof(float) * ng->nv, cudaMemcpyDeviceToDevice), "copy row (split)")) return rc::CudaError;
                }
            }
        }
        // tile-structured buffers [tile][pos][L]: the moving voices are a contiguous run of tiles
        const size_t tile0 = L > 0 ? (size_t) cut / L : 0;
        const size_t newTiles = L > 0 ? (size_t) (ng->nv + L - 1) / L : 0;
        auto cloneTiles = [&](const float* src, size_t perTileFloats, float** dst) -> bool {
            *dst = nullptr;
            if (!src || newTiles == 0 || perTileFloats == 0) return true;
            const size_t n = newTiles * perTileFloats;
            if (!cuda(dmalloc((void**) dst, sizeof(float) * n), "cudaMalloc tile buffer (split)")) return false;
            return cuda(dmemcpy(*dst, src + tile0 * perTileFloats, sizeof(float) * n, cudaMemcpyDeviceToDevice), "copy tile buffer (split)");
        };
        for (auto& kv : g.tapShared) {
            float* d = nullptr;
            if (!cloneTiles(kv.second, (size_t) blockSize_ * L, &d)) return rc::CudaError;
            ng->tapShared[kv.first] = d;
        }
        for (auto& kv : g.nodes) {
            Node n = kv.second;   // host-side copy: props, inlets, fades, resource handles, row indices (same layout)
            n.ring = nullptr; n.tapPrivate = nullptr;
            // per-voice host vectors follow their voices: capture relays, the arrays sample and seq-family voices read (rows moved above)
            auto slice = [cut](auto& from, auto& to) {
                const size_t c = std::min<size_t>(cut, from.size());
                to.assign(from.begin() + c, from.end());
                from.resize(c);
            };
            slice(kv.second.relay, n.relay);
            slice(kv.second.voiceArrays, n.voiceArrays);
            if (kv.second.ring) {
                if (!cloneTiles(kv.second.ring, (size_t) kv.second.size * L, &n.ring)) return rc::CudaError;
                n.ringFloats = newTiles * (size_t) kv.second.size * L;
            }
            if (kv.second.tapPrivate && !cloneTiles(kv.second.tapPrivate, (size_t) blockSize_ * L, &n.tapPrivate)) return rc::CudaError;
            if (kv.second.conv) {
                auto cs = std::make_shared<ConvolverState>();
                std::string err;
                if (!convolver_clone_range(*kv.second.conv, cut, ng->nv, *cs, stream_, err)) return fail(rc::CudaError, err);
                n.conv = cs;
                // the old state keeps its (now partly unused) storage
                if (!convolver_truncate(*kv.second.conv, cut, stream_, err)) return fail(rc::CudaError, err);
            }
            ng->nodes.emplace(kv.first, std::move(n));
        }
        const bool hadActive = (bool) g.active, hadPending = (bool) g.pending;
        const int nIn = g.active ? g.active->nIn : (g.pending ? g.pending->nIn : 0);
        g.nv = cut;   // Vpad (the row stride) and the tile buffers of the old group stay as allocated
        Group* ngp = ng.get();
        groups_.insert(groups_.begin() + i + 1, std::move(ng));
        if (hadActive || hadPending) {   // the moved voices keep rendering the same sequence, now through their own program
            std::shared_ptr<Program> p;
            int rcode = compile(*ngp, nIn, p);
            if (rcode != rc::Ok) return rcode;
            if (hadActive && !hadPending) ngp->active = p; else ngp->pending = p;
        }
        return rc::Ok;
    }
    return rc::Ok;
}

int Engine::applyInstructions(int vb, int ve, const char* json, size_t len) {
    Value doc;
    bool parsed = true;
    std::string parseError;
    try {
        doc = parseJson(json, len);           // outside the lock: the render thread never waits for a JSON parse
    } catch (const std::exception& e) {   // the reference throws here (JSON.h:146-154); the C ABI maps it to a code
        parsed = false; parseError = e.what();
    }
    Lock lk(mu_);
    dsetdev();
    if (vb < 0) vb = 0;
    if (ve < 0 || ve > numVoices_) ve = numVoices_;
    if (vb >= ve) return fail(rc::BadArgument, "empty voice range");
    if (!parsed) return fail(rc::InvalidInstructionFormat, parseError);
    lastError_.clear();
    if (!doc.isArray()) return fail(rc::InvalidInstructionFormat, "batch is not an array");
    return applyBatch(vb, ve, doc.asArray());
}

int Engine::applyBatch(int vb, int ve, const std::vector<Value>& batch) {
    steadyValid_ = false;
    if (!isValueOnlyBatch(batch, vb, ve)) {
        int r = splitGroupsAt(vb);
        if (r != rc::Ok) return r;
        if ((r = splitGroupsAt(ve)) != rc::Ok) return r;
    }
    for (auto& g : groups_) {
        const int b = std::max(vb, g->v0), e = std::min(ve, g->v0 + g->nv);
        if (b >= e) continue;
        int r = applyToGroup(*g, batch, b - g->v0, e - g->v0);
        if (r != rc::Ok) { if (lastError_.empty()) lastError_ = "instruction failed"; return r; }
    }
    return rc::Ok;
}

// Binary instruction batch (include/elem_b200.h "binary batch format"): little-endian, unaligned.
namespace {
struct BinReader {
    const unsigned char* p; const unsigned char* end; bool ok = true;
    template <typename T> T get() { T v{}; if ((size_t) (end - p) < sizeof(T)) { ok = false; return v; } std::memcpy(&v, p, sizeof(T)); p += sizeof(T); return v; }
    std::string str(size_t n) { if ((size_t) (end - p) < n) { ok = false; return std::string(); } std::string s(reinterpret_cast<const char*>(p), n); p += n; return s; }
};
}

int Engine::applyBinary(int vb, int ve, const void* data, size_t bytes) {
    BinReader r{static_cast<const unsigned char*>(data), static_cast<const unsigned char*>(data) + bytes};
    if (r.get<uint32_t>() != 0x49324245u /* "EB2I" */ || r.get<uint32_t>() != 1u) { Lock lk(mu_); return fail(rc::InvalidInstructionFormat, "binary batch: bad magic or version"); }
    const uint32_t count = r.get<uint32_t>();
    std::vector<Value> batch;
    batch.reserve(count);
    for (uint32_t i = 0; i < count && r.ok; ++i) {          // decoded outside the lock, like the JSON text
        Value ins = Value::array();
        auto& a = ins.asArray();
        const uint8_t op = r.get<uint8_t>();
        a.push_back(Value::number(op));
        switch (op) {
            case 0: { const int32_t id = r.get<int32_t>(); const uint16_t n = r.get<uint16_t>(); a.push_back(Value::number(id)); a.push_back(Value::string(r.str(n))); } break;
            case 2: { for (int k = 0; k < 3; ++k) a.push_back(Value::number(r.get<int32_t>())); } break;
            case 3: {
                const int32_t id = r.get<int32_t>(); const uint16_t n = r.get<uint16_t>();
                a.push_back(Value::number(id)); a.push_back(Value::string(r.str(n)));
                const uint8_t vt = r.get<uint8_t>();
                switch (vt) {
                    case 0: a.push_back(Value::null()); break;
                    case 1: a.push_back(Value::boolean(r.get<uint8_t>() != 0)); break;
                    case 2: a.push_back(Value::number(r.get<double>())); break;
                    case 3: { const uint32_t len = r.get<uint32_t>(); a.push_back(Value::string(r.str(len))); } break;
                    case 4: { const uint32_t len = r.get<uint32_t>(); Value arr = Value::array(); arr.asArray().reserve(len);
                              for (uint32_t k = 0; k < len && r.ok; ++k) arr.asArray().push_back(Value::number(r.get<float>())); a.push_back(arr); } break;
                    case 5: { const uint32_t len = r.get<uint32_t>(); const std::string js = r.str(len);      // anything else travels as JSON text
                              try { a.push_back(parseJson(js.data(), js.size())); } catch (const std::exception&) { r.ok = false; } } break;
                    default: r.ok = false; break;
                }
            } break;
            case 4: { const uint32_t n = r.get<uint32_t>(); Value roots = Value::array(); for (uint32_t k = 0; k < n && r.ok; ++k) roots.asArray().push_back(Value::number(r.get<int32_t>())); a.push_back(roots); } break;
            case 5: break;
            default: r.ok = false; break;
        }
        batch.push_back(std::move(ins));
    }
    Lock lk(mu_);
    dsetdev();
    if (!r.ok) return fail(rc::InvalidInstructionFormat, "binary batch: truncated or malformed");
    if (vb < 0) vb = 0;
    if (ve < 0 || ve > numVoices_) ve = numVoices_;
    if (vb >= ve) return fail(rc::BadArgument, "empty voice range");
    lastError_.clear();
    return applyBatch(vb, ve, batch);
}

// The targets of a per-voice call, every check done before anything changes: the range, the node in every group, its kind.
template <class KindOk>
int Engine::voiceTargets(int32_t nodeId, int vb, int count, KindOk kindOk, const char* kindError, std::vector<VoiceTarget>& out) {
    out.clear();
    if (!voiceRangeOk(vb, count, numVoices_)) return fail(rc::BadArgument, "voice range out of bounds");
    for (auto& gp : groups_) {
        Group& g = *gp;
        const int b = std::max(vb, g.v0), e = std::min(vb + count, g.v0 + g.nv);
        if (b >= e) continue;
        auto it = g.nodes.find(nodeId);
        if (it == g.nodes.end()) { out.clear(); return fail(rc::NodeNotFound, "node not found"); }
        if (!kindOk(it->second.kind)) { out.clear(); return fail(rc::InvalidPropertyType, kindError); }
        out.push_back(VoiceTarget{g, it->second, b - g.v0, e - g.v0, b - vb});
    }
    return rc::Ok;
}

// The checks of an array poll of one node (pollReadouts, processOfflineReadouts): the range, the node in every group, a meter or a snapshot,
// and the same one of the two in every group (the arrays mean one thing).
int Engine::readoutTargets(int32_t nodeId, int vb, int count, std::vector<VoiceTarget>& out) {
    const int r = voiceTargets(nodeId, vb, count, [](NodeKind k) { return k == NodeKind::Meter || k == NodeKind::Snapshot; },
                               "readouts are polled from meter and snapshot nodes", out);
    if (r != rc::Ok) return r;
    for (const VoiceTarget& t : out)
        if (t.n.kind != out.front().n.kind) { out.clear(); return fail(rc::InvalidPropertyType, "the node is a meter in one voice group and a snapshot in another"); }
    return rc::Ok;
}

std::string Engine::nodeType(int voice, int32_t nodeId) const {
    Lock lk(mu_);
    for (auto& g : groups_) {
        if (voice < g->v0 || voice >= g->v0 + g->nv) continue;
        auto it = g->nodes.find(nodeId);
        return it == g->nodes.end() ? std::string() : it->second.typeName;
    }
    return std::string();
}

int Engine::setConstTable(const int32_t* nodeIds, int nProps, const float* values, int vb, int count) {
    Lock lk(mu_);
    dsetdev();
    if (nProps < 0 || !voiceRangeOk(vb, count, numVoices_)) return fail(rc::BadArgument, "voice range out of bounds");
    // every check before any change: a failed call changes nothing
    std::vector<std::vector<VoiceTarget>> targets((size_t) nProps);
    for (int p = 0; p < nProps; ++p) {
        const int r = voiceTargets(nodeIds[p], vb, count, [](NodeKind k) { return k == NodeKind::Const; },
                                   "property table rows must address const nodes", targets[(size_t) p]);
        if (r != rc::Ok) return r;
    }
    for (int p = 0; p < nProps; ++p)
        for (auto& t : targets[(size_t) p]) {
            const float* src = values + (size_t) p * count;
            const int r = writeColumns(t.g, t.n.paramRow, 1, t.b, t.e - t.b, src + t.at, "property table upload");
            if (r != rc::Ok) return r;
            t.n.props["value"] = Value::number(src[t.last()]);
        }
    return rc::Ok;
}

int Engine::setPropertyPerVoice(int32_t nodeId, const char* key, const double* values, int vb, int count) {
    Lock lk(mu_);
    // Vectorised SET_PROPERTY (SURVEY.md §8f N2): values[i] goes to voice vb+i. Same semantics as `count`
    // single-voice [3,id,key,value] batches, without `count` JSON parses.
    dsetdev();
    const std::string k(key);
    // every check before any change: a failed call changes nothing
    std::vector<VoiceTarget> targets;
    int r = voiceTargets(nodeId, vb, count, [&](NodeKind kind) { const PerVoiceProp* p = perVoiceProp(kind, k); return p && p->bits; },
                         "property is not per-voice capable", targets);
    if (r != rc::Ok || targets.empty()) return r;
    const PerVoiceProp& prop = *perVoiceProp(targets[0].n.kind, k);   // the key names one kind
    std::vector<uint32_t> bits((size_t) count);
    for (int i = 0; i < count; ++i)
        if (!prop.bits(values[i], bits[(size_t) i])) return fail(rc::InvalidPropertyValue, "sample offsets must not be negative");
    for (auto& t : targets) {
        for (int row : {t.n.*prop.base + prop.row, prop.shadow ? t.n.shadowRow : -1})
            if (row >= 0 && (r = writeColumns(t.g, row, 1, t.b, t.e - t.b, bits.data() + t.at, "per-voice prop upload")) != rc::Ok) return r;
        t.n.props[k] = Value::number(values[t.last()]);
    }
    return rc::Ok;
}

int Engine::setPathPerVoice(int32_t nodeId, const char* const* names, int numNames, const int32_t* index, int vb, int count) {
    Lock lk(mu_);
    dsetdev();
    if (numNames < 0) return fail(rc::BadArgument, "voice range out of bounds");
    for (int i = 0; i < count; ++i)
        if (index[i] < 0 || index[i] >= numNames) return fail(rc::BadArgument, "name index out of range");
    // every check before any change: a failed call changes nothing
    std::vector<VoiceTarget> targets;
    const int rt = voiceTargets(nodeId, vb, count, [](NodeKind k) { return k == NodeKind::Convolve || k == NodeKind::Sample; },
                                "property is not per-voice capable", targets);
    if (rt != rc::Ok) return rt;
    std::vector<std::shared_ptr<Resource>> res((size_t) numNames);
    for (int k = 0; k < numNames; ++k) {
        auto it = names[k] ? resources_.find(names[k]) : resources_.end();
        if (it == resources_.end()) return fail(rc::InvalidPropertyValue, std::string("no shared resource named ") + (names[k] ? names[k] : "(null)"));
        res[(size_t) k] = it->second;
    }
    if (count == 0) return rc::Ok;
    steadyValid_ = false;
    std::vector<std::shared_ptr<IrSpectra>> spectra((size_t) numNames);   // computed (or found in the bank) once per name
    auto spectraOf = [&](int k, std::string& err) -> std::shared_ptr<IrSpectra> {
        if (!spectra[(size_t) k]) {
            const Resource& r = *res[(size_t) k];
            static const std::vector<float> none;
            const auto& ch0 = r.channels.empty() ? none : r.channels[0];
            spectra[(size_t) k] = irBank_.acquire(&r, res[(size_t) k], ch0.data(), ch0.size(), planOnly_, stream_, err);
        }
        return spectra[(size_t) k];
    };
    for (auto& t : targets) {
        Group& g = t.g;
        Node& n = t.n;
        const int last = index[t.last()];
        if (n.kind == NodeKind::Sample) {
            const int r = assignSampleBuffers(g, n, res, index + t.at, t.b, t.e);
            if (r != rc::Ok) return r;
            n.props["path"] = Value::string(names[last]);
            continue;
        }
        std::string err;
        const bool hadResource = (bool) n.resource;
        if (n.resourceDirty || !n.conv) {
            // the whole-group state the next compile would have made (a fresh convolver on the node's `path`, or none: silence)
            auto cs = std::make_shared<ConvolverState>();
            static const std::vector<float> none;
            const auto& ch0 = (!n.resource || n.resource->channels.empty()) ? none : n.resource->channels[0];
            if (!convolver_init(*cs, irBank_, n.resource.get(), n.resource, ch0.data(), ch0.size(), g.nv, planOnly_, stream_, err)) return fail(rc::CudaError, err);
            n.conv = cs;
            n.resourceDirty = false;
        }
        std::vector<std::shared_ptr<IrSpectra>> h((size_t) (t.e - t.b));
        for (int i = 0; i < t.e - t.b; ++i)
            if (!(h[(size_t) i] = spectraOf(index[t.at + i], err))) return fail(rc::CudaError, err);
        if (!convolver_assign(*n.conv, t.b, t.e - t.b, h, stream_, err)) return fail(rc::CudaError, err);
        n.resource = res[(size_t) last];
        n.props["path"] = Value::string(names[last]);
        if (!hadResource) g.codeDirty = true;   // the program emitted silence for a convolver without an IR
    }
    return rc::Ok;
}

int Engine::resetVoices(const int32_t* voices, size_t count) {
    Lock lk(mu_);
    dsetdev();
    if (count == 0) return rc::Ok;
    if (!voices) return fail(rc::BadArgument, "resetVoices: null voice list");
    std::vector<int32_t> vs(voices, voices + count);
    for (int32_t v : vs)
        if (v < 0 || v >= numVoices_) return fail(rc::BadArgument, "resetVoices: voice index out of range");
    std::sort(vs.begin(), vs.end());
    vs.erase(std::unique(vs.begin(), vs.end()), vs.end());

    // runs: the voices of one voice tile; the groups they touch, in voice order
    std::vector<int> runStart, runGroup;
    std::vector<Group*> touched;
    std::vector<int> touchedFirst;   // index in vs of each touched group's first voice
    size_t gi = 0;
    int lastTile = -1;
    for (size_t i = 0; i < vs.size(); ++i) {
        const int v = vs[i];
        while (v >= groups_[gi]->v0 + groups_[gi]->nv) ++gi;
        Group& g = *groups_[gi];
        const int tile = (v - g.v0) / std::max(1, g.tileWidth);
        if (touched.empty() || touched.back() != &g) { touched.push_back(&g); touchedFirst.push_back((int) i); lastTile = -1; }
        if (tile != lastTile) { runStart.push_back((int) i); runGroup.push_back((int) touched.size() - 1); lastTile = tile; }
    }
    runStart.push_back((int) vs.size());
    touchedFirst.push_back((int) vs.size());

    // the reset plans of the touched groups (fresh state: freshRowBits / shadowedRow)
    std::vector<ResetGroup> pg;
    std::vector<ResetBuf> pb;
    std::vector<ResetConv> pc;
    std::vector<ResetRow> pr;
    for (size_t t = 0; t < touched.size(); ++t) {
        Group& g = *touched[t];
        ResetGroup G{};
        G.rows = g.dRows; G.v0 = g.v0; G.Vpad = g.Vpad; G.L = std::max(1, g.tileWidth);
        G.row0 = (int) pr.size(); G.buf0 = (int) pb.size(); G.conv0 = (int) pc.size();
        auto addBuf = [&](float* base, long long positions) {
            if (!base || positions <= 0) return;
            pb.push_back(ResetBuf{base, positions, G.tilePositions});
            G.tilePositions += positions;
        };
        std::vector<Node*> nodes;
        for (auto& kv : g.nodes) nodes.push_back(&kv.second);
        std::sort(nodes.begin(), nodes.end(), [](const Node* a, const Node* b) { return a->id < b->id; });
        for (Node* np : nodes) {
            Node& n = *np;
            if (n.stateRow >= 0) {
                const bool custom = n.kind == NodeKind::Custom;
                const int rows = custom ? customTypes_[n.fn].nState : typeTable().at(n.typeName).stateRows;
                const int dblRows = custom ? 0 : typeTable().at(n.typeName).doubleRows;
                for (int k = 0; k < rows;) {
                    const bool dbl = k < dblRows;
                    if (dbl) pr.push_back(ResetRow{n.stateRow + k, RESET_ROW_DOUBLE, 0u});
                    else if (k == shadowedRow(n.kind)) pr.push_back(ResetRow{n.stateRow + k, RESET_ROW_SHADOW, (uint32_t) n.shadowRow});
                    else pr.push_back(ResetRow{n.stateRow + k, RESET_ROW_BITS, freshRowBits(n.kind, k)});
                    k += dbl ? 2 : 1;
                }
            }
            addBuf(n.ring, n.ringPositions);
            addBuf(n.tapPrivate, blockSize_);
            if (n.conv)
                for (const ConvRegion& r : convolver_channel_regions(*n.conv)) {
                    const long long quads = (long long) (r.bytesPerChannel / sizeof(float4));
                    pc.push_back(ResetConv{static_cast<float*>(r.base), quads, G.convQuads});
                    G.convQuads += quads;
                }
            for (int i = touchedFirst[t]; i < touchedFirst[t + 1] && !n.relay.empty(); ++i) {   // the host-side capture relays
                const size_t u = (size_t) (vs[(size_t) i] - g.v0);
                if (u < n.relay.size()) n.relay[u].clear();
            }
        }
        for (auto& kv : g.tapShared) addBuf(kv.second, blockSize_);
        G.nRows = (int) pr.size() - G.row0; G.nBufs = (int) pb.size() - G.buf0; G.nConvs = (int) pc.size() - G.conv0;
        pg.push_back(G);
    }

    // one blob: groups, buffers, convolver regions, rows (8-byte aligned parts first); uploaded only when it changed
    const size_t offB = pg.size() * sizeof(ResetGroup), offC = offB + pb.size() * sizeof(ResetBuf),
                 offR = offC + pc.size() * sizeof(ResetConv), planBytes = offR + pr.size() * sizeof(ResetRow);
    std::vector<char> blob(planBytes);
    std::memcpy(blob.data(), pg.data(), offB);
    if (!pb.empty()) std::memcpy(blob.data() + offB, pb.data(), offC - offB);
    if (!pc.empty()) std::memcpy(blob.data() + offC, pc.data(), offR - offC);
    if (!pr.empty()) std::memcpy(blob.data() + offR, pr.data(), planBytes - offR);
    char* const oldPlan = dResetPlan_;
    if (!grow(dResetPlan_, resetPlanCap_, planBytes, "cudaMalloc reset plan", false, 2)) return rc::CudaError;
    if (dResetPlan_ != oldPlan || blob != resetPlanUp_) {
        if (!cuda(dmemcpy(dResetPlan_, blob.data(), planBytes, cudaMemcpyHostToDevice), "upload reset plan")) { resetPlanUp_.clear(); return rc::CudaError; }
        resetPlanUp_.swap(blob);
    }
    // the call: voices, run starts, run groups
    const size_t nRuns = runGroup.size();
    std::vector<int> call;
    call.reserve(vs.size() + 2 * nRuns + 1);
    call.insert(call.end(), vs.begin(), vs.end());
    call.insert(call.end(), runStart.begin(), runStart.end());
    call.insert(call.end(), runGroup.begin(), runGroup.end());
    if (!grow(dResetCall_, resetCallCap_, call.size(), "cudaMalloc reset voices", false, 2)) return rc::CudaError;
    if (!cuda(dmemcpy(dResetCall_, call.data(), sizeof(int) * call.size(), cudaMemcpyHostToDevice), "upload reset voices")) return rc::CudaError;   // pageable: staged before the call returns

    // the slices of a run: about 2048 items per CTA for the run with the most work
    long long maxWork = 0;
    for (size_t r = 0; r < nRuns; ++r) {
        const ResetGroup& G = pg[(size_t) runGroup[r]];
        const long long m = runStart[r + 1] - runStart[r];
        maxWork = std::max(maxWork, m * (G.nRows + G.tilePositions + G.convQuads));
        long long bytes = m * (G.tilePositions * 4 + G.convQuads * 16);
        for (int k = 0; k < G.nRows; ++k) bytes += m * (pr[(size_t) (G.row0 + k)].kind == RESET_ROW_DOUBLE ? 8 : 4);
        resetBytes_ += (uint64_t) bytes;
    }
    const int slices = (int) std::min<long long>(65535, std::max<long long>(1, (maxWork + 2047) / 2048));
    ResetLaunch a;
    a.groups = reinterpret_cast<const ResetGroup*>(dResetPlan_);
    a.bufs = reinterpret_cast<const ResetBuf*>(dResetPlan_ + offB);
    a.convs = reinterpret_cast<const ResetConv*>(dResetPlan_ + offC);
    a.rows = reinterpret_cast<const ResetRow*>(dResetPlan_ + offR);
    a.voices = dResetCall_;
    a.runStart = dResetCall_ + vs.size();
    a.runGroup = dResetCall_ + vs.size() + nRuns + 1;
    if (!planOnly_ && !cuda(launch_reset_voices(a, (int) nRuns, slices, stream_), "reset kernel launch")) return rc::CudaError;
    ++launches_;
    return rc::Ok;
}

int Engine::gc(int voice, std::vector<int32_t>& pruned) {
    Lock lk(mu_);   // Runtime.h:221-272
    pruned.clear();
    for (auto& gp : groups_) {
        Group& g = *gp;
        if (voice < g.v0 || voice >= g.v0 + g.nv) continue;
        std::set<int32_t> live;
        if (g.active) live.insert(g.active->nodeIds.begin(), g.active->nodeIds.end());
        if (g.pending) live.insert(g.pending->nodeIds.begin(), g.pending->nodeIds.end());
        for (auto& q : g.superseded) live.insert(q->nodeIds.begin(), q->nodeIds.end());
        dsync();
        for (auto it = g.nodes.begin(); it != g.nodes.end();) {
            if (!live.count(it->first)) {
                pruned.push_back(it->first);
                if (it->second.ring) dfree(it->second.ring);
                if (it->second.tapPrivate) dfree(it->second.tapPrivate);
                it = g.nodes.erase(it);
            } else ++it;
        }
    }
    std::sort(pruned.begin(), pruned.end());
    return rc::Ok;
}

void Engine::reset() {
    Lock lk(mu_);
    // Runtime.h:449-458: only SampleNode does anything on reset(): noteOff on both readers (their target gains)
    dsetdev();
    for (auto& gp : groups_)
        for (auto& kv : gp->nodes)
            if (kv.second.kind == NodeKind::Sample)
                for (int k : {SAMPLE_TARGET_GAIN0, SAMPLE_TARGET_GAIN1}) fillRowBits(*gp, kv.second.stateRow + k, 0, gp->nv, 0u);
}

// Voice vb + i (group-relative, i < ve - vb) of sample node n plays res[index[i]] from the next block on with fresh readers
// (Sample.h:94-99: gain 0, target 0, pos 0); currentReader and change.lastIn are kept.
int Engine::assignSampleBuffers(Group& g, Node& n, const std::vector<std::shared_ptr<Resource>>& res, const int32_t* index, int vb, int ve) {
    const int cnt = ve - vb;
    if (cnt <= 0) return rc::Ok;
    std::vector<VoiceArray> arrs;
    for (auto& r : res) {
        const int e = ensureResourceOnDevice(*r);
        if (e != rc::Ok) return e;
        arrs.push_back(VoiceArray{r, (uint64_t) (uintptr_t) r->dChannel0, (uint32_t) r->numSamples + 1u});
    }
    int e = assignVoiceArrays(g, n, arrs, index, vb, ve);
    if (e != rc::Ok) return e;
    // the readers: positions are double rows (2 * vb ..), then the gain rows
    for (int k : {SAMPLE_POS0, SAMPLE_POS1})
        if (!cuda(dmemset(g.dRows + (size_t) (n.stateRow + k) * g.Vpad + 2 * (size_t) vb, 0, sizeof(double) * cnt), "sample reader reset")) return rc::CudaError;
    for (int k = SAMPLE_TARGET_GAIN0; k < SAMPLE_GAINS_END; ++k)
        if ((e = fillRowBits(g, n.stateRow + k, vb, ve, 0u)) != rc::Ok) return e;
    return rc::Ok;
}

// ---------------------------------------------------------------------------------------------------------
// compile: sorted node list -> render program
int Engine::chooseTileWidth(int nv) const {
    if (opt_.tileWidth > 0) {
        int L = 1;
        while (L * 2 <= std::min(32, opt_.tileWidth)) L *= 2;
        return L;
    }
    const int target = midRangeDense(nv) ? 4096 : opt_.targetTiles;
    int L = 32;
    while (L > 1 && (nv + L - 1) / L < target) L >>= 1;
    return L;
}

void Engine::traverse(Group& g, std::set<int32_t>& visited, std::vector<int32_t>& order, int32_t n) {   // Runtime.h:503-518
    if (visited.count(n)) return;
    // A cycle would recurse forever in the reference; break it by marking the node before descending when we
    // see it again on the stack (front ends never emit cycles).
    static thread_local std::set<int32_t> onStack;
    if (onStack.count(n)) return;
    onStack.insert(n);
    auto it = g.nodes.find(n);
    if (it != g.nodes.end())
        for (auto& in : it->second.inlets) traverse(g, visited, order, in.source);
    onStack.erase(n);
    order.push_back(n);
    visited.insert(n);
}

constexpr uint32_t OP_HOST_CONV = 0xF0;   // host-only pseudo opcode of a Convolve node: lowered to STOREBUF + K3 + LOADBUF by the stage split

struct Compiler {
    Engine& E;
    Group& g;
    int nIn;
    Program& prog;

    struct PendingOp {
        uint32_t opcode = 0, mode = 0, state = NO_STATE, aux0 = 0, aux1 = 0;
        uint64_t ptr = 0;
        int32_t outNode = 0;               // node whose output this op produces (0x7fffffff+k for temporaries)
        std::vector<std::pair<uint32_t, int32_t>> operands;   // (kind, node id | param row)
        struct Step { uint32_t fn; uint32_t kind; int32_t ref; };   // OP_CHAIN: acc = fn(acc, operand) / fn(acc)
        std::vector<Step> steps;
        std::vector<uint32_t> imm;         // raw immediate words behind the operands (control nodes)
        int slot = 0;                      // output slot (allocateSlots)
        bool dead = false;                 // absorbed into a later chain
    };
    using Segments = std::vector<std::vector<PendingOp>>;   // one op list per root, indexed by root index: the root's sub-sequence
    Segments segs;
    std::vector<std::pair<int, int32_t>> promotes;   // (root index, tapOut node id)
    int32_t tempCounter = 0;

    int32_t newTemp() { return INT32_MIN + (++tempCounter); }

    // device floats, zeroed; false with lastError set when CUDA fails
    bool zeroedFloats(float*& p, size_t floats, const char* what) {
        return E.cuda(E.dmalloc((void**) &p, sizeof(float) * floats), what) && E.cuda(E.dmemset(p, 0, sizeof(float) * floats), what);
    }

    template <class F> static void forEachSlotUse(const PendingOp& op, F&& f) {   // in operand order
        for (auto& o : op.operands) if (o.first == K_SLOT) f(o.second);
        for (auto& st : op.steps) if (!chain_fn_is_unary(st.fn) && st.kind == K_SLOT) f(st.ref);
    }

    // The values read in a later cut than the one that produced them, in order of first use (ring and buffer indices follow that
    // order into the program words).  cut(s, i) is the cut (K1 stage, warp pipeline stage) of op i of segment s.
    template <class Cut> static std::vector<int32_t> crossingValues(const Segments& segs, Cut cut) {
        std::unordered_map<int32_t, int> producedIn;
        for (size_t s = 0; s < segs.size(); ++s)
            for (size_t i = 0; i < segs[s].size(); ++i) producedIn[segs[s][i].outNode] = cut(s, i);
        std::vector<int32_t> crossing;
        std::unordered_set<int32_t> seen;
        for (size_t s = 0; s < segs.size(); ++s)
            for (size_t i = 0; i < segs[s].size(); ++i)
                forEachSlotUse(segs[s][i], [&](int32_t id) {
                    auto p = producedIn.find(id);
                    if (p != producedIn.end() && p->second < cut(s, i) && seen.insert(id).second) crossing.push_back(id);
                });
        return crossing;
    }

    // Slots by liveness, one linear scan over a section's ops in order: an op's output takes the slot freed last (or a new one) before
    // its operands' slots are freed, so it never shares a slot with one of its own inputs; an operand's slot is freed after its last use
    // in the section, operands in order, and an output nobody reads in the section at once.  Values in `ring` get no slot here.  Slots
    // are numbered from `base`; returns how many were taken.
    static int allocateSlots(Segments& section, const std::unordered_map<int32_t, int>& ring, int base) {
        std::unordered_map<int32_t, size_t> lastUse;
        size_t i = 0;
        for (auto& ops : section)
            for (auto& op : ops) { forEachSlotUse(op, [&](int32_t id) { lastUse[id] = i; }); ++i; }
        std::unordered_map<int32_t, int> slotOf;
        std::vector<int> freeSlots;
        int n = 0;
        i = 0;
        for (auto& ops : section)
            for (auto& op : ops) {
                const bool inRing = ring.count(op.outNode) != 0;
                if (!inRing) {
                    int s = n;
                    if (!freeSlots.empty()) { s = freeSlots.back(); freeSlots.pop_back(); }
                    else ++n;
                    op.slot = base + s;
                    slotOf[op.outNode] = s;
                }
                forEachSlotUse(op, [&](int32_t id) {
                    auto so = slotOf.find(id);
                    if (so != slotOf.end() && lastUse[id] == i) { freeSlots.push_back(so->second); slotOf.erase(so); }
                });
                if (!inRing && !lastUse.count(op.outNode)) { freeSlots.push_back(op.slot - base); slotOf.erase(op.outNode); }
                ++i;
            }
        return n;
    }

    static void putDouble(PendingOp& op, double d) {
        uint64_t b;
        std::memcpy(&b, &d, 8);
        op.aux0 = (uint32_t) b; op.aux1 = (uint32_t) (b >> 32);
    }
    static uint32_t fbits(float f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }

    std::pair<uint32_t, int32_t> operandFor(const Inlet& in) {
        auto it = g.nodes.find(in.source);
        if (it == g.nodes.end() || in.channel != 0) return {K_ZERO, 0};
        const Node& c = it->second;
        if (c.kind == NodeKind::Const || c.kind == NodeKind::Sr) return {K_PARAM, c.paramRow};
        return {K_SLOT, c.id};
    }

    int emitNode(Node& n, int rootIndex);
};

int Compiler::emitNode(Node& n, int rootIndex) {
    if (n.kind == NodeKind::Const || n.kind == NodeKind::Sr) return rc::Ok;   // folded into PARAM operands

    std::vector<PendingOp>& ops = segs[(size_t) rootIndex];
    const bool leaf = n.inlets.empty();
    const bool sourceNode = n.kind == NodeKind::Rand || n.kind == NodeKind::TapIn || n.kind == NodeKind::Time || n.kind == NodeKind::Metro;
    if (leaf && !sourceNode) prog.usesHostInputs = true;
    // Inputs as the node's process() sees them: children, or — for a leaf — the host input channels
    // (GraphRenderSequence.h:126-135).
    std::vector<std::pair<uint32_t, int32_t>> inputs;
    if (!leaf) {
        for (auto& in : n.inlets) inputs.push_back(operandFor(in));
    } else if (n.kind != NodeKind::In && !sourceNode) {
        for (int ch = 0; ch < nIn; ++ch) {
            PendingOp ld;
            ld.opcode = OP_LOADIN; ld.aux0 = (uint32_t) ch; ld.outNode = newTemp();
            ops.push_back(ld);
            inputs.push_back({K_SLOT, ld.outNode});
            prog.usesHostInputs = true;
        }
    }
    const int numCh = leaf ? nIn : (int) n.inlets.size();

    bool evNode = n.kind == NodeKind::Metro;
    PendingOp op;
    op.outNode = n.id;
    op.state = (n.stateRow >= 0) ? (uint32_t) n.stateRow : NO_STATE;   // rewritten to a smem index later
    auto zeros = [&]() { op.opcode = OP_FILL0; op.state = NO_STATE; op.operands.clear(); };
    auto take = [&](int k) { op.operands.assign(inputs.begin(), inputs.begin() + k); };
    // The seq family reads the group's sequence (ptr = data, aux0 = count), or after setSeqPerVoice each voice's own: mode bit 3 and four
    // parameter rows after the inputs (data pointer low / high word, count, generation).  A voice without a sequence reads count 0.
    auto seqSource = [&]() {
        if (n.paramRow >= 0) { op.mode |= 8u; for (int k = 0; k < SEQ_PARAM_ROWS; ++k) op.operands.push_back({K_PARAM, n.paramRow + k}); }
        else if (n.seqData) { op.aux0 = (uint32_t) n.seqData->count; op.ptr = (uint64_t) (uintptr_t) n.seqData->d; prog.pinned.push_back(n.seqData); }
    };

    switch (n.kind) {
        case NodeKind::In: {   // Math.h:107-122
            const int ch = n.channel;
            if (ch < 0 || ch >= numCh) { zeros(); break; }
            if (leaf) { op.opcode = OP_LOADIN; op.aux0 = (uint32_t) ch; prog.usesHostInputs = true; }
            else { op.opcode = OP_COPY; op.operands = {operandFor(n.inlets[ch])}; }
        } break;
        // Math.h:9-89 — element-wise nodes become one-node chains; fuseChains() merges runs of them
        case NodeKind::Unary:
            if (numCh < 1) { zeros(); break; }
            op.opcode = OP_CHAIN; take(1); op.steps.push_back({n.fn, K_ZERO, 0});
            break;
        case NodeKind::Binary:
            if (numCh < 2) { zeros(); break; }
            op.opcode = OP_CHAIN; take(1); op.steps.push_back({n.fn, inputs[1].first, inputs[1].second});
            break;
        case NodeKind::Reduce:   // left fold over the children in order (Math.h:71-84)
            if (numCh < 1) { zeros(); break; }
            op.opcode = OP_CHAIN; take(1);
            for (int j = 1; j < numCh; ++j) op.steps.push_back({n.fn, inputs[j].first, inputs[j].second});
            break;
        case NodeKind::Root:
            op.opcode = OP_ROOT; op.aux0 = (uint32_t) rootIndex;
            if (numCh >= 1) take(1);
            break;
        case NodeKind::Phasor:
            if (numCh < 1) { zeros(); break; }
            op.opcode = OP_PHASOR; op.aux0 = fbits(1.0f / (float) E.sr_); take(1);   // Core.h:90
            break;
        case NodeKind::SPhasor:
            if (numCh < 2) { zeros(); break; }
            op.opcode = OP_SPHASOR; op.aux0 = fbits(1.0f / (float) E.sr_); take(2);
            break;
        case NodeKind::Counter: if (numCh < 1) { zeros(); break; } op.opcode = OP_COUNTER; take(1); break;
        case NodeKind::Accum: if (numCh < 2) { zeros(); break; } op.opcode = OP_ACCUM; take(2); break;
        case NodeKind::Latch: if (numCh < 2) { zeros(); break; } op.opcode = OP_LATCH; take(2); break;
        case NodeKind::MaxHold: if (numCh < 2) { zeros(); break; } op.opcode = OP_MAXHOLD; op.aux0 = n.holdSamples; take(2); break;
        case NodeKind::Rand: op.opcode = OP_RAND; break;
        case NodeKind::Pole: if (numCh < 2) { zeros(); break; } op.opcode = OP_POLE; take(2); break;
        case NodeKind::Env: if (numCh < 3) { zeros(); break; } op.opcode = OP_ENV; take(3); break;
        case NodeKind::Biquad: if (numCh < 6) { zeros(); break; } op.opcode = OP_BIQUAD; take(6); break;
        case NodeKind::Prewarp: if (numCh < 1) { zeros(); break; } op.opcode = OP_PREWARP; putDouble(op, 1.0 / E.sr_); take(1); break;
        case NodeKind::MM1p: if (numCh < 2) { zeros(); break; } op.opcode = OP_MM1P; op.mode = (uint32_t) n.mode; take(2); break;
        case NodeKind::Svf: if (numCh < 3) { zeros(); break; } op.opcode = OP_SVF; op.mode = (uint32_t) n.mode; putDouble(op, E.sr_); take(3); break;
        case NodeKind::SvfShelf: if (numCh < 4) { zeros(); break; } op.opcode = OP_SVFSHELF; op.mode = (uint32_t) n.mode; putDouble(op, E.sr_); take(4); break;
        case NodeKind::Z: if (numCh < 1) { zeros(); break; } op.opcode = OP_Z; take(1); break;
        case NodeKind::Blep:
            if (numCh < 1) { zeros(); break; }
            op.opcode = OP_BLEP; op.mode = n.fn; op.aux0 = fbits((float) E.sr_); take(1);
            break;
        case NodeKind::PassThrough: if (numCh < 1) { zeros(); break; } op.opcode = OP_COPY; take(1); break;
        case NodeKind::Custom: {   // a registered device node type: missing inputs give zeros like every builtin
            const auto& ct = E.customTypes_[n.fn];
            if (numCh < ct.nIn) { zeros(); break; }
            op.opcode = OP_CUSTOM; op.aux0 = n.fn; op.aux1 = (uint32_t) ct.nState; take(ct.nIn);
            op.imm = {fbits((float) E.sr_)};
            prog.hasCustom = true;
        } break;


        // ---- sequencing / control nodes (SURVEY.md §8f N3) ----
        case NodeKind::Once: if (numCh < 1) { zeros(); break; } op.opcode = OP_ONCE; take(1); break;
        case NodeKind::Seq:
        case NodeKind::Seq2: {   // Core.h:497-500, Seq2.h:100-103: zeros without a trigger input or a sequence
            if (numCh < 1 || !anySeq(n)) { zeros(); break; }
            op.opcode = n.kind == NodeKind::Seq ? OP_SEQ : OP_SEQ2;
            take(std::min(numCh, 2));
            op.mode = (n.seqHold ? 1u : 0u) | (n.seqLoop ? 2u : 0u) | (numCh > 1 ? 4u : 0u);
            seqSource();
            op.imm = {(uint32_t) std::min<uint64_t>(n.seqOffset, 0xFFFFFFFFu), n.seqGen};
        } break;
        case NodeKind::SparSeq: {   // SparSeq.h:259-262: zeros without a trigger input; the loop-point logic still runs without a sequence
            if (numCh < 1) { zeros(); break; }
            op.opcode = OP_SPARSEQ;
            take(std::min(numCh, 2));
            op.mode = (numCh > 1 ? 4u : 0u);
            seqSource();
            uint64_t tb; std::memcpy(&tb, &n.tickIntervalSamples, 8);
            op.imm = {(uint32_t) n.seqOffset, n.follow ? 1u : 0u, (uint32_t) n.interpolate, n.seqGen, n.loopGen,
                      (uint32_t) n.loopStart, (uint32_t) n.loopEnd, (uint32_t) tb, (uint32_t) (tb >> 32)};
        } break;
        case NodeKind::SparSeq2: {  // SparSeq2.h:90-91
            if (numCh < 1 || !anySeq(n)) { zeros(); break; }
            op.opcode = OP_SPARSEQ2; take(1);
            op.mode = (n.interpolate == 1) ? 1u : 0u;
            seqSource();
            op.imm = {n.seqGen};
        } break;
        case NodeKind::Time: op.opcode = OP_TIME; break;                                     // wasm/SampleTime.h:16-23
        case NodeKind::Metro: op.opcode = OP_METRO; putDouble(op, (double) n.intervalSamps); break;   // wasm/Metro.h:39-55


        // ---- analysis nodes (SURVEY.md §8f N4) ----
        case NodeKind::Meter: if (numCh < 1) { zeros(); break; } op.opcode = OP_METER; take(1); evNode = true; break;
        case NodeKind::Snapshot: if (numCh < 2) { zeros(); break; } op.opcode = OP_SNAPSHOT; take(2); evNode = true; break;
        case NodeKind::Scope:
        case NodeKind::Fft:
        case NodeKind::Capture: {
            evNode = true;
            const size_t floats = (size_t) g.nTiles() * g.tileWidth * (size_t) n.size;
            if (!n.ring) {
                if (!zeroedFloats(n.ring, floats, "analysis ring")) return rc::CudaError;
                n.ringFloats = floats;
                n.ringPositions = n.size;
            }
            if (n.kind == NodeKind::Scope || n.kind == NodeKind::Fft) {
                if (numCh < 1) { zeros(); break; }
                const int ringCh = n.kind == NodeKind::Scope ? (int) SCOPE_CHANNELS : 1;
                op.opcode = OP_SCOPE; take(std::min(numCh, ringCh)); op.aux1 = (uint32_t) ringCh;
                if (prog.dynNodes.size() >= (size_t) MAX_DYN) return E.fail(rc::InvariantViolation, "more than 16 scope nodes in one graph");
                op.aux0 = (uint32_t) prog.dynNodes.size();
                prog.dynNodes.push_back(n.id);
            } else {
                if (numCh < 2) { zeros(); break; }
                op.opcode = OP_CAPTURE; take(2);
                op.aux0 = (uint32_t) (n.size - CAPTURE_SCRATCH);
            }
            op.ptr = (uint64_t) (uintptr_t) n.ring;
        } break;

        case NodeKind::Delay:      // Delays.h:92-106
        case NodeKind::SDelay: {   // Delays.h:221-245
            if (n.ringDirty) {
                E.dsync();
                if (n.ring) { E.dfree(n.ring); n.ring = nullptr; }
                n.ringFloats = (size_t) n.size * ((size_t) g.nTiles() * g.tileWidth);
                n.ringPositions = n.size;
                if (n.ringFloats && !zeroedFloats(n.ring, n.ringFloats, "delay ring")) return rc::CudaError;
                int r = E.fillRowBits(g, n.stateRow, 0, g.nv, freshRowBits(n.kind, 0));   // writeIndex
                if (r != rc::Ok) return r;
                n.ringDirty = false;
            }
            if (n.kind == NodeKind::Delay) {
                if (numCh < 3) { zeros(); break; }
                op.opcode = OP_DELAY; op.aux0 = (uint32_t) n.size; op.ptr = (uint64_t) (uintptr_t) n.ring; take(3);
            } else {
                if (numCh < 1 || n.size == 0) { zeros(); break; }
                op.opcode = OP_SDELAY; op.aux0 = (uint32_t) n.size; op.aux1 = (uint32_t) n.length; op.ptr = (uint64_t) (uintptr_t) n.ring; take(1);
            }
        } break;

        case NodeKind::Table: {   // Table.h:44-57
            if (numCh == 0 || !n.resource || n.resource->numSamples == 0) { zeros(); break; }
            int r = E.ensureResourceOnDevice(*n.resource);
            if (r != rc::Ok) return r;
            op.opcode = OP_TABLE; op.aux0 = (uint32_t) n.resource->numSamples; op.ptr = (uint64_t) (uintptr_t) n.resource->dChannel0; take(1);
            if (!prog.stagedTable && n.resource->numSamples <= (size_t) TABLE_SMEM_MAX_FLOATS) {
                prog.stagedTable = n.resource->dChannel0;
                prog.stagedTableFloats = (int) ((n.resource->numSamples + 3) / 4 * 4);
            }
        } break;

        case NodeKind::Sample: {  // Sample.h:83-134: zeros without a trigger; a voice without a buffer gets zeros on the device
            if (numCh < 1) { zeros(); break; }
            op.opcode = OP_SAMPLE; take(std::min(numCh, 2));
            op.mode = (uint32_t) n.mode | (numCh >= 2 ? 4u : 0u);
            // VariablePitchLerpReader(float sampleRate, ...): 1 - exp(-1 / (0.01 * sampleRate)) in double, stored as float
            op.aux0 = fbits((float) (1.0 - std::exp(-1.0 / (0.01 * (double) (float) E.sr_))));
            for (int k = 0; k < SAMPLE_PARAM_ROWS; ++k) op.operands.push_back({K_PARAM, n.paramRow + k});
        } break;

        case NodeKind::TapIn:
        case NodeKind::TapOut: {
            const size_t floats = (size_t) g.nTiles() * g.tileWidth * E.blockSize_;
            float* shared = nullptr;
            if (!n.tapName.empty()) {   // Feedback.h:29-33: created on first request by either side
                auto it = g.tapShared.find(n.tapName);
                if (it == g.tapShared.end()) {
                    if (!zeroedFloats(shared, floats, "tap")) return rc::CudaError;
                    g.tapShared[n.tapName] = shared;
                } else shared = it->second;
            }
            if (n.kind == NodeKind::TapIn) {
                if (!shared) { zeros(); break; }
                op.opcode = OP_TAPIN; op.ptr = (uint64_t) (uintptr_t) shared;
            } else {
                if (!n.tapPrivate && !zeroedFloats(n.tapPrivate, floats, "tapOut")) return rc::CudaError;
                if (shared) promotes.push_back({rootIndex, n.id});
                if (numCh < 1) { zeros(); break; }
                op.opcode = OP_TAPOUT; op.ptr = (uint64_t) (uintptr_t) n.tapPrivate; take(1);
            }
        } break;

        case NodeKind::Convolve: {   // wasm/Convolve.h:58-85: zeros without an input or a loaded IR
            if (numCh == 0 || !n.resource) { zeros(); break; }
            if (n.resourceDirty || !n.conv) {   // a new `path` makes a fresh convolver (Convolve.h:45-51)
                auto cs = std::make_shared<ConvolverState>();
                const auto& ch0 = n.resource->channels.empty() ? std::vector<float>() : n.resource->channels[0];
                std::string err;
                if (!convolver_init(*cs, E.irBank_, n.resource.get(), n.resource, ch0.data(), ch0.size(), g.nv, E.planOnly_, E.stream_, err)) return E.fail(rc::CudaError, err);
                n.conv = cs;
                n.resourceDirty = false;
            }
            op.opcode = OP_HOST_CONV; take(1);
        } break;

        default: zeros(); break;
    }
    if (evNode) prog.evNodes.push_back({n.id, rootIndex});
    ops.push_back(std::move(op));
    return rc::Ok;
}

int Engine::compile(Group& g, int nIn, std::shared_ptr<Program>& out) {
    auto prog = std::make_shared<Program>();
    prog->planOnly = planOnly_;
    prog->nIn = nIn;
    g.codeDirty = false;
    if (g.tileWidth == 0) g.tileWidth = chooseTileWidth(g.nv);

    // Root order: Runtime.h:544-559 — iterate currentRoots ascending; active roots are pushed to the FRONT,
    // inactive (fading out) ones to the back.
    std::list<int32_t> sortedRoots;
    for (int32_t id : g.currentRoots) {
        auto it = g.nodes.find(id);
        if (it == g.nodes.end() || it->second.kind != NodeKind::Root) continue;
        auto ap = it->second.props.find("active");
        const bool isActive = ap != it->second.props.end() && ap->second.isBool() && ap->second.asBool();
        if (isActive) sortedRoots.push_front(id); else sortedRoots.push_back(id);
    }
    if (sortedRoots.size() > (size_t) MAX_ROOTS) return fail(rc::InvariantViolation, "more than 16 simultaneous roots");

    Compiler C{*this, g, nIn, *prog};
    std::set<int32_t> visited;
    for (int32_t rid : sortedRoots) {
        const int r = (int) prog->rootIds.size();
        prog->rootIds.push_back(rid);
        std::vector<int32_t> order;
        traverse(g, visited, order, rid);
        C.segs.emplace_back();
        for (int32_t nid : order) {
            auto it = g.nodes.find(nid);
            if (it == g.nodes.end()) continue;
            prog->nodeIds.push_back(nid);
            int rcode = C.emitNode(it->second, r);
            if (rcode != rc::Ok) return rcode;
        }
    }
    using PendingOp = Compiler::PendingOp;
    using Segments = Compiler::Segments;
    using Step = PendingOp::Step;
    Segments& segs = C.segs;
    bool hasConv = false;
    for (auto& ops : segs) for (auto& op : ops) if (op.opcode == OP_HOST_CONV) hasConv = true;

    // ---- chain fusion -------------------------------------------------------------------------------------
    // An element-wise node whose output has exactly one use, by a later element-wise node of the same root
    // sub-sequence, is folded into its consumer: as the head of the consumer's chain when it is the first
    // operand, or — for the other operands of a fold — by ending the producer's chain with the reversed step
    // fn(running value, acc).  Every node is still evaluated exactly once, with the same operand values in the
    // same left-fold order (Math.h:71-84), so results are bit-identical; only the evaluation ORDER of
    // independent stateless nodes changes, and the intermediates stay in registers.
    if (opt_.fuseChains) {
        std::unordered_map<int32_t, int> uses;   // over the whole program: a value read once, but by another root's op, stays
        for (auto& ops : segs) for (auto& op : ops) Compiler::forEachSlotUse(op, [&](int32_t id) { ++uses[id]; });
        for (auto& ops : segs) {
            std::unordered_map<int32_t, size_t> producer;   // value id -> index of the (still open) chain producing it in this segment
            std::vector<PendingOp> outOps;
            for (PendingOp& op : ops) {
                if (op.opcode != OP_CHAIN) { outOps.push_back(std::move(op)); continue; }
                auto absorbable = [&](uint32_t kind, int32_t ref) -> long {
                    if (kind != K_SLOT) return -1;
                    auto u = uses.find(ref);
                    if (u == uses.end() || u->second != 1) return -1;
                    auto p = producer.find(ref);
                    if (p == producer.end()) return -1;
                    const auto& pop = outOps[p->second];
                    if (pop.dead || pop.opcode != OP_CHAIN) return -1;
                    return (long) p->second;
                };
                // head: the first operand's producer continues into this chain
                PendingOp cur = op;
                cur.steps.clear();
                {
                    long pi = absorbable(op.operands[0].first, op.operands[0].second);
                    if (pi >= 0) {
                        cur.operands = outOps[pi].operands;
                        cur.steps = outOps[pi].steps;
                        outOps[pi].dead = true;
                    }
                }
                for (const Step& st : op.steps) {
                    long pi = chain_fn_is_unary(st.fn) ? -1 : absorbable(st.kind, st.ref);
                    if (pi < 0 || cur.steps.size() + outOps[pi].steps.size() > 200) { cur.steps.push_back(st); continue; }
                    // flush the running value to a temporary, then restart from the absorbed producer and finish
                    // with the reversed step: value = fn(running, producer)
                    uint32_t runKind = cur.operands[0].first;
                    int32_t runRef = cur.operands[0].second;
                    if (!cur.steps.empty()) {
                        PendingOp flushed = cur;
                        flushed.outNode = C.newTemp();
                        flushed.state = NO_STATE;
                        outOps.push_back(flushed);
                        runKind = K_SLOT; runRef = flushed.outNode;
                    }
                    cur.operands = outOps[pi].operands;
                    cur.steps = outOps[pi].steps;
                    outOps[pi].dead = true;
                    cur.steps.push_back({st.fn | CHAIN_REVERSED, runKind, runRef});
                }
                // keep every op's operand block within 255 words: flush the first 100 steps into a temporary and continue from it
                while (cur.steps.size() > 120) {
                    PendingOp head = cur;
                    head.steps.assign(cur.steps.begin(), cur.steps.begin() + 100);
                    head.outNode = C.newTemp();
                    outOps.push_back(head);
                    cur.operands = {{K_SLOT, head.outNode}};
                    cur.steps.erase(cur.steps.begin(), cur.steps.begin() + 100);
                }
                producer[cur.outNode] = outOps.size();
                outOps.push_back(std::move(cur));
            }
            ops.clear();   // drop absorbed ops
            for (auto& op : outOps) if (!op.dead) ops.push_back(std::move(op));
        }

        // ---- re-schedule each root sub-sequence to shorten live ranges -----------------------------------------
        // Depth-first from the sinks of the segment, visiting the operand with the larger sub-tree first
        // (Sethi-Ullman order).  Any topological order gives the same results — every op is a function of its
        // operand values and its own private state only — but this one keeps a 64-partial additive voice at 3
        // live slots instead of 65.
        for (auto& ops : segs) {
            const size_t n = ops.size();
            std::unordered_map<int32_t, size_t> prodIdx;      // value id -> op index inside this segment
            for (size_t k = 0; k < n; ++k) prodIdx[ops[k].outNode] = k;
            std::vector<std::vector<size_t>> deps(n);
            std::vector<int> consumers(n, 0);
            for (size_t k = 0; k < n; ++k)
                Compiler::forEachSlotUse(ops[k], [&](int32_t id) {
                    auto p = prodIdx.find(id);
                    if (p != prodIdx.end() && p->second != k) { deps[k].push_back(p->second); ++consumers[p->second]; }
                });
            std::vector<long> weight(n, -1);
            std::function<long(size_t)> subtree = [&](size_t k) -> long {
                long& w = weight[k];
                if (w >= 0) return w;
                w = 1;
                for (size_t d : deps[k]) w += subtree(d);
                return w;
            };
            std::vector<char> done(n, 0);
            std::vector<PendingOp> sched;
            std::function<void(size_t)> emit = [&](size_t k) {
                if (done[k]) return;
                done[k] = 1;
                std::vector<size_t> ds = deps[k];
                std::stable_sort(ds.begin(), ds.end(), [&](size_t a, size_t b) { return subtree(a) > subtree(b); });
                for (size_t d : ds) emit(d);
                sched.push_back(std::move(ops[k]));
            };
            for (size_t k = 0; k < n; ++k) if (consumers[k] == 0) emit(k);
            for (size_t k = 0; k < n; ++k) emit(k);   // anything unreachable (cannot happen) keeps its place
            ops.swap(sched);
        }

        // ---- group independent constant-frequency phasors into runs ----------------------------------------------
        // A phasor fed by a parameter depends on nothing, so it may run anywhere in its segment.  With L < 32 voices
        // per warp only L lanes work in a recurrence; a run of R <= 32/L such phasors is executed by R lane groups
        // in one serial loop (render_kernel.cu, OP_PHASOR with aux1 = R).  Followers are pulled forward to sit
        // right behind the leader; the look-ahead is bounded so live ranges stay short.  Programs cut into stages
        // (convolve) insert spill ops between ops: they keep their phasors ungrouped.
        const int maxRun = hasConv ? 1 : std::min(8, 32 / std::max(1, g.tileWidth));
        auto isParamPhasor = [](const PendingOp& op) {
            return op.opcode == OP_PHASOR && op.operands.size() == 1 && op.operands[0].first != K_SLOT;
        };
        for (auto& ops : segs)
            for (size_t i = 0; i < ops.size(); ++i) {
                if (!isParamPhasor(ops[i]) || ops[i].aux1 != 0 || ops[i].mode == 1) continue;
                uint32_t run = 1;
                for (size_t j = i + 1; j < ops.size() && j < i + 1 + (size_t) 4 * maxRun && (int) run < maxRun; ++j) {
                    if (!isParamPhasor(ops[j]) || ops[j].mode == 1) continue;
                    PendingOp follower = ops[j];
                    follower.mode = 1;                     // marks "member of a run" (never dispatched on its own)
                    ops.erase(ops.begin() + (long) j);
                    ops.insert(ops.begin() + (long) (i + run), follower);
                    ++run;
                }
                ops[i].aux1 = run;                         // run length, 1 = a lone constant-frequency phasor
            }
    }

    // ---- stages: a `convolve` node is a whole-block operation (K3) that cannot live inside the sample-tiled
    // interpreter, so the program is cut into K1 stages around it.  Values that cross a stage boundary travel
    // through per-voice block buffers in HBM (OP_STOREBUF / OP_LOADBUF); root ops always run in the last stage.
    std::vector<Segments> stageOps;   // per K1 stage, one op list per root
    if (!hasConv) {
        stageOps.push_back(std::move(segs));
    } else {
        std::unordered_map<int32_t, int> stageOfValue;       // stage in which the value becomes available to K1
        std::vector<std::vector<int>> stageOfOp(segs.size());
        int lastStage = 0;
        for (size_t s = 0; s < segs.size(); ++s)
            for (auto& op : segs[s]) {
                int st = 0;
                Compiler::forEachSlotUse(op, [&](int32_t id) { auto it = stageOfValue.find(id); if (it != stageOfValue.end()) st = std::max(st, it->second); });
                stageOfOp[s].push_back(st);
                stageOfValue[op.outNode] = (op.opcode == OP_HOST_CONV) ? st + 1 : st;
                lastStage = std::max(lastStage, stageOfValue[op.outNode]);
            }
        for (size_t s = 0; s < segs.size(); ++s)
            for (size_t i = 0; i < segs[s].size(); ++i) if (segs[s][i].opcode == OP_ROOT) stageOfOp[s][i] = lastStage;
        const int nStages = lastStage + 1;
        const size_t blockFloats = (size_t) g.Vpad * blockSize_;
        auto newBlockBuffer = [&]() -> float* {
            float* p = nullptr;
            const bool ok = C.zeroedFloats(p, blockFloats, "stage buffer");
            if (p) prog->blockBuffers.push_back(p);   // freed with the program
            return ok ? p : nullptr;
        };
        // buffers: one per convolve node (in, out) and one per ordinary value that crosses stages
        std::unordered_map<int32_t, float*> spillOf;         // value id -> HBM block buffer holding it
        std::unordered_set<int32_t> bypassed;                // host input values convolvers read where they lie
        prog->stages.resize(nStages);
        for (size_t s = 0; s < segs.size(); ++s)
            for (size_t i = 0; i < segs[s].size(); ++i) {
                auto& op = segs[s][i];
                if (op.opcode != OP_HOST_CONV) continue;
                Node& n = g.nodes.at(op.outNode);
                // A convolver fed straight by a host input channel (`convolve(in)`) reads that channel where it lies: no K1 staging
                // copy, and — when nothing else lives in the stage — no K1 launch at all for it.
                int inChannel = -1;
                if (op.operands.size() == 1 && op.operands[0].first == K_SLOT)
                    for (auto& ops : segs)
                        for (auto& ld : ops) if (ld.outNode == op.operands[0].second && ld.opcode == OP_LOADIN) inChannel = (int) ld.aux0;
                float* inB = inChannel >= 0 ? nullptr : newBlockBuffer();
                float* outB = newBlockBuffer();
                if ((inChannel < 0 && !inB) || !outB) return rc::CudaError;
                prog->stages[stageOfOp[s][i]].convolves.push_back({n.id, inB, outB, inChannel});
                spillOf[op.outNode] = outB;
                op.ptr = (uint64_t) (uintptr_t) inB;
                if (inChannel >= 0) { op.mode = 1; bypassed.insert(op.operands[0].second); }   // mode 1: no STOREBUF needed
            }
        // LOADINs whose only consumers are bypassed convolvers are dead
        std::unordered_set<int32_t> otherUses;
        for (auto& ops : segs)
            for (auto& op : ops) if (!(op.opcode == OP_HOST_CONV && op.mode == 1)) Compiler::forEachSlotUse(op, [&](int32_t id) { otherUses.insert(id); });
        for (auto& ops : segs)
            for (auto& op : ops) if (op.opcode == OP_LOADIN && bypassed.count(op.outNode) && !otherUses.count(op.outNode)) op.dead = true;
        // convolver outputs already have their buffer
        for (int32_t id : Compiler::crossingValues(segs, [&](size_t s, size_t i) { return stageOfOp[s][i]; }))
            if (!spillOf.count(id) && !(spillOf[id] = newBlockBuffer())) return rc::CudaError;

        stageOps.assign(nStages, Segments(segs.size()));
        for (int st = 0; st < nStages; ++st) {
            bool anyWork = false;
            std::unordered_set<int32_t> producedHere;
            for (size_t s = 0; s < segs.size(); ++s) {
                auto& out = stageOps[st][s];
                std::unordered_map<int32_t, int32_t> loaded;   // value id -> temp id loaded in this stage+segment
                for (size_t i = 0; i < segs[s].size(); ++i) {
                    if (stageOfOp[s][i] != st || segs[s][i].dead) continue;
                    PendingOp op = segs[s][i];
                    // reload operands that were produced in an earlier stage (or by a convolver)
                    auto fix = [&](uint32_t& kind, int32_t& ref) {
                        if (kind != K_SLOT || producedHere.count(ref)) return;
                        auto sp = spillOf.find(ref);
                        if (sp == spillOf.end()) return;
                        auto l = loaded.find(ref);
                        if (l == loaded.end()) {
                            PendingOp ld;
                            ld.opcode = OP_LOADBUF; ld.outNode = C.newTemp();
                            ld.ptr = (uint64_t) (uintptr_t) sp->second;
                            out.push_back(ld);
                            l = loaded.emplace(ref, ld.outNode).first;
                        }
                        ref = l->second;
                    };
                    for (auto& o : op.operands) fix(o.first, o.second);
                    for (auto& stp : op.steps) if (!chain_fn_is_unary(stp.fn)) fix(stp.kind, stp.ref);
                    if (op.opcode == OP_HOST_CONV && op.mode == 1) continue;   // reads the host input channel directly
                    if (op.opcode == OP_HOST_CONV) {          // stage the convolver input
                        op.opcode = OP_STOREBUF; op.state = NO_STATE; op.outNode = C.newTemp();
                        out.push_back(op);
                        continue;
                    }
                    out.push_back(op);
                    producedHere.insert(op.outNode);
                    auto sp = spillOf.find(op.outNode);
                    if (sp != spillOf.end()) {                // the value is needed by a later stage
                        PendingOp stb;
                        stb.opcode = OP_STOREBUF; stb.outNode = C.newTemp();
                        stb.operands = {{K_SLOT, op.outNode}};
                        stb.ptr = (uint64_t) (uintptr_t) sp->second;
                        out.push_back(stb);
                    }
                }
                anyWork = anyWork || !out.empty();
            }
            prog->stages[st].empty = !anyWork;
        }
        // `convolve -> root` (a reverb send, BASELINE config 4): the last stage is [LOADBUF conv.out][ROOT of it] and nothing else
        if (opt_.fuseConvRoot && g.tileWidth == 1 && nStages >= 2 && prog->rootIds.size() == 1 && C.promotes.empty()) {
            const auto& body = stageOps[nStages - 1][0];
            if (body.size() == 2 && body[0].opcode == OP_LOADBUF && body[1].opcode == OP_ROOT && body[1].operands.size() == 1 &&
                body[1].operands[0].first == K_SLOT && body[1].operands[0].second == body[0].outNode) {
                for (int st = 0; st < nStages - 1 && prog->fusedConvStage < 0; ++st)
                    for (size_t ci = 0; ci < prog->stages[st].convolves.size(); ++ci)
                        if ((uint64_t) (uintptr_t) prog->stages[st].convolves[ci].out == body[0].ptr) {
                            prog->fusedConvStage = st; prog->fusedConvIndex = (int) ci; prog->fusedRoot = (int) body[1].aux0;
                            break;
                        }
            }
        }
    }

    // ---- warp pipeline for one-voice groups (BASELINE config 5: thousands of different graphs, one voice each) ----------------
    // With one voice per warp every recurrence owns a single lane and the warp is latency bound.  The op list (one root sub-sequence,
    // already in its final order) is cut into W contiguous stages of about equal cost; render_groups_pipe_kernel gives each stage its
    // own warp, and the warps work on consecutive sample tiles of the same graph at the same time.  A value that crosses a cut lives in
    // a ring slot with W buffers (tile index mod W), everything else in slots private to its stage.  Same ops, same order of evaluation
    // per value: bit-identical output (tests/test_parity_gpu.py::test_pipelined_groups_equal_the_unpipelined_path).
    std::vector<int> pipeStageOf;            // per op of the one segment of stageOps[0]; empty = not pipelined
    {
        const bool batchedGroup = groups_.size() > 1 && opt_.batchGroups;
        int W = std::min(opt_.pipelineStages, (int) MAX_PIPE);
        bool ok = W > 1 && batchedGroup && g.tileWidth == 1 && stageOps.size() == 1 && prog->rootIds.size() == 1 && C.promotes.empty() &&
                  prog->evNodes.empty() && prog->dynNodes.empty() && !prog->hasCustom;
        // cycles of one 32-sample tile at L = 1, dispatch included: measured per opcode with the cycle-counter build (-DEB_OPPROF);
        // -1: an op the pipeline does not take
        auto costOf = [](const PendingOp& op) -> long {
            switch (op.opcode) {
                case OP_CHAIN: {
                    long c = 350;
                    for (auto& st : op.steps) {
                        const uint32_t fn = st.fn & 0xFF;
                        if (fn <= F_EXP && fn != F_CEIL && fn != F_FLOOR && fn != F_ROUND && fn != F_SQRT && fn != F_ABS) c += 450;
                        else if (fn == F_DIV || fn == F_MOD || fn == F_POW) c += 150;
                        else c += 60;
                    }
                    return c;
                }
                case OP_PHASOR: return op.mode == 1 ? 0 : 1850;          // a run costs what its leader costs
                case OP_SPHASOR: return 2200;
                case OP_COUNTER: case OP_ACCUM: case OP_LATCH: case OP_MAXHOLD: return 1500;
                case OP_RAND: return 450;
                case OP_POLE: return 1850;
                case OP_ENV: return 2000;
                case OP_BIQUAD: return 2600;
                case OP_PREWARP: return 1350;
                case OP_MM1P: return 6800;
                case OP_SVF: return 3450;
                case OP_SVFSHELF: return 4500;
                case OP_BLEP: return 2500;
                case OP_DELAY: return 3300;
                case OP_SDELAY: case OP_TABLE: return 800;
                case OP_Z: return 700;
                case OP_ROOT: return 1100;
                case OP_FILL0: case OP_COPY: return 300;
                default: return -1;
            }
        };
        if (ok)
            for (auto& op : stageOps[0][0]) ok = ok && costOf(op) >= 0;
        if (ok) {
            const auto& sops = stageOps[0][0];
            // units: an op, or a phasor run (leader + its followers), which must stay together
            std::vector<std::pair<size_t, size_t>> units;     // [first op, one past the last op)
            std::vector<long> ucost;
            for (size_t i = 0; i < sops.size();) {
                size_t j = i + 1;
                if (sops[i].opcode == OP_PHASOR && sops[i].aux1 > 1) j = i + sops[i].aux1;
                long c = 0;
                for (size_t k = i; k < j && k < sops.size(); ++k) c += costOf(sops[k]);
                units.push_back({i, std::min(j, sops.size())});
                ucost.push_back(c);
                i = j;
            }
            const int n = (int) units.size();
            if (n >= 2 * W) {
                // linear partition: minimise the most expensive stage (O(n^2 W), n <= a few hundred)
                std::vector<long> pre(n + 1, 0);
                for (int i = 0; i < n; ++i) pre[i + 1] = pre[i] + ucost[i];
                const long INF = (long) 1 << 60;
                std::vector<std::vector<long>> best(W + 1, std::vector<long>(n + 1, INF));
                std::vector<std::vector<int>> cut(W + 1, std::vector<int>(n + 1, 0));
                best[0][0] = 0;
                for (int w = 1; w <= W; ++w)
                    for (int i = w; i <= n; ++i)
                        for (int j = w - 1; j < i; ++j) {
                            if (best[w - 1][j] >= INF) continue;
                            const long c = std::max(best[w - 1][j], pre[i] - pre[j]);
                            if (c < best[w][i]) { best[w][i] = c; cut[w][i] = j; }
                        }
                std::vector<int> bounds(W + 1, 0);
                bounds[W] = n;
                for (int w = W; w >= 1; --w) bounds[w - 1] = cut[w][bounds[w]];
                pipeStageOf.assign(sops.size(), 0);
                for (int w = 0; w < W; ++w)
                    for (int u = bounds[w]; u < bounds[w + 1]; ++u)
                        for (size_t k = units[u].first; k < units[u].second; ++k) pipeStageOf[k] = w;
                for (size_t i = 0; i < sops.size(); ++i)          // roots write the graph's output accumulator: last stage only
                    if (sops[i].opcode == OP_ROOT && pipeStageOf[i] != W - 1) { pipeStageOf.clear(); break; }
                if (!pipeStageOf.empty()) { prog->pipeW = W; prog->pipeDepth = W; }
            }
        }
    }

    // ---- per stage: slot allocation by liveness, then encoding ----
    std::unordered_map<uint32_t, uint32_t> smemIndexOfRow;
    int nStateRows = 0;
    auto mapState = [&](Node& n) -> uint32_t {
        if (n.stateRow < 0) return NO_STATE;
        auto it = smemIndexOfRow.find((uint32_t) n.stateRow);
        if (it != smemIndexOfRow.end()) return it->second;
        const TypeInfo ti = n.kind == NodeKind::Custom ? TypeInfo{NodeKind::Custom, n.fn, customTypes_[n.fn].nState, 0} : typeTable().at(n.typeName);
        if (ti.doubleRows > 0 && (nStateRows & 1)) {   // keep doubles 8-byte aligned in shared memory
            prog->stateMap.push_back(STATE_PAD);
            nStateRows += 1;
        }
        const uint32_t idx = (uint32_t) nStateRows;
        for (int k = 0; k < ti.doubleRows; k += 2) prog->stateMap.push_back(((uint32_t) n.stateRow + k) | STATE_DOUBLE_FLAG);
        for (int k = ti.doubleRows; k < ti.stateRows; ++k) prog->stateMap.push_back((uint32_t) n.stateRow + k);
        nStateRows += ti.stateRows;
        smemIndexOfRow[(uint32_t) n.stateRow] = idx;
        return idx;
    };
    std::unordered_map<int32_t, uint32_t> smemParamOfRow;
    auto emitEnd = [&]() { for (int k = 0; k < 8; ++k) prog->code.push_back(k == 0 ? make_w0(OP_END, 0, 0, 0) : 0u); };
    int nSlotsMax = 1;
    prog->nOps = 0;
    if (prog->stages.empty()) prog->stages.resize(1);
    for (size_t stg = 0; stg < stageOps.size(); ++stg) {
        prog->stages[stg].codeOffset = (uint32_t) prog->code.size();

        // the sections K1 walks: the stage, or one per pipeline stage, each [SEG header][ops] per root
        std::vector<Segments> sections;
        int nSlots = 0;
        if (stg == 0 && !pipeStageOf.empty()) {
            const auto& sops = stageOps[0][0];
            std::unordered_map<int32_t, int> ringOf;   // ring values: read in a later pipeline stage than the one that produces them
            for (int32_t id : Compiler::crossingValues(stageOps[0], [&](size_t, size_t i) { return pipeStageOf[i]; }))
                ringOf.emplace(id, (int) ringOf.size());
            sections.assign(prog->pipeW, Segments(1));
            for (size_t i = 0; i < sops.size(); ++i) sections[pipeStageOf[i]][0].push_back(sops[i]);
            int privBase = 0;   // private slots: liveness inside each stage, every stage in its own index range, rings behind them
            for (auto& sec : sections) privBase += Compiler::allocateSlots(sec, ringOf, privBase);
            const int ringBase = std::max(privBase, 1);
            nSlots = ringBase + (int) ringOf.size() * prog->pipeDepth;
            if (nSlots >= MAX_SLOTS) {                                       // does not fit the 8-bit slot field: keep the program in one piece
                sections.clear(); prog->pipeW = 1; prog->pipeDepth = 1;
            } else {
                for (auto& sec : sections)
                    for (auto& op : sec[0]) {
                        auto rg = ringOf.find(op.outNode);
                        if (rg != ringOf.end()) op.slot = ringBase + rg->second * prog->pipeDepth;
                    }
                prog->pipeRingBase = ringBase;
            }
        }
        if (sections.empty()) {
            sections.push_back(std::move(stageOps[stg]));
            nSlots = Compiler::allocateSlots(sections[0], {}, 0);
            if (nSlots > MAX_SLOTS) return fail(rc::InvariantViolation, "graph needs more than 255 live intermediates");
        }
        nSlotsMax = std::max(nSlotsMax, nSlots);

        std::unordered_map<int32_t, int> producerSlot;   // every value is produced exactly once per stage
        for (auto& sec : sections)
            for (auto& ops : sec)
                for (auto& op : ops) producerSlot[op.outNode] = op.slot;
        auto encodeOperand = [&](uint32_t kind, int32_t ref) -> uint32_t {
            if (kind == K_SLOT) {
                auto ps = producerSlot.find(ref);
                if (ps == producerSlot.end()) return make_operand(K_PARAM, 0);   // never produced: reads as zero
                return make_operand(K_SLOT, (uint32_t) ps->second);
            }
            if (kind == K_PARAM) {
                auto it = smemParamOfRow.find(ref);
                if (it == smemParamOfRow.end()) {
                    prog->paramMap.push_back((uint32_t) ref);
                    it = smemParamOfRow.emplace(ref, (uint32_t) prog->paramMap.size()).first;   // 1-based
                }
                return make_operand(K_PARAM, it->second);
            }
            return make_operand(K_PARAM, 0);
        };
        auto operandWords = [](const PendingOp& op) -> size_t {
            size_t n = op.operands.size() + 2 * op.steps.size() + op.imm.size();
            return (n + 3) & ~(size_t) 3;
        };
        auto emitOp = [&](const PendingOp& op) -> int {
            ++prog->nOps;
            uint32_t st = NO_STATE;
            if (op.state != NO_STATE) {
                auto it = g.nodes.find(op.outNode);
                if (it != g.nodes.end()) st = mapState(it->second);
            }
            const size_t nOperandWords = operandWords(op);
            if (nOperandWords > 255) return fail(rc::InvariantViolation, "operand block of one op exceeds 255 words");
            prog->code.push_back(make_w0(op.opcode, (uint32_t) nOperandWords, (uint32_t) op.slot, op.mode));
            prog->code.push_back(st);
            prog->code.push_back(op.aux0);
            prog->code.push_back(op.opcode == OP_DELAY ? (uint32_t) ++prog->nDelayBuf : op.aux1);   // OP_DELAY: 1 + its read-window buffer
            prog->code.push_back((uint32_t) op.ptr);
            prog->code.push_back((uint32_t) (op.ptr >> 32));
            prog->code.push_back((uint32_t) (op.opcode == OP_CHAIN ? op.steps.size() : op.operands.size()));
            prog->code.push_back(0);
            size_t written = 0;
            for (auto& o : op.operands) { prog->code.push_back(encodeOperand(o.first, o.second)); ++written; }
            for (auto& stp : op.steps) {
                prog->code.push_back(stp.fn);
                prog->code.push_back(chain_fn_is_unary(stp.fn) ? 0u : encodeOperand(stp.kind, stp.ref));
                written += 2;
            }
            for (uint32_t w : op.imm) { prog->code.push_back(w); ++written; }
            for (; written < nOperandWords; ++written) prog->code.push_back(0);
            return rc::Ok;
        };
        const bool piped = sections.size() > 1;
        for (size_t w = 0; w < sections.size(); ++w) {
            if (piped) {   // one code section per pipeline stage, closed by its own END; state rows in stage order
                prog->pipeCode[w] = (uint32_t) prog->code.size() - prog->stages[stg].codeOffset;
                prog->pipeState[w] = (unsigned short) prog->stateMap.size();
                prog->pipeSrow[w] = (unsigned short) nStateRows;
            }
            for (size_t r = 0; r < sections[w].size(); ++r) {   // per root: [SEG header: root index, words to skip][its ops]
                size_t words = 0;
                for (auto& op : sections[w][r]) words += OP_HEADER_WORDS + operandWords(op);
                prog->code.insert(prog->code.end(), {make_w0(OP_SEG, 0, 0, 0), NO_STATE, (uint32_t) r, (uint32_t) words, 0u, 0u, 0u, 0u});
                for (auto& op : sections[w][r]) {
                    const int rcode = emitOp(op);
                    if (rcode != rc::Ok) return rcode;
                }
            }
            if (piped) emitEnd();
        }
        if (piped) for (int w = prog->pipeW; w <= MAX_PIPE; ++w) prog->pipeState[w] = (unsigned short) prog->stateMap.size();
        emitEnd();
        if (stg + 1 == stageOps.size()) {   // tap promotion records live behind the last stage only
            for (auto& pr : C.promotes) {
                Node& n = g.nodes.at(pr.second);
                float* dst = g.tapShared[n.tapName];
                const uint64_t sb = (uint64_t) (uintptr_t) n.tapPrivate, db = (uint64_t) (uintptr_t) dst;
                prog->code.push_back(make_w0(OP_PROMOTE, 0, 0, 0));
                prog->code.push_back((uint32_t) pr.first);
                prog->code.push_back((uint32_t) sb); prog->code.push_back((uint32_t) (sb >> 32));
                prog->code.push_back((uint32_t) db); prog->code.push_back((uint32_t) (db >> 32));
                prog->code.push_back(0); prog->code.push_back(0);
            }
        }
        emitEnd();
    }
    prog->nStateRows = (nStateRows + 1) & ~1;
    prog->nSlots = nSlotsMax;

    // ---- upload: code, stateMap and paramMap in ONE allocation; the copies are stream-ordered in front of the first launch and their
    // sources are members of the Program, so nothing has to be waited for here ----
    {
        const size_t codeW = (prog->code.size() + 3) & ~(size_t) 3, smW = (prog->stateMap.size() + 3) & ~(size_t) 3, pmW = prog->paramMap.size();
        if (!cuda(dmalloc((void**) &prog->dCode, sizeof(uint32_t) * (codeW + smW + pmW + 4)), "cudaMalloc program")) return rc::CudaError;
        if (!cuda(dmemcpy(prog->dCode, prog->code.data(), sizeof(uint32_t) * prog->code.size(), cudaMemcpyHostToDevice), "upload code")) return rc::CudaError;
        if (!prog->stateMap.empty()) {
            prog->dStateMap = prog->dCode + codeW;
            if (!cuda(dmemcpy(prog->dStateMap, prog->stateMap.data(), sizeof(uint32_t) * prog->stateMap.size(), cudaMemcpyHostToDevice), "upload stateMap")) return rc::CudaError;
        }
        if (!prog->paramMap.empty()) {
            prog->dParamMap = prog->dCode + codeW + smW;
            if (!cuda(dmemcpy(prog->dParamMap, prog->paramMap.data(), sizeof(uint32_t) * prog->paramMap.size(), cudaMemcpyHostToDevice), "upload paramMap")) return rc::CudaError;
        }
    }
    // Per-program specialisation of K1 (spec_host.h).  Not for groups that render through the batched many-groups launch (that
    // kernel is the interpreter by construction: one launch serves different programs), not for multi-stage programs.
    const bool batched = groups_.size() > 1 && opt_.batchGroups && !prog->hasCustom;
    if (prog->hasCustom) {
        // Registered device node types exist only inside a kernel compiled for the program: specialisation is mandatory and
        // synchronous, whatever the "specialize" option says, and a body that does not compile fails the COMMIT.
        if (prog->stages.size() > 1) return fail(rc::InvariantViolation, "a registered node type cannot share a graph with convolve");
        prog->specJob = specialise_request(prog->code, g.tileWidth, opt_.niter, device_, customSource());
        specialise_wait(*prog->specJob);
        if (prog->specJob->state.load(std::memory_order_acquire) < 0)
            return fail(rc::InvariantViolation, "registered node type failed to compile: " + prog->specJob->log);
    } else if (opt_.specialize && !batched && prog->stages.size() <= 1 && (int) prog->code.size() <= opt_.specializeMaxWords) {
        prog->specJob = specialise_request(prog->code, g.tileWidth, opt_.niter, device_, std::string(), midRangeDense(g.nv) ? 8 : opt_.specMinBlocks,
                                            opt_.specOpprof);   // NVRTC on the compile-queue thread
        if (opt_.specialize >= 2) {                                                          // synchronous mode: wait for the compiler here
            specialise_wait(*prog->specJob);
            if (prog->specJob->state.load(std::memory_order_acquire) < 0 && opt_.specializeStrict)
                return fail(rc::InvariantViolation, "K1 specialisation failed: " + prog->specJob->log);
        }
    }
    out = prog;
    return rc::Ok;
}

// ---------------------------------------------------------------------------------------------------------
// process
float* Engine::voiceInDevicePtr(size_t nIn) {
    Lock lk(mu_);
    return grow(dInVoice_, inVoiceFloats_, (size_t) numVoices_ * nIn * blockSize_, "cudaMalloc voice in", true) ? dInVoice_ : nullptr;
}

float* Engine::sharedInDevicePtr(size_t nIn) {
    Lock lk(mu_);
    return grow(dInShared_, inSharedFloats_, nIn * blockSize_, "cudaMalloc shared in", true) ? dInShared_ : nullptr;
}

int Engine::enqueueBlock(size_t nIn, size_t nOut, size_t numSamples, bool perVoiceIn, bool materialise, bool mix, bool allReduce) {
    Lock lk(mu_);
    // A plan-only engine cannot render.  With option "plan_dry_run" it still walks the whole host side of a block — program swap,
    // recompiles, descriptors, fades, event mirrors — and skips exactly the CUDA calls: the thread-safety tests (TSAN, no GPU) use it.
    if (planOnly_ && !planDryRun_) return fail(rc::CudaError, "plan-only runtime (no CUDA device): rendering is impossible, there is no CPU fallback");
    dsetdev();
    if (numSamples > (size_t) blockSize_ || nOut > (size_t) MAX_WIDE_OUT_CHANNELS) return fail(rc::BadArgument, "numSamples > blockSize or too many output channels");
    if (nOut > (size_t) MAX_OUT_CHANNELS && mix && allReduce && peerAttached_ && peer_.world > 1)
        return fail(rc::BadArgument, "the cross-GPU mix bus carries at most 8 output channels (its exchange buffer is sized at export)");
    BlockIO io;
    io.nIn = nIn; io.nOut = nOut; io.numSamples = numSamples; io.perVoiceIn = perVoiceIn; io.allReduce = allReduce;
    io.inPitch = io.outPitch = io.mixPitch = blockSize_;
    // input rows the caller never wrote read as zero
    if (nIn && !(io.in = perVoiceIn ? voiceInDevicePtr(nIn) : sharedInDevicePtr(nIn))) return rc::CudaError;
    if (materialise) {
        const size_t of = (size_t) numVoices_ * nOut * blockSize_;
        // K1 writes [voice][nOut] in the dense layout, and new memory is not cleared: the wide path clears the buffer again
        if (nOut <= (size_t) MAX_OUT_CHANNELS || of > outVoiceFloats_) wide_.outZeroValid = false;
        if (!grow(dOutVoice_, outVoiceFloats_, of, "cudaMalloc voice out")) return rc::CudaError;
        io.voiceOut = dOutVoice_;
    }
    // the mix bus and its mapped host copy grow to the widest nOut used (elem_b200_mix_device: the pointer moves then)
    if (nOut * blockSize_ > mixFloats_) {
        if (!grow(dMix_, mixFloats_, nOut * blockSize_, "cudaMalloc mix", true)) return rc::CudaError;
        if (hMixHost_) allocMixHost();
    }
    if (mix) io.mix = dMix_;
    return enqueueBlock(io);
}

// One block (the engine lock is held): the walk over the voice groups unless the steady-state key matches, then the launches every
// block ends with — the many-groups buckets, the mix bus (K2, K2w or silence) and the cross-GPU sum (K4).
int Engine::enqueueBlock(const BlockIO& io) {
    const bool dry = planOnly_;
    const size_t nOut = io.nOut, numSamples = io.numSamples;
    // Past MAX_OUT_CHANNELS the mix bus is compact (DESIGN.md section 3): per channel, only the partial rows of the groups that aim at it
    const bool wide = nOut > (size_t) MAX_OUT_CHANNELS;
    // the scatter to [voice][nOut] writes the engine's own buffer at pitch blockSize
    if (wide && io.voiceOut && io.voiceOut != dOutVoice_) return fail(rc::BadArgument, "renderOffline: at most 8 output channels");
    if (!steadyValid_ || !io.sameSteadyKey(steadyIO_)) {
        const int r = walkGroups(io);
        if (r != rc::Ok) return r;
    }
    for (auto& sb : steadyBuckets_) {
        BatchBuffers& bb = batch_[sb.key];
        auto ev = timedBegin();
        if (!dry && !cuda(sb.pipeStages >= 1
                              ? launch_render_groups_pipe(bb.dDescs, bb.dTileStart, sb.nGroups, sb.totalTiles, sb.pipeStages, sb.maxSlots, sb.smemOut, sb.maxState, sb.maxParams, sampleTime_, io.col, io.col, stream_, opt_.niter)
                              : launch_render_groups(bb.dDescs, bb.dTileStart, sb.nGroups, sb.totalTiles, sb.L, sb.maxSlots, sb.smemOut, sb.maxState, sb.maxParams, sb.wpc, sampleTime_, io.col, io.col, stream_, opt_.niter),
                  "render groups kernel launch")) return rc::CudaError;
        timedEnd(ev, 0);
        ++launches_;
    }
    // With the cross-GPU sum behind it, K2 leaves this rank's partial mix in PeerMix::own (K4 pushes it to the peers from there and
    // writes the total to the mix bus): no staging copy, no in-place hazard between K4's CTAs.
    const bool exchange = io.mix && io.allReduce && peerAttached_ && peer_.world > 1;
    if (exchange) ++peerEpoch_;
    if (wide) {
        const int rw = dry ? rc::Ok : launchWide(io);
        if (rw != rc::Ok) return rw;
    } else if (io.mix) {
        float* const mixOut = exchange ? peer_.own : io.mix + io.col;
        const int pitch = exchange ? blockSize_ : io.mixPitch;
        if (steadyTiles_ > 0) {
            auto ev = timedBegin();
            if (!dry && !cuda(launch_mix_reduce(dPartial_, mixOut, pitch, dMixScratch_, dMixTickets_, steadyTiles_, (int) nOut, blockSize_, (int) numSamples, stream_, exchange ? HostDeliver{} : takeDeliver()), "mix reduce launch")) return rc::CudaError;
            timedEnd(ev, 1);
            ++launches_;
        } else if (!cuda(dzeroBlock(mixOut, pitch, nOut), "memset mix")) return rc::CudaError;   // an offline chunk's slots are reused: every block writes its column
    }
    if (exchange) {   // K4: the cross-GPU sum of the mix bus, in the same stream
        auto ev = timedBegin();
        if (!cuda(launch_mix_exchange(peer_, dMix_, (int) (nOut * blockSize_), peerEpoch_, dPeerStatus_, stream_, takeDeliver()), "mix exchange launch")) return rc::CudaError;
        timedEnd(ev, 3);
        ++launches_;
    }
    sampleTime_ += (int64_t) numSamples;   // wasm/Main.cpp:217
    return rc::Ok;
}

// The slow walk of a block: program swaps and recompiles, the wide plan, buffers, the launches of voice groups that run on their own (K1 /
// K3), fades and event mirrors, and the many-groups buckets (steadyBuckets_) with their descriptors uploaded when they changed.
int Engine::walkGroups(const BlockIO& io) {
    const bool dry = planOnly_;
    const size_t nIn = io.nIn, nOut = io.nOut, numSamples = io.numSamples;
    const bool perVoiceIn = io.perVoiceIn, materialise = io.voiceOut != nullptr, mix = io.mix != nullptr;
    const bool wide = nOut > (size_t) MAX_OUT_CHANNELS;
    steadyValid_ = false;
    bool allSteady = !(io.allReduce && peerAttached_ && peer_.world > 1), allBatched = true;

    // Runtime::process: swap in the newest render sequence (Runtime.h:277-285); recompile when the number of
    // host input channels a leaf node sees has changed.
    for (auto& gp : groups_) {
        Group& g = *gp;
        if (g.pending) { g.active = g.pending; g.pending.reset(); g.superseded.clear(); }
        if (g.active && g.codeDirty) {
            // A property that is baked into the program (svf.mode, delay.size, seq data, ...) was set after the last
            // COMMIT: the reference's nodes pick such changes up at the top of their next process() through atomics
            // and SPSC queues (e.g. Delays.h:92-95, Core.h:470-495); here the sequence is recompiled.
            std::shared_ptr<Program> p;
            int r = compile(g, (int) nIn, p);
            if (r != rc::Ok) return r;
            g.active = p;
        }
        if (g.active && g.active->nIn != (int) nIn) {
            if (g.active->usesHostInputs) {   // leaf nodes see the host channels: GraphRenderSequence.h:126-135
                std::shared_ptr<Program> p;
                int r = compile(g, (int) nIn, p);
                if (r != rc::Ok) return r;
                g.active = p;
            } else g.active->nIn = (int) nIn;
        }
    }
    // Wide path: each group's mix channels, the run of compact partial rows it owns ([tile][mix channel]) and its run of compact
    // per-voice output rows ([voice][mix channel]), in engine order
    std::vector<std::vector<int>> wideCh;
    std::vector<size_t> wideRowBase, wideOutBase;
    size_t wideRows = 0, wideOutRows = 0;
    if (wide) {
        wideCh.resize(groups_.size()); wideRowBase.assign(groups_.size(), 0); wideOutBase.assign(groups_.size(), 0);
        for (size_t gi = 0; gi < groups_.size(); ++gi) {
            const Group& g = *groups_[gi];
            if (g.active && g.nTiles()) wideCh[gi] = mixChannels(g, *g.active, nOut);
            wideRowBase[gi] = wideRows; wideOutBase[gi] = wideOutRows;
            wideRows += (size_t) g.nTiles() * wideCh[gi].size();
            wideOutRows += (size_t) g.nv * wideCh[gi].size();
        }
        // the row list of channel c (CSR): groups in engine order, tiles in order; then K2's tile groups of each list
        WidePlan& w = wide_;
        std::vector<int> rowPtr(nOut + 1, 0);
        for (size_t gi = 0; gi < groups_.size(); ++gi)
            for (int c : wideCh[gi]) rowPtr[c + 1] += groups_[gi]->nTiles();
        for (size_t c = 0; c < nOut; ++c) rowPtr[c + 1] += rowPtr[c];
        w.rows.assign(rowPtr[nOut], 0);
        std::vector<int> pos(rowPtr.begin(), rowPtr.end() - 1);
        for (size_t gi = 0; gi < groups_.size(); ++gi) {
            const int nC = (int) wideCh[gi].size(), nT = groups_[gi]->nTiles();
            for (int k = 0; k < nC; ++k)
                for (int t = 0; t < nT; ++t) w.rows[pos[wideCh[gi][k]]++] = (int) wideRowBase[gi] + t * nC + k;
        }
        w.segs.clear(); w.nScratch = 0;
        for (size_t c = 0; c < nOut; ++c) {
            const int n = rowPtr[c + 1] - rowPtr[c];
            const int G = n == 0 ? 1 : std::min(MIX_REDUCE_MAX_GROUPS, (n + 255) / 256);
            const int per = ((n + G - 1) / G + 31) / 32 * 32;
            const int sc = G > 1 ? w.nScratch : -1;
            if (G > 1) w.nScratch += G;
            for (int k = 0; k < G; ++k) {
                const int b = std::min(n, k * per), e = std::min(n, k * per + per);
                w.segs.push_back(WideSeg{(int) c, rowPtr[c] + b, e - b, G, k, sc});
            }
        }
        // K2w takes the segments of fewer than WIDE_BIG_ROWS rows first (a warp each), then the larger ones (a CTA each)
        w.nSmall = (int) (std::stable_partition(w.segs.begin(), w.segs.end(), [](const WideSeg& sg) { return sg.rowCount < WIDE_BIG_ROWS; }) - w.segs.begin());
        w.dstRow.clear();
        if (materialise)
            for (size_t gi = 0; gi < groups_.size(); ++gi) {
                const Group& g = *groups_[gi];
                for (int v = 0; v < (wideCh[gi].empty() ? 0 : g.nv); ++v)
                    for (int c : wideCh[gi]) w.dstRow.push_back((g.v0 + v) * (int) nOut + c);
            }
    }
    size_t tiles = 0;
    for (auto& g : groups_) tiles += (size_t) g->nTiles();
    if (!grow(dPartial_, partialFloats_, wide ? std::max<size_t>(1, wideRows) * blockSize_ : std::max<size_t>(1, tiles) * nOut * blockSize_, "cudaMalloc partial", true))
        return rc::CudaError;
    if (materialise && wide && !grow(dOutCompact_, outCompactFloats_, std::max<size_t>(1, wideOutRows) * blockSize_, "cudaMalloc compact voice out"))
        return rc::CudaError;
    if (wide && !dry) {
        const int r = uploadWidePlan();
        if (r != rc::Ok) return r;
    }

    int tileBase = 0;
    std::map<int, std::vector<LaunchParams>> buckets;   // tile width -> single-stage groups launched together
    for (auto& gp : groups_) {
        Group& g = *gp;
        const size_t gi = (size_t) (&gp - groups_.data());
        const int nTiles = g.nTiles();
        if (!g.active || nTiles == 0) {
            allSteady = false;
            // no render sequence yet: outputs are silence (Runtime.h:287-289 leaves the host buffers untouched;
            // we define the voice's contribution as zero)
            if (nTiles && mix && !wide) dmemset(dPartial_ + (size_t) tileBase * nOut * blockSize_, 0, sizeof(float) * (size_t) nTiles * nOut * blockSize_);
            if (materialise) dzeroBlock(io.voiceOut + (size_t) g.v0 * nOut * io.outPitch + io.col, io.outPitch, (size_t) g.nv * nOut);
            tileBase += nTiles;
            continue;
        }
        Program& p = *g.active;
        LaunchParams P{};
        P.code = p.dCode;
        P.stateMap = p.dStateMap;
        P.paramMap = p.dParamMap;
        P.nParams = (int) p.paramMap.size();
        P.rows = g.dRows;
        // wide: the group's own runs of compact rows, per-voice I/O indexed from its first voice (voice0 = 0)
        const std::vector<int>* const gch = wide ? &wideCh[gi] : nullptr;
        float* const voiceOut = wide ? (gch->empty() ? nullptr : dOutCompact_ + wideOutBase[gi] * blockSize_) : io.voiceOut;
        float* const partialOut = wide ? (gch->empty() ? nullptr : dPartial_ + wideRowBase[gi] * blockSize_) : dPartial_;
        // input rows without this block's column (the many-groups launches take it as an argument; single-group launches are handed
        // pointers that include it)
        const float* const inShared = (!perVoiceIn && nIn) ? io.in : nullptr;
        const float* const inVoice = (perVoiceIn && nIn) ? io.in + (wide ? (size_t) g.v0 * nIn * io.inPitch : 0) : nullptr;
        P.inShared = inShared;
        P.inVoice = inVoice;
        P.outVoice = materialise ? voiceOut : nullptr;
        P.mixPartial = mix ? partialOut : nullptr;
        P.nStateEntries = (int) p.stateMap.size();
        P.nStateRows = p.nStateRows;
        P.nSlots = p.nSlots;
        P.Vpad = g.Vpad;
        P.nv = g.nv;
        P.voice0 = wide ? 0 : g.v0;
        P.tileWidth = g.tileWidth;
        P.numSamples = (int) numSamples;
        P.blockSize = blockSize_;
        P.nIn = (int) nIn;
        P.nOut = wide ? (int) gch->size() : (int) nOut;
        P.inStride = io.inPitch;
        P.outStride = io.outPitch;
        P.tileBase = wide ? 0 : tileBase;
        uint32_t runMask = 0;
        for (size_t ri = 0; ri < p.rootIds.size(); ++ri) {
            auto it = g.nodes.find(p.rootIds[ri]);
            if (it == g.nodes.end()) continue;
            Node& rn = it->second;
            const bool stillRunning = rn.fade.on() || !rn.fade.settled();                     // Core.h:28-31
            const bool chanOk = rn.channel >= 0 && (size_t) rn.channel < nOut;                // GraphRenderSequence.h:214-219
            if (stillRunning && chanOk) runMask |= (1u << ri);
            if (rn.fade.on()) runMask |= (1u << (16 + ri));                                   // promoteTapBuffers: :200-205
            int chan = rn.channel;
            if (wide) {   // the compact index of the channel among the group's mix channels
                const auto at = std::lower_bound(gch->begin(), gch->end(), chan);
                chan = (chanOk && at != gch->end() && *at == chan) ? (int) (at - gch->begin()) : -1;
            }
            P.roots[ri] = RootDyn{rn.fade.current, rn.fade.step, rn.fade.target, chan};
            if (rn.fade.current != rn.fade.target) allSteady = false;        // the descriptor changes while a root fades
        }
        if (!p.evNodes.empty() || !p.dynNodes.empty() || g.codeDirty || g.pending) allSteady = false;
        P.runMask = runMask;
        P.sampleTime = sampleTime_;
        P.tableSrc = p.stagedTable; P.tableFloats = p.stagedTableFloats; P.tableSmem = -1;   // the launcher places it (single-group launches)
        P.pipeW = p.pipeW; P.pipeRingBase = p.pipeRingBase; P.pipeDepth = p.pipeDepth;
        for (int w = 0; w < MAX_PIPE; ++w) { P.pipeCode[w] = p.pipeCode[w]; P.pipeSrow[w] = p.pipeSrow[w]; }
        for (int w = 0; w <= MAX_PIPE; ++w) P.pipeState[w] = p.pipeState[w];
        for (size_t di = 0; di < p.dynNodes.size(); ++di) {
            auto it = g.nodes.find(p.dynNodes[di]);
            if (it != g.nodes.end()) P.dyn[di] = it->second.scopeW;
        }
        for (auto& ev : p.evNodes) {       // host mirrors of what is identical for every voice of the group
            if (!((runMask >> ev.root) & 1u)) continue;
            auto it = g.nodes.find(ev.node);
            if (it == g.nodes.end()) continue;
            Node& en = it->second;
            if ((en.kind == NodeKind::Scope || en.kind == NodeKind::Fft) && (en.inlets.empty() ? nIn : en.inlets.size()) >= 1) {          // MultiChannelRingBuffer::write, :36-62
                const uint32_t mask = SCOPE_RING - 1, w = en.scopeW, r = en.scopeR, n = (uint32_t) numSamples;
                const uint32_t freeSlots = (r > w) ? (r - w) : ((uint32_t) SCOPE_RING - (w - r));
                en.scopeW = (w + n) & mask;
                if (n >= freeSlots) en.scopeR = (en.scopeW + 1) & mask;
            } else if (en.kind == NodeKind::Metro) {                        // Metro.h:44-55
                const double is = (double) en.intervalSamps;
                for (size_t i = 0; i < numSamples; ++i) {
                    const double t = (double) (sampleTime_ + (int64_t) i) / is;
                    const float nextOut = (float) ((t - std::floor(t)) < 0.5);
                    if (en.metroLastOut < 0.5f && nextOut >= 0.5f) en.metroFlag = true;
                    en.metroLastOut = nextOut;
                }
            }
        }

        // launch geometry: spread warps over the SMs first, then stack them
        int wpc = opt_.warpsPerCta;
        if (wpc <= 0) wpc = nTiles >= smCount_ * 8 ? 4 : (nTiles >= smCount_ * 4 ? 2 : 1);
        const size_t perWarp = render_smem_bytes(p.nSlots, P.nOut, p.nStateRows, (int) p.paramMap.size(), 1, g.tileWidth, opt_.niter) +
                               render_delay_buf_floats(p.nDelayBuf, g.tileWidth, opt_.niter) * sizeof(float);
        while (wpc > 1 && perWarp * wpc > 200 * 1024) wpc >>= 1;
        if (perWarp > 220 * 1024) return fail(rc::InvariantViolation, "graph state does not fit in shared memory");
        const size_t nStages = std::max<size_t>(1, p.stages.size());
        if (nStages == 1 && groups_.size() > 1 && opt_.batchGroups && !p.hasCustom) {
            // heterogeneous voice groups: collect single-stage groups per tile geometry and launch each bucket once
            P.code = p.dCode + (p.stages.empty() ? 0 : p.stages[0].codeOffset);
            // one-voice groups launch through the pipeline kernel (programs that were not cut simply use warp 0 of their CTA): one
            // launch for all of them whether or not every program could be cut
            const int bkey = g.tileWidth + ((p.pipeW > 1 || (g.tileWidth == 1 && opt_.pipelineStages > 1)) ? PIPE_BUCKET : 0);
            buckets[bkey].push_back(P);
            buckets[bkey].back().sampleTime = 0;      // the many-groups kernel takes the clock as an argument: descriptors stay equal block to block
        } else
        for (size_t stg = 0; stg < nStages; ++stg) {
            allBatched = false;
            const bool last = stg + 1 == nStages;
            P.code = p.dCode + (p.stages.empty() ? 0 : p.stages[stg].codeOffset);
            P.outVoice = (last && materialise) ? voiceOut + io.col : nullptr;   // outputs and taps belong to the last stage
            P.inShared = inShared ? inShared + io.col : nullptr;
            P.inVoice = inVoice ? inVoice + io.col : nullptr;
            P.mixPartial = (last && mix) ? partialOut : nullptr;
            auto ev = timedBegin();
            const bool emptyStage = !p.stages.empty() && ((p.stages[stg].empty && !last) || (last && p.fusedConvStage >= 0));   // fused: K3's epilogue did the root
            if (!emptyStage) {
                const SpecKernel* spec = nullptr;
                if (p.specJob) {   // the cubin arrived: load it on this thread (its CUDA context is current), a matter of milliseconds
                    const int st = specialise_ensure_loaded(*p.specJob);
                    if (st == 2) spec = &p.specJob->kernel;
                    else if (st < 0 && (opt_.specializeStrict || p.hasCustom)) return fail(rc::CudaError, "K1 specialisation failed: " + p.specJob->log);
                }
                P.nDelayBuf = p.nDelayBuf;      // (the many-groups launches above reserve no read-window buffers: 0)
                if (!dry && !cuda(launch_render_block(P, wpc, opt_.niter, stream_, spec), "render kernel launch")) return rc::CudaError;
                ++launches_;
            }
            timedEnd(ev, 0);   // recorded around a skipped stage too
            if (p.stages.empty()) continue;
            // K3: the convolvers fed by this stage (ConvolutionNode::process, wasm/Convolve.h:58-85); a call longer
            // than what is left of the current 512-sample partition is cut like FFTConvolver.cpp:155-203 does
            for (size_t cvi = 0; cvi < p.stages[stg].convolves.size(); ++cvi) {
                auto& cv = p.stages[stg].convolves[cvi];
                auto it = g.nodes.find(cv.node);
                if (it == g.nodes.end() || !it->second.conv) continue;
                ConvolverState& cs = *it->second.conv;
                ConvEpilogue epi;
                if (p.fusedConvStage == (int) stg && p.fusedConvIndex == (int) cvi) {
                    const RootDyn& rd = P.roots[p.fusedRoot];
                    epi.active = true;
                    epi.running = ((runMask >> p.fusedRoot) & 1u) != 0;
                    epi.gain0 = rd.gain0; epi.step = rd.step; epi.target = rd.target; epi.channel = rd.channel;
                    epi.nOut = P.nOut; epi.blockSize = blockSize_;
                    epi.mixPartial = mix ? partialOut : nullptr; epi.tileBase = P.tileBase;
                    epi.outVoice = materialise ? voiceOut + io.col : nullptr;
                    epi.voice0 = P.voice0; epi.outStride = P.outStride; epi.outOffset = 0;
                }
                int offset = 0;
                while (offset < (int) numSamples) {
                    const int n = cs.maxS == 0 ? (int) numSamples - offset
                                                     : std::min((int) numSamples - offset, CONV_BLOCK - cs.fill);
                    auto ev3 = timedBegin();
                    const float* cin = cv.in;
                    int cinStride = blockSize_;
                    if (cv.inChannel >= 0) {   // straight from the host input rows: per-voice [voice][nIn][inPitch] or shared [nIn][inPitch]
                        if (perVoiceIn) { cin = io.in + ((size_t) g.v0 * nIn + cv.inChannel) * io.inPitch + io.col; cinStride = (int) nIn * io.inPitch; }
                        else { cin = io.in + (size_t) cv.inChannel * io.inPitch + io.col; cinStride = 0; }
                    }
                    if (!dry && !cuda(convolver_process_chunk(cs, cin, cinStride, cv.out, blockSize_, offset, n, stream_, epi), "convolver launch")) return rc::CudaError;
                    if (dry) { offset += n; continue; }
                    timedEnd(ev3, 2);
                    ++launches_;
                    offset += n;
                }
            }
        }

        for (size_t ri = 0; ri < p.rootIds.size(); ++ri) {
            if (!(runMask & (1u << ri))) continue;
            auto it = g.nodes.find(p.rootIds[ri]);
            if (it != g.nodes.end()) it->second.fade.advance((int) numSamples);
        }
        tileBase += nTiles;
    }
    steadyBuckets_.clear();
    for (auto& kv : buckets) {
        auto& descs = kv.second;
        const int L = kv.first % PIPE_BUCKET;
        std::vector<int> tileStart(descs.size());
        int total = 0, maxSlots = 1, maxState = 0, maxParams = 0, pipeStages = 0, smemOut = 0;
        for (size_t i = 0; i < descs.size(); ++i) {
            tileStart[i] = total;
            smemOut = std::max(smemOut, descs[i].nOut);   // = nOut unless wide
            total += (descs[i].nv + L - 1) / L;
            maxSlots = std::max(maxSlots, descs[i].nSlots);
            maxState = std::max(maxState, descs[i].nStateRows);
            maxParams = std::max(maxParams, descs[i].nParams);
            if (kv.first >= PIPE_BUCKET) pipeStages = std::max(pipeStages, std::max(1, descs[i].pipeW));
        }
        // descriptors change only while roots fade or when graphs change: re-upload only then
        BatchBuffers& bb = batch_[kv.first];
        const size_t dbytes = descs.size() * sizeof(LaunchParams), tbytes = tileStart.size() * sizeof(int);
        if (descs.size() > bb.capDescs) bb.lastDescs.clear();
        if (!grow(bb.dDescs, bb.capDescs, descs.size(), "cudaMalloc group descriptors", false, 2) ||
            !grow(bb.dTileStart, bb.capTiles, descs.size(), "cudaMalloc tile table", false, 2)) return rc::CudaError;
        if (!dry && (bb.lastDescs.size() != dbytes || std::memcmp(bb.lastDescs.data(), descs.data(), dbytes) != 0)) {
            if (!cuda(cudaMemcpyAsync(bb.dDescs, descs.data(), dbytes, cudaMemcpyHostToDevice, stream_), "upload group descriptors")) return rc::CudaError;
            if (!cuda(cudaMemcpyAsync(bb.dTileStart, tileStart.data(), tbytes, cudaMemcpyHostToDevice, stream_), "upload tile table")) return rc::CudaError;
            bb.lastDescs.assign(reinterpret_cast<const char*>(descs.data()), reinterpret_cast<const char*>(descs.data()) + dbytes);
        }
        int wpc = opt_.warpsPerCta;
        if (wpc <= 0) wpc = total >= smCount_ * 8 ? 4 : (total >= smCount_ * 4 ? 2 : 1);
        while (wpc > 1 && render_smem_bytes(maxSlots, smemOut, maxState, maxParams, wpc, L, opt_.niter) > 200 * 1024) wpc >>= 1;
        steadyBuckets_.push_back(SteadyBucket{L, (int) descs.size(), total, maxSlots, maxState, maxParams, wpc, pipeStages, kv.first, smemOut});
    }
    steadyValid_ = allSteady && allBatched && !buckets.empty() && !dry;
    steadyIO_ = io;
    steadyTiles_ = tileBase;
    return rc::Ok;
}

std::vector<int> Engine::mixChannels(const Group& g, const Program& p, size_t nOut) const {
    std::vector<int> ch;
    for (int32_t id : p.rootIds) {
        auto it = g.nodes.find(id);
        if (it == g.nodes.end()) continue;
        const int c = it->second.channel;
        if (c >= 0 && (size_t) c < nOut) ch.push_back(c);
    }
    std::sort(ch.begin(), ch.end());
    ch.erase(std::unique(ch.begin(), ch.end()), ch.end());
    return ch;
}

// Upload what changed of the wide plan (row lists, segments, output rows) and grow K2w's scratch and tickets.
int Engine::uploadWidePlan() {
    WidePlan& w = wide_;
    auto upload = [&](auto& dev, size_t& cap, const auto& host, auto& shadow, const char* what) -> bool {
        typedef typename std::remove_reference<decltype(host)>::type::value_type T;
        const size_t n = std::max<size_t>(1, host.size());
        if (n > cap) shadow.clear();
        if (!grow(dev, cap, n, what, false, 2)) return false;
        const size_t bytes = host.size() * sizeof(T);
        if (shadow.size() == bytes / sizeof(shadow[0]) && std::memcmp(shadow.data(), host.data(), bytes) == 0) return true;
        if (bytes && !cuda(dmemcpy(dev, host.data(), bytes, cudaMemcpyHostToDevice), what)) return false;
        shadow.resize(bytes / sizeof(shadow[0]));
        if (bytes) std::memcpy(shadow.data(), host.data(), bytes);
        return true;
    };
    if (!upload(w.dRows, w.capRows, w.rows, w.upRows, "upload wide row lists")) return rc::CudaError;
    if (!upload(w.dSegs, w.capSegs, w.segs, w.upSegs, "upload wide segments")) return rc::CudaError;
    if (!upload(w.dDst, w.capDst, w.dstRow, w.upDst, "upload wide output rows")) return rc::CudaError;
    if (!grow(dWideScratch_, wideScratchFloats_, (size_t) w.nScratch * blockSize_, "cudaMalloc wide mix scratch", false, 2) ||
        !grow(dWideTickets_, wideTicketCount_, (size_t) w.nScratch * ((blockSize_ + 31) / 32), "cudaMalloc wide mix tickets", true, 2))
        return rc::CudaError;
    return rc::Ok;
}

// The device half of a wide block after K1 / K3: per-voice outputs scattered to [voice][nOut] (every other channel zero), then K2w,
// which also hands the mix bus to the host.
int Engine::launchWide(const BlockIO& io) {
    WidePlan& w = wide_;
    const size_t nOut = io.nOut, numSamples = io.numSamples;
    if (io.voiceOut) {
        // The channels no root of a voice aims at stay zero from block to block: the whole buffer is cleared only when the rows the
        // scatter writes (or nOut) changed, or something else wrote it since (the narrow path, a reallocation).
        if (!w.outZeroValid || w.outZeroNOut != nOut || w.outZeroRows != w.dstRow) {
            if (!cuda(dmemset(dOutVoice_, 0, sizeof(float) * (size_t) numVoices_ * nOut * blockSize_), "memset voice out")) return rc::CudaError;
            w.outZeroValid = true; w.outZeroNOut = nOut; w.outZeroRows = w.dstRow;
        }
        if (!cuda(launch_voice_out_scatter(dOutCompact_, w.dDst, (int) w.dstRow.size(), dOutVoice_, blockSize_, (int) numSamples, stream_), "voice out scatter launch")) return rc::CudaError;
        if (!w.dstRow.empty() && numSamples) ++launches_;
    }
    if (io.mix) {
        auto ev = timedBegin();
        const int nBig = (int) w.segs.size() - w.nSmall;
        if (!cuda(launch_mix_reduce_wide(dPartial_, w.dRows, w.dSegs, w.nSmall, nBig, (int) nOut, io.mix + io.col, io.mixPitch,
                                         dWideScratch_, dWideTickets_, blockSize_, (int) numSamples, stream_, takeDeliver()), "wide mix reduce launch")) return rc::CudaError;
        timedEnd(ev, 1);
        launches_ += (w.nSmall > 0) + (nBig > 0);
    }
    return rc::Ok;
}

HostDeliver Engine::takeDeliver() {
    HostDeliver hd;
    if (!deliverArmed_ || !hMixHost_ || planOnly_) return hd;
    deliverArmed_ = false;
    deliverLaunched_ = true;
    hd.out = dMixHostAlias_; hd.flag = dMixFlagAlias_; hd.done = dDeliverDone_; hd.seq = ++deliverSeq_;
    return hd;
}

std::pair<cudaEvent_t, cudaEvent_t> Engine::timedBegin() {
    std::pair<cudaEvent_t, cudaEvent_t> ev{nullptr, nullptr};
    if (!timeKernels_) return ev;
    if (!eventPool_.empty()) { ev = eventPool_.back(); eventPool_.pop_back(); }
    else { cudaEventCreate(&ev.first); cudaEventCreate(&ev.second); }
    cudaEventRecord(ev.first, stream_);
    return ev;
}

void Engine::timedEnd(std::pair<cudaEvent_t, cudaEvent_t> ev, int kind) {
    if (!timeKernels_) return;
    cudaEventRecord(ev.second, stream_);
    timed_[kind].push_back(ev);
}

int Engine::peerBarrier() {
    Lock lk(mu_);
    if (planOnly_ || !peerAttached_ || peer_.world <= 1) return rc::Ok;
    dsetdev();
    if (!cuda(launch_mix_exchange(peer_, dMix_, 0, ++peerEpoch_, dPeerStatus_, stream_), "peer barrier launch")) return rc::CudaError;
    return rc::Ok;
}

double Engine::takeKernelTimeMs(uint64_t* count) {
    Lock lk(mu_);
    if (planOnly_) { if (count) *count = 0; return 0.0; }
    cudaStreamSynchronize(stream_);
    for (int k = 0; k < 4; ++k) {
        lastKindMs_[k] = 0.0; lastKindCount_[k] = timed_[k].size();
        for (auto& ev : timed_[k]) {
            float ms = 0.0f;
            if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) lastKindMs_[k] += ms;
            eventPool_.push_back(ev);
        }
        timed_[k].clear();
    }
    if (count) *count = lastKindCount_[0];
    return lastKindMs_[0];
}

int Engine::renderOffline(size_t nOut, size_t numBlocks, float* hostOut, size_t chunkBlocks) {
    Lock lk(mu_);
    if (planOnly_) return fail(rc::CudaError, "plan-only runtime (no CUDA device): rendering is impossible, there is no CPU fallback");
    if (!hostOut || nOut == 0 || nOut > (size_t) MAX_OUT_CHANNELS) return fail(rc::BadArgument, "renderOffline: bad arguments");
    return offlineLoop(nullptr, 0, nullptr, nullptr, hostOut, nOut, numBlocks * (size_t) blockSize_, chunkBlocks, nullptr);
}

// The arguments every offline call with inputs checks, before rendering anything (the engine lock is held).
int Engine::offlineArgs(const float* const* in, size_t nIn, const float* inVoices, float* voicesOut, size_t nOut) {
    if (in && inVoices) return fail(rc::BadArgument, "processOffline: shared and per-voice inputs are exclusive");
    if (nIn > 0 && !in && !inVoices) return fail(rc::BadArgument, "processOffline: nIn > 0 without inputs");
    if (nOut == 0 || nOut > (size_t) MAX_WIDE_OUT_CHANNELS || (voicesOut && nOut > (size_t) MAX_OUT_CHANNELS))
        return fail(rc::BadArgument, "processOffline: nOut must be 1..4096 (1..8 with per-voice outputs)");
    if (processAllReduce_ && peerAttached_ && peer_.world > 1)
        return fail(rc::BadArgument, "processOffline: the mix bus is not summed across GPUs offline (option process_allreduce = 0 renders this rank alone)");
    if (planOnly_) return fail(rc::CudaError, "plan-only runtime (no CUDA device): rendering is impossible, there is no CPU fallback");
    return rc::Ok;
}

int Engine::processOffline(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                           size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime) {
    Lock lk(mu_);
    const int r = offlineArgs(in, nIn, inVoices, voicesOut, nOut);
    if (r != rc::Ok) return r;
    return offlineLoop(nIn ? in : nullptr, nIn, nIn ? inVoices : nullptr, mixOut, voicesOut, nOut, numSamples, chunkBlocks, sampleTime);
}

int Engine::processOfflineEvents(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                                 size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime, int vb, int ve,
                                 BlockEventFn cb, void* user) {
    Lock lk(mu_);
    if (!cb) return fail(rc::BadArgument, "processOfflineEvents: no event callback");
    if (vb < 0 || vb > numVoices_ || ve > numVoices_ || (ve >= 0 && ve < vb))
        return fail(rc::BadArgument, "processOfflineEvents: the voice range is out of bounds");
    const int r = offlineArgs(in, nIn, inVoices, voicesOut, nOut);
    if (r != rc::Ok) return r;
    EventLog log;
    log.vb = vb; log.ve = ve; log.cb = cb; log.user = user;
    return offlineLoop(nIn ? in : nullptr, nIn, nIn ? inVoices : nullptr, mixOut, voicesOut, nOut, numSamples, chunkBlocks, sampleTime, &log);
}

int Engine::processOfflineReadouts(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                                   size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime,
                                   const int32_t* nodeIds, int numNodes, int vb, int count, float* a, float* b, uint8_t* fresh) {
    Lock lk(mu_);
    if (numNodes < 1 || !nodeIds) return fail(rc::BadArgument, "processOfflineReadouts: no node to poll");
    if (count < 1 || !a || !fresh) return fail(rc::BadArgument, "processOfflineReadouts: count < 1, or a or fresh is NULL");
    ReadoutLog ro;
    ro.nodes.assign(nodeIds, nodeIds + numNodes);
    if (std::set<int32_t>(ro.nodes.begin(), ro.nodes.end()).size() != ro.nodes.size()) return fail(rc::BadArgument, "processOfflineReadouts: a node is listed twice");
    ro.targets.resize((size_t) numNodes);
    for (int j = 0; j < numNodes; ++j) {
        const int r = readoutTargets(ro.nodes[j], vb, count, ro.targets[j]);
        if (r != rc::Ok) return r;
    }
    const int r = offlineArgs(in, nIn, inVoices, voicesOut, nOut);
    if (r != rc::Ok) return r;
    ro.vb = vb; ro.count = count; ro.a = a; ro.b = b; ro.fresh = fresh;
    ro.numBlocks = (numSamples + blockSize_ - 1) / blockSize_;
    return offlineLoop(nIn ? in : nullptr, nIn, nIn ? inVoices : nullptr, mixOut, voicesOut, nOut, numSamples, chunkBlocks, sampleTime, nullptr, &ro);
}

// The chunk loop of both offline entry points (the engine lock is held).  Blocks are enqueued back to back with no host synchronisation in
// between; chunk buffers of C blocks per row carry the inputs up and the outputs down, two of each on the device and two PINNED on the host.
// The user's buffers are pageable and strided; a 2-D copy straight from or into them would be staged by the driver row by row,
// synchronously.  So a chunk travels as ONE contiguous async copy between pinned and device memory, and this thread moves rows between the
// user's buffers and pinned memory while the GPU renders: it fills chunk k + 1's inputs (uploaded on their own stream) and scatters
// chunk k - 1's outputs while chunk k renders.  With an event log, K5 follows every block, the log travels down with the chunk's outputs
// and its events are delivered once the chunk is scattered.
int Engine::offlineLoop(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                        size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime, EventLog* log, ReadoutLog* ro) {
    dsetdev();
    const size_t bs = (size_t) blockSize_, numBlocks = (numSamples + bs - 1) / bs;
    if (numBlocks == 0) return rc::Ok;
    const bool perVoiceIn = inVoices != nullptr;
    const size_t inRows = perVoiceIn ? (size_t) numVoices_ * nIn : (in ? nIn : 0);
    const size_t outRows = voicesOut ? (size_t) numVoices_ * nOut : 0, mixRows = mixOut ? nOut : 0;
    const size_t maxRows = std::max(inRows, std::max(outRows, mixRows));
    if (log) {
        const int r = eventLogBegin(*log);
        if (r != rc::Ok) return r;
    }
    const size_t logWords = log ? log->blockWords : ro ? ro->blockWords() : 0;               // a block's event log or readout records
    const size_t blockFloats = std::max(maxRows * bs, logWords);                            // the largest chunk buffer, per block
    size_t C = chunkBlocks ? chunkBlocks : 8;
    while (C > 1 && blockFloats * C * sizeof(float) > ((size_t) 256 << 20)) C >>= 1;        // two chunk buffers of at most 256 MiB each
    if (C > numBlocks) C = numBlocks;
    const size_t W = C * bs, numChunks = (numBlocks + C - 1) / C;                           // W: floats per chunk row
    auto ensure = [&](OfflineBuf& b, size_t floats) {
        for (int i = 0; i < 2; ++i)
            if (!grow(b.dev[i], b.devFloats[i], floats, "cudaMalloc offline chunk") ||
                !grow(b.pinned[i], b.pinnedFloats[i], floats, "cudaMallocHost offline chunk", false, 1, true)) return false;
        return true;
    };
    if ((outRows && !ensure(offOut_, outRows * W)) || (inRows && !ensure(offIn_, inRows * W)) || (mixRows && !ensure(offMix_, mixRows * W)) ||
        (logWords && !ensure(offLog_, logWords * C))) return rc::CudaError;
    cudaStream_t copyStream = nullptr, upStream = nullptr;
    cudaEvent_t rendered[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr}, uploaded[2] = {nullptr, nullptr};
    int rcode = rc::Ok;
    for (int i = 0; i < 2; ++i) {
        if (outRows) cudaMemsetAsync(offOut_.dev[i], 0, outRows * W * sizeof(float), stream_);    // voices without a render sequence stay silent
        cudaEventCreateWithFlags(&rendered[i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&copied[i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&uploaded[i], cudaEventDisableTiming);
    }
    cudaStreamCreateWithFlags(&copyStream, cudaStreamNonBlocking);
    if (inRows) cudaStreamCreateWithFlags(&upStream, cudaStreamNonBlocking);
    steadyValid_ = false;
    auto stage = [&](size_t chunk) -> bool {       // user rows -> pinned slot (zero past numSamples) -> device slot
        const int slot = (int) (chunk & 1);
        if (!cuda(cudaEventSynchronize(uploaded[slot]), "wait for an offline input upload")) return false;   // the upload two chunks back
        float* const dst = offIn_.pinned[slot];
        const size_t s0 = chunk * W, n = std::min(W, numSamples - s0);
        for (size_t row = 0; row < inRows; ++row) {
            std::memcpy(dst + row * W, perVoiceIn ? inVoices + row * numSamples + s0 : in[row] + s0, n * sizeof(float));
            if (n < W) std::memset(dst + row * W + n, 0, (W - n) * sizeof(float));
        }
        cudaStreamWaitEvent(upStream, rendered[slot], 0);                                      // the chunk two back no longer reads the device slot
        if (!cuda(cudaMemcpyAsync(offIn_.dev[slot], dst, inRows * W * sizeof(float), cudaMemcpyHostToDevice, upStream), "H2D offline input chunk")) return false;
        return cuda(cudaEventRecord(uploaded[slot], upStream), "record an offline input upload");
    };
    struct Pending { bool valid = false; size_t chunk = 0, blocks = 0; int slot = 0; } prev;
    auto scatter = [&](const Pending& pc) {          // pinned chunk [row][W] -> user rows, truncated to numSamples
        if (!pc.valid) return;
        if (!cuda(cudaEventSynchronize(copied[pc.slot]), "wait for an offline chunk")) { rcode = rc::CudaError; return; }
        const size_t s0 = pc.chunk * W, width = std::min(pc.blocks * bs, numSamples - s0);
        for (size_t row = 0; row < outRows; ++row)
            std::memcpy(voicesOut + row * numSamples + s0, offOut_.pinned[pc.slot] + row * W, width * sizeof(float));
        for (size_t c = 0; c < mixRows; ++c)
            std::memcpy(mixOut[c] + s0, offMix_.pinned[pc.slot] + c * W, width * sizeof(float));
        if (log) rcode = eventLogReplay(*log, pc.slot, pc.chunk * C);
        if (ro)
            for (size_t k = 0; k < pc.blocks; ++k)
                readoutScatter(*ro, reinterpret_cast<const uint32_t*>(offLog_.pinned[pc.slot]) + k * logWords, pc.chunk * C + k);
    };
    if (inRows && !stage(0)) rcode = rc::CudaError;
    BlockIO io;                                                                                 // block b: column b % C of its chunk's slot
    io.nIn = nIn; io.nOut = nOut; io.numSamples = bs; io.perVoiceIn = perVoiceIn;
    io.inPitch = io.outPitch = io.mixPitch = (int) W;
    for (size_t b = 0; b < numBlocks && rcode == rc::Ok; ++b) {
        const size_t chunk = b / C, inChunk = b % C;
        const int slot = (int) (chunk & 1);
        if (inChunk == 0) {
            if (chunk >= 2) cudaStreamWaitEvent(stream_, copied[slot], 0);                       // the chunk two back has left these device buffers
            if (inRows) cudaStreamWaitEvent(stream_, uploaded[slot], 0);                         // this chunk's inputs have arrived
        }
        if (sampleTime) sampleTime_ = *sampleTime + (int64_t) (b * bs);                          // as process() with userData, block by block
        io.in = inRows ? offIn_.dev[slot] : nullptr;
        io.voiceOut = outRows ? offOut_.dev[slot] : nullptr;
        io.mix = mixRows ? offMix_.dev[slot] : nullptr;
        io.col = (int) (inChunk * bs);
        rcode = enqueueBlock(io);
        if (rcode == rc::Ok && log) rcode = eventLogBlock(*log, slot, inChunk);
        if (rcode == rc::Ok && ro) rcode = readoutBlock(*ro, slot, inChunk);
        const bool lastOfChunk = inChunk + 1 == C || b + 1 == numBlocks;
        if (rcode == rc::Ok && lastOfChunk) {
            // the pinned buffers of this slot were scattered when chunk - 1 was enqueued (below), i.e. before these copies are issued
            cudaEventRecord(rendered[slot], stream_);
            cudaStreamWaitEvent(copyStream, rendered[slot], 0);
            if (outRows && !cuda(cudaMemcpyAsync(offOut_.pinned[slot], offOut_.dev[slot], outRows * W * sizeof(float), cudaMemcpyDeviceToHost, copyStream), "D2H offline chunk")) rcode = rc::CudaError;
            if (mixRows && !cuda(cudaMemcpyAsync(offMix_.pinned[slot], offMix_.dev[slot], mixRows * W * sizeof(float), cudaMemcpyDeviceToHost, copyStream), "D2H offline mix chunk")) rcode = rc::CudaError;
            if (log && log->used[slot] && !cuda(cudaMemcpyAsync(offLog_.pinned[slot], offLog_.dev[slot], log->used[slot] * sizeof(uint32_t), cudaMemcpyDeviceToHost, copyStream), "D2H offline event log")) rcode = rc::CudaError;
            if (ro && !cuda(cudaMemcpyAsync(offLog_.pinned[slot], offLog_.dev[slot], (inChunk + 1) * logWords * sizeof(uint32_t), cudaMemcpyDeviceToHost, copyStream), "D2H offline readouts")) rcode = rc::CudaError;
            cudaEventRecord(copied[slot], copyStream);
            if (rcode == rc::Ok && inRows && chunk + 1 < numChunks && !stage(chunk + 1)) rcode = rc::CudaError;   // overlaps with this chunk's render
            Pending cur; cur.valid = true; cur.chunk = chunk; cur.blocks = inChunk + 1; cur.slot = slot;
            scatter(prev);                                                                      // overlaps with the GPU rendering what was just enqueued
            prev = cur;
        }
    }
    if (rcode == rc::Ok) scatter(prev);
    steadyValid_ = false;
    cudaStreamSynchronize(stream_);
    if (copyStream) { cudaStreamSynchronize(copyStream); cudaStreamDestroy(copyStream); }
    if (upStream) { cudaStreamSynchronize(upStream); cudaStreamDestroy(upStream); }
    for (int i = 0; i < 2; ++i) {
        if (rendered[i]) cudaEventDestroy(rendered[i]);
        if (copied[i]) cudaEventDestroy(copied[i]);
        if (uploaded[i]) cudaEventDestroy(uploaded[i]);
    }
    return rcode;
}

int Engine::synchronize() {
    if (planOnly_) return rc::Ok;
    const cudaError_t e = cudaStreamSynchronize(stream_);     // no lock while waiting for the GPU
    if (e == cudaSuccess) return rc::Ok;
    Lock lk(mu_);
    cuda(e, "stream synchronize");
    return rc::CudaError;
}

int Engine::process(const float* const* in, size_t nIn, float* const* out, size_t nOut, size_t numSamples, const int64_t* sampleTime) {
    float* hOut = nullptr;
    uint32_t waitSeq = 0;
    bool polled = false;
    {
        Lock lk(mu_);   // held while the block is ENQUEUED; the wait for the GPU below runs without it (the control thread may work meanwhile)
        if (planOnly_) return fail(rc::CudaError, "plan-only runtime (no CUDA device): rendering is impossible, there is no CPU fallback");
        dsetdev();
        if (sampleTime) sampleTime_ = *sampleTime;   // BlockContext::userData as the wasm host passes it (wasm/Main.cpp:206-215)
        if (numSamples > (size_t) blockSize_) return fail(rc::BadArgument, "numSamples > blockSize");
        if (!grow(hPinned_, pinnedFloats_, (nIn + nOut) * blockSize_, "cudaMallocHost", false, 1, true)) return rc::CudaError;
        if (nIn) {
            float* d = sharedInDevicePtr(nIn);
            if (!d) return rc::CudaError;
            for (size_t c = 0; c < nIn; ++c) std::memcpy(hPinned_ + c * blockSize_, in[c], sizeof(float) * numSamples);
            if (!cuda(dmemcpy(d, hPinned_, sizeof(float) * nIn * blockSize_, cudaMemcpyHostToDevice), "H2D inputs")) return rc::CudaError;
        }
        // With peers attached every rank's process() returns the mix of ALL ranks (K4), like one Runtime over all the voices would.
        deliverArmed_ = hostDeliver_ && nOut > 0 && hMixHost_ != nullptr;
        deliverLaunched_ = false;
        int r = enqueueBlock(nIn, nOut, numSamples, false, false, true, processAllReduce_ && peerAttached_ && peer_.world > 1);
        deliverArmed_ = false;
        if (r != rc::Ok) return r;
        if (deliverLaunched_) {
            hOut = hMixHost_;
            waitSeq = deliverSeq_;
            polled = true;
        } else {
            hOut = hPinned_ + nIn * blockSize_;
            if (nOut) {
                if (!cuda(dmemcpy(hOut, dMix_, sizeof(float) * nOut * blockSize_, cudaMemcpyDeviceToHost), "D2H mix")) return rc::CudaError;
            }
        }
    }
    if (polled) {
        // The kernel that finishes the mix bus has stored it into mapped host memory and raises the sequence word behind it: poll that
        // word (no D2H copy launch, no stream synchronize wake-up).  A failed launch never raises it — the stream is queried every
        // ~20 us so that an error (or a finished stream) ends the wait.
        using clk = std::chrono::steady_clock;
        auto lastQuery = clk::now();
        for (;;) {
            if (*hMixFlag_ == waitSeq) break;
            for (int k = 0; k < 32; ++k) cpuRelax();
            const auto now = clk::now();
            if (now - lastQuery > std::chrono::microseconds(20)) {
                lastQuery = now;
                const cudaError_t q = cudaStreamQuery(stream_);
                if (q == cudaErrorNotReady) continue;
                if (q != cudaSuccess) { Lock lk(mu_); cuda(q, "stream query while waiting for the mix bus"); return rc::CudaError; }
                if (*hMixFlag_ == waitSeq) break;
                Lock lk(mu_);
                return fail(rc::CudaError, "the render stream finished without delivering the mix bus");
            }
        }
        std::atomic_thread_fence(std::memory_order_acquire);
    } else {
        int r = synchronize();
        if (r != rc::Ok) return r;
    }
    // hPinned_ belongs to the render thread: only process() (re)allocates it
    for (size_t c = 0; c < nOut; ++c) std::memcpy(out[c], hOut + c * blockSize_, sizeof(float) * numSamples);
    return rc::Ok;
}

int Engine::processVoices(const float* in, size_t nIn, float* outVoices, float* mix, size_t nOut, size_t numSamples) {
    {
        Lock lk(mu_);
        if (planOnly_) return fail(rc::CudaError, "plan-only runtime (no CUDA device): rendering is impossible, there is no CPU fallback");
        dsetdev();
        if (numSamples > (size_t) blockSize_) return fail(rc::BadArgument, "numSamples > blockSize");
        const bool perVoiceIn = in != nullptr && nIn > 0;
        if (perVoiceIn) {
            float* d = voiceInDevicePtr(nIn);
            if (!d) return rc::CudaError;
            // host layout [voice][nIn][numSamples] -> device [voice][nIn][blockSize]
            if (!cuda(cudaMemcpy2DAsync(d, sizeof(float) * blockSize_, in, sizeof(float) * numSamples, sizeof(float) * numSamples,
                                        (size_t) numVoices_ * nIn, cudaMemcpyHostToDevice, stream_), "H2D voice inputs")) return rc::CudaError;
        }
        int r = enqueueBlock(nIn, nOut, numSamples, perVoiceIn, outVoices != nullptr, mix != nullptr);
        if (r != rc::Ok) return r;
        if (outVoices) {
            if (!cuda(cudaMemcpy2DAsync(outVoices, sizeof(float) * numSamples, dOutVoice_, sizeof(float) * blockSize_, sizeof(float) * numSamples,
                                        (size_t) numVoices_ * nOut, cudaMemcpyDeviceToHost, stream_), "D2H voice outputs")) return rc::CudaError;
        }
        if (mix) {
            if (!cuda(cudaMemcpy2DAsync(mix, sizeof(float) * numSamples, dMix_, sizeof(float) * blockSize_, sizeof(float) * numSamples,
                                        nOut, cudaMemcpyDeviceToHost, stream_), "D2H mix")) return rc::CudaError;
        }
    }
    return synchronize();
}

} // namespace eb
