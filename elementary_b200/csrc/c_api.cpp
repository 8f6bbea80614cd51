// c_api.cpp — extern "C" shim over eb::Engine; see include/elem_b200.h for the contract and the reference
// interface each entry point replaces.
#include "../../include/elem_b200.h"

#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "graph_host.h"
#include "kernels.h"

static_assert(eb::MAX_WIDE_OUT_CHANNELS == ELEM_B200_MAX_OUT_CHANNELS, "the header documents the output channel cap");

struct elem_b200_runtime {
    eb::Engine* engine;
    std::string scratch;
};

static thread_local std::string g_createError;

extern "C" {

int elem_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

elem_b200_runtime* elem_b200_create(double sampleRate, int blockSize, int numVoices, int device) {
    if (blockSize <= 0 || numVoices <= 0 || sampleRate <= 0) { g_createError = "bad argument"; return nullptr; }
    // device == -1: plan-only runtime — the host logic (instruction interpreter, return codes, gc, graph
    // compilation) runs without a GPU; every process/enqueue call fails with -1.  Used by the CPU test-suite.
    if (device != -1) {
        int n = elem_b200_device_count();
        if (device < 0 || device >= n) { g_createError = "no such CUDA device (this library has no CPU fallback)"; return nullptr; }
    }
    try {
        auto* rt = new elem_b200_runtime{new eb::Engine(sampleRate, blockSize, numVoices, device), {}};
        if (!rt->engine->mixDevicePtr()) { g_createError = rt->engine->lastError(); delete rt->engine; delete rt; return nullptr; }
        return rt;
    } catch (const std::exception& e) {
        g_createError = e.what();
        return nullptr;
    }
}

void elem_b200_destroy(elem_b200_runtime* rt) {
    if (!rt) return;
    delete rt->engine;
    delete rt;
}

#define GUARD(expr)                                                   \
    if (!rt) return eb::rc::BadArgument;                              \
    try { return (expr); }                                            \
    catch (const std::bad_alloc&) { return eb::rc::InvariantViolation; } \
    catch (...) { return eb::rc::InvalidInstructionFormat; }

int elem_b200_apply_instructions(elem_b200_runtime* rt, int voiceBegin, int voiceEnd, const char* json, size_t len) {
    if (!json) return eb::rc::BadArgument;
    GUARD(rt->engine->applyInstructions(voiceBegin, voiceEnd, json, len));
}

int elem_b200_apply_binary(elem_b200_runtime* rt, int voiceBegin, int voiceEnd, const void* data, size_t bytes) {
    if (!data) return eb::rc::BadArgument;
    GUARD(rt->engine->applyBinary(voiceBegin, voiceEnd, data, bytes));
}

int elem_b200_set_const_table(elem_b200_runtime* rt, const int32_t* nodeIds, int numProps, const float* values, int voiceBegin, int count) {
    if (!nodeIds || !values) return eb::rc::BadArgument;
    GUARD(rt->engine->setConstTable(nodeIds, numProps, values, voiceBegin, count));
}

int elem_b200_set_property_per_voice(elem_b200_runtime* rt, int32_t nodeId, const char* key, const double* values, int voiceBegin, int count) {
    if (!key || !values) return eb::rc::BadArgument;
    GUARD(rt->engine->setPropertyPerVoice(nodeId, key, values, voiceBegin, count));
}

int elem_b200_set_path_per_voice(elem_b200_runtime* rt, int32_t nodeId, const char* const* names, int numNames, const int32_t* index, int voiceBegin, int count) {
    if ((numNames > 0 && !names) || (count > 0 && !index)) return eb::rc::BadArgument;
    GUARD(rt->engine->setPathPerVoice(nodeId, names, numNames, index, voiceBegin, count));
}

int elem_b200_set_seq_per_voice(elem_b200_runtime* rt, int32_t nodeId, const char* const* seqs, int numSeqs, const int32_t* index, int voiceBegin, int count) {
    if ((numSeqs > 0 && !seqs) || (count > 0 && !index)) return eb::rc::BadArgument;
    GUARD(rt->engine->setSeqPerVoice(nodeId, seqs, numSeqs, index, voiceBegin, count));
}

int elem_b200_reset_voices(elem_b200_runtime* rt, const int32_t* voices, size_t count) {
    if (count > 0 && !voices) return eb::rc::BadArgument;
    GUARD(rt->engine->resetVoices(voices, count));
}
uint64_t elem_b200_reset_bytes_written(elem_b200_runtime* rt) { return rt ? rt->engine->resetBytesWritten() : 0; }

int elem_b200_process(elem_b200_runtime* rt, const float* const* in, size_t nIn, float* const* out, size_t nOut, size_t numSamples, void* userData) {
    GUARD(rt->engine->process(in, nIn, out, nOut, numSamples, static_cast<const int64_t*>(userData)));
}

void elem_b200_set_current_time(elem_b200_runtime* rt, int64_t sampleTime) { if (rt) rt->engine->setCurrentTime(sampleTime); }
int64_t elem_b200_current_time(elem_b200_runtime* rt) { return rt ? rt->engine->currentTime() : 0; }

int elem_b200_process_voices(elem_b200_runtime* rt, const float* in, size_t nIn, float* outVoices, float* mix, size_t nOut, size_t numSamples) {
    GUARD(rt->engine->processVoices(in, nIn, outVoices, mix, nOut, numSamples));
}

int elem_b200_render_offline(elem_b200_runtime* rt, size_t nOut, size_t numBlocks, float* hostOut, size_t chunkBlocks) {
    GUARD(rt->engine->renderOffline(nOut, numBlocks, hostOut, chunkBlocks));
}

int elem_b200_process_offline(elem_b200_runtime* rt, const float* const* in, size_t nIn, const float* inVoices,
                              float* const* mixOut, float* voicesOut, size_t nOut, size_t numSamples, size_t chunkBlocks, void* userData) {
    GUARD(rt->engine->processOffline(in, nIn, inVoices, mixOut, voicesOut, nOut, numSamples, chunkBlocks, static_cast<const int64_t*>(userData)));
}

int elem_b200_process_offline_events(elem_b200_runtime* rt, const float* const* in, size_t nIn, const float* inVoices,
                                     float* const* mixOut, float* voicesOut, size_t nOut, size_t numSamples,
                                     size_t chunkBlocks, void* userData, int voiceBegin, int voiceEnd,
                                     elem_b200_block_event_cb cb, void* user) {
    GUARD(rt->engine->processOfflineEvents(in, nIn, inVoices, mixOut, voicesOut, nOut, numSamples, chunkBlocks, static_cast<const int64_t*>(userData),
                                           voiceBegin, voiceEnd, cb, user));
}

int elem_b200_process_offline_readouts(elem_b200_runtime* rt, const float* const* in, size_t nIn, const float* inVoices,
                                       float* const* mixOut, float* voicesOut, size_t nOut, size_t numSamples,
                                       size_t chunkBlocks, void* userData,
                                       const int32_t* nodeIds, int numNodes, int voiceBegin, int count,
                                       float* a, float* b, uint8_t* fresh) {
    GUARD(rt->engine->processOfflineReadouts(in, nIn, inVoices, mixOut, voicesOut, nOut, numSamples, chunkBlocks, static_cast<const int64_t*>(userData),
                                             nodeIds, numNodes, voiceBegin, count, a, b, fresh));
}

int elem_b200_enqueue_block(elem_b200_runtime* rt, size_t nIn, size_t nOut, size_t numSamples, int flags) {
    GUARD(rt->engine->enqueueBlock(nIn, nOut, numSamples, (flags & 1) != 0, (flags & 2) != 0, (flags & 4) != 0, (flags & 8) != 0));
}

int elem_b200_peer_export(elem_b200_runtime* rt, void* handleOut64) {
    if (!handleOut64) return eb::rc::BadArgument;
    GUARD(rt->engine->peerExport(handleOut64));
}
int elem_b200_peer_attach(elem_b200_runtime* rt, int rank, int world, const void* handles) {
    if (!handles) return eb::rc::BadArgument;
    GUARD(rt->engine->peerAttach(rank, world, handles));
}
int elem_b200_peer_status(elem_b200_runtime* rt) { return rt ? rt->engine->peerStatus() : 0; }
int elem_b200_peer_barrier(elem_b200_runtime* rt) { GUARD(rt->engine->peerBarrier()); }

int elem_b200_synchronize(elem_b200_runtime* rt) { GUARD(rt->engine->synchronize()); }

float* elem_b200_mix_device(elem_b200_runtime* rt) { return rt ? rt->engine->mixDevicePtr() : nullptr; }
float* elem_b200_voice_out_device(elem_b200_runtime* rt) { return rt ? rt->engine->voiceOutDevicePtr() : nullptr; }
float* elem_b200_voice_in_device(elem_b200_runtime* rt, size_t nIn) { return rt ? rt->engine->voiceInDevicePtr(nIn) : nullptr; }
float* elem_b200_shared_in_device(elem_b200_runtime* rt, size_t nIn) { return rt ? rt->engine->sharedInDevicePtr(nIn) : nullptr; }
void elem_b200_set_stream(elem_b200_runtime* rt, void* s) { if (rt) rt->engine->setStream(static_cast<cudaStream_t>(s)); }

int elem_b200_add_shared_resource(elem_b200_runtime* rt, const char* name, const float* const* channels, size_t numChannels, size_t numSamples) {
    if (!rt || !name) return 0;
    try { return rt->engine->addSharedResource(name, channels, numChannels, numSamples); } catch (...) { return 0; }
}

void elem_b200_prune_shared_resources(elem_b200_runtime* rt) { if (rt) rt->engine->pruneSharedResources(); }

int elem_b200_list_shared_resources(elem_b200_runtime* rt, char* buf, size_t cap) {
    if (!rt) return 0;
    auto names = rt->engine->listSharedResources();
    std::string s;
    for (auto& n : names) { s += n; s += '\n'; }
    if (buf && cap) {
        const size_t k = s.size() < cap - 1 ? s.size() : cap - 1;
        std::memcpy(buf, s.data(), k);
        buf[k] = 0;
    }
    return (int) names.size();
}

int elem_b200_gc(elem_b200_runtime* rt, int voice, int32_t* ids, size_t cap) {
    if (!rt) return 0;
    std::vector<int32_t> pruned;
    rt->engine->gc(voice, pruned);
    for (size_t i = 0; i < pruned.size() && i < cap; ++i) ids[i] = pruned[i];
    return (int) pruned.size();
}

void elem_b200_reset(elem_b200_runtime* rt) { if (rt) rt->engine->reset(); }

namespace {
struct EventTrampoline { elem_b200_event_cb cb; void* user; };
void relayEvent(const char* type, const char* json, int /*voice*/, void* t) {
    auto* tr = static_cast<EventTrampoline*>(t);
    if (tr->cb) tr->cb(type, json, tr->user);
}
}

int elem_b200_process_queued_events_range(elem_b200_runtime* rt, int voiceBegin, int voiceEnd, elem_b200_event_cb cb, void* user) {
    EventTrampoline tr{cb, user};
    GUARD(rt->engine->processQueuedEvents(voiceBegin, voiceEnd, relayEvent, &tr));
}

void elem_b200_process_queued_events(elem_b200_runtime* rt, elem_b200_event_cb cb, void* user) {
    (void) elem_b200_process_queued_events_range(rt, 0, -1, cb, user);
}

int elem_b200_poll_readouts(elem_b200_runtime* rt, int32_t nodeId, int voiceBegin, int count, float* a, float* b, uint8_t* fresh, int flags) {
    GUARD(rt->engine->pollReadouts(nodeId, voiceBegin, count, a, b, fresh, (flags & ELEM_B200_READOUT_DEVICE) != 0));
}

int elem_b200_node_type(elem_b200_runtime* rt, int voice, int32_t nodeId, char* buf, size_t cap) {
    if (!rt) return 0;
    try {
        const std::string s = rt->engine->nodeType(voice, nodeId);
        if (s.empty()) return 0;
        if (buf && cap) { const size_t k = s.size() < cap - 1 ? s.size() : cap - 1; std::memcpy(buf, s.data(), k); buf[k] = 0; }
        return (int) s.size() + 1;
    } catch (...) { return 0; }
}

int elem_b200_set_option(elem_b200_runtime* rt, const char* key, double value) {
    if (!key) return eb::rc::BadArgument;
    GUARD(rt->engine->setOption(key, value));
}

int elem_b200_describe(elem_b200_runtime* rt, char* buf, size_t cap) {
    if (!rt) return 0;
    const std::string s = rt->engine->describe();
    if (buf && cap) {
        const size_t k = s.size() < cap - 1 ? s.size() : cap - 1;
        std::memcpy(buf, s.data(), k);
        buf[k] = 0;
    }
    return (int) s.size() + 1;
}

int elem_b200_register_node_type(elem_b200_runtime* rt, const char* type, int numInputs, int numStateFloats, const char* cudaBody) {
    if (!type || !cudaBody) return eb::rc::BadArgument;
    GUARD(rt->engine->registerNodeType(type, numInputs, numStateFloats, cudaBody));
}
int elem_b200_has_node_type(elem_b200_runtime* rt, const char* type) { return (rt && type && rt->engine->hasNodeType(type)) ? 1 : 0; }

int elem_b200_snapshot(elem_b200_runtime* rt, int voice, char* buf, size_t cap) {
    if (!rt) return 0;
    try {
        const std::string s = rt->engine->snapshot(voice);
        if (buf && cap) { const size_t k = s.size() < cap - 1 ? s.size() : cap - 1; std::memcpy(buf, s.data(), k); buf[k] = 0; }
        return (int) s.size() + 1;
    } catch (...) { return 0; }
}

int elem_b200_debug_opprof(elem_b200_runtime* rt, unsigned long long* out128, int reset) {
    if (!rt || !out128) return -1;
    rt->engine->synchronize();
    if (eb::debug_opprof_read(out128, reset != 0) != cudaSuccess) return -1;
    return rt->engine->specOpprofRead(out128, reset != 0) ? 0 : -1;     // + specialised kernels compiled with option spec_opprof
}

int elem_b200_program_words(elem_b200_runtime* rt, int voice, uint32_t* buf, size_t cap) {
    if (!rt) return 0;
    try {
        auto w = rt->engine->programWords(voice);
        if (buf) std::memcpy(buf, w.data(), sizeof(uint32_t) * (w.size() < cap ? w.size() : cap));
        return (int) w.size();
    } catch (...) { return 0; }
}

long elem_b200_specialize_dry_run(elem_b200_runtime* rt, int voice, char* logBuf, size_t cap) {
    if (!rt) return -1;
    try {
        std::string log;
        const long n = rt->engine->specializeDryRun(voice, log);
        if (logBuf && cap) { const size_t k = log.size() < cap - 1 ? log.size() : cap - 1; std::memcpy(logBuf, log.data(), k); logBuf[k] = 0; }
        return n;
    } catch (...) { return -1; }
}

uint64_t elem_b200_kernel_launches(elem_b200_runtime* rt) { return rt ? rt->engine->kernelLaunches() : 0; }

double elem_b200_take_kernel_time_ms(elem_b200_runtime* rt, uint64_t* count) {
    if (!rt) { if (count) *count = 0; return 0.0; }
    return rt->engine->takeKernelTimeMs(count);
}

double elem_b200_last_convolve_time_ms(elem_b200_runtime* rt, uint64_t* count) {
    if (!rt) { if (count) *count = 0; return 0.0; }
    return rt->engine->lastConvolveTimeMs(count);
}

void elem_b200_last_kernel_times(elem_b200_runtime* rt, double* ms4, uint64_t* counts4) {
    double ms[4] = {0, 0, 0, 0};
    uint64_t n[4] = {0, 0, 0, 0};
    if (rt) rt->engine->lastKernelTimes(ms, n);
    for (int i = 0; i < 4; ++i) { if (ms4) ms4[i] = ms[i]; if (counts4) counts4[i] = n[i]; }
}

const char* elem_b200_last_error(elem_b200_runtime* rt) {
    if (!rt) return g_createError.c_str();
    rt->scratch = rt->engine->lastError();
    return rt->scratch.c_str();
}

const char* elem_b200_describe_return_code(int c) {   // Types.h:62-85
    switch (c) {
        case 0: return "Ok";
        case 1: return "Node type not recognized";
        case 2: return "Node not found";
        case 3: return "Attempting to create a node that already exists";
        case 4: return "Attempting to create a node type that already exists";
        case 5: return "Invalid value type for the given node property";
        case 6: return "Invalid value for the given node property";
        case 7: return "Invariant violation";
        case 8: return "Invalid instruction format";
        case -1: return "CUDA error";
        case -2: return "Bad argument";
        default: return "Return code not recognized";
    }
}

} // extern "C"
