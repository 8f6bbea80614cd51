// graph_host.h — host side of the H100 engine: the part of elem::Runtime (runtime/elem/Runtime.h:40-577) that
// is NOT the per-block walk: node table, instruction interpreter, DFS topological sort, root activation and
// fades, garbage collection, shared resources — plus what is new here: voice groups, device storage and the
// compilation of the sorted node list into a render program (program.h) for the fused kernel.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "convolve.h"
#include "kernels.h"
#include "program.h"
#include "value.h"

namespace eb {

// Same numbering as elem::ReturnCode (runtime/elem/Types.h:51-60); negative values are ours (CUDA failures).
namespace rc {
constexpr int Ok = 0, UnknownNodeType = 1, NodeNotFound = 2, NodeAlreadyExists = 3, NodeTypeAlreadyExists = 4,
              InvalidPropertyType = 5, InvalidPropertyValue = 6, InvariantViolation = 7, InvalidInstructionFormat = 8;
constexpr int CudaError = -1, BadArgument = -2;
}

enum class NodeKind : uint8_t {
    In, Unary, Binary, Reduce, Root, Const, Sr, Phasor, SPhasor, Counter, Accum, Latch, MaxHold, Rand,
    Delay, SDelay, Z, Pole, Env, Biquad, Prewarp, MM1p, Svf, SvfShelf, TapIn, TapOut, Table, Blep, Convolve,
    PassThrough,  // analysis nodes whose events are not produced: audio passes through
    Once, Seq, Seq2, SparSeq, SparSeq2, Time, Metro,  // sequencing / control nodes (SURVEY.md §8f N3)
    Meter, Snapshot, Scope, Capture, Fft,             // analysis nodes feeding processQueuedEvents (SURVEY.md §8f N4)
    Custom,                                           // a device node type registered at run time (registerNodeType)
    Sample                                            // sample playback (Sample.h)
};

// A read-only device array owned jointly by the node that uploaded it and by every compiled program that points at it
// (sequence data of seq/seq2/sparseq/sparseq2: the reference hands such data to the audio thread through a
// RefCountedPool + SPSC queue, Core.h:447-466).
struct DeviceArray {
    void* d = nullptr;
    size_t bytes = 0, count = 0;
    bool planOnly = false;
    ~DeviceArray();
};
struct VoiceArray;   // graph_host.cpp: the per-voice setters
struct Node;
struct Group;
// One voice group a per-voice call reaches: node n of group g, group-relative voices [b, e), which are voices [at, at + e - b) of the call.
struct VoiceTarget { Group& g; Node& n; int b, e, at; int last() const { return at + e - b - 1; } };

struct Inlet { int32_t source; int32_t channel; };

// Float mirror of helpers/GainFade.h:16-121 (only what RootNode uses).
struct GainFade {
    float current = 0.0f, target = 1.0f, step = 0.0f, inStep = 0.0f, outStep = 0.0f;
    void init(double sr);
    void setFadeInMs(double sr, double ms);
    void setFadeOutMs(double sr, double ms);
    void fadeIn()  { target = 1.0f; updateStep(); }
    void fadeOut() { target = 0.0f; updateStep(); }
    bool on() const { return target > 0.5f; }
    bool settled() const;
    void advance(int numSamples);   // what GainFade::process does to currentGain after a block
    void updateStep() { step = (current > target) ? outStep : inStep; }
};

struct Resource {
    std::string name;
    std::vector<std::vector<float>> channels;   // host copy (always float: AudioBufferResource.h:13-24)
    float* dChannel0 = nullptr;                 // device copy of channel 0 (padded with zeros to a multiple of 16 bytes: TMA bulk copies)
    size_t numSamples = 0;
};

struct ConvolverState;   // convolve.h
struct SpecKernel;       // spec_host.h
struct SpecJob;

struct Node {
    int32_t id = 0;
    NodeKind kind = NodeKind::Const;
    uint32_t fn = 0;                 // UnaryFn / BinaryFn / ReduceFn / blep mode
    std::string typeName;
    std::vector<Inlet> inlets;
    std::map<std::string, Value> props;

    int paramRow = -1;               // const / sr: per-voice parameter row; sample, seq family (from its first setSeqPerVoice): the first of its rows
    int stateRow = -1;               // first scalar state row (even-aligned when it holds doubles)
    int shadowRow = -1;              // rand / once: the seed / arm last set for each voice, outside the state rows (resetVoices)
    int mode = 0;                    // svf / svfshelf / mm1p / sample mode
    int channel = 0;                 // in.channel, root.channel (-1 default for root)
    GainFade fade;                   // root
    int size = 0, length = 0;        // delay / sdelay
    bool ringDirty = true;           // (re)allocate + zero + reset writeIndex at next compile (Delays.h:92-95)
    float* ring = nullptr;
    size_t ringFloats = 0;
    int ringPositions = 0;           // the ring is [tile][ringPositions][L] floats
    uint32_t holdSamples = 0xFFFFFFFFu;   // maxhold
    std::string tapName;
    float* tapPrivate = nullptr;     // tapOut private delayBuffer
    std::shared_ptr<Resource> resource;   // table / convolve
    std::vector<std::shared_ptr<const void>> voiceArrays;   // sample / seq family with paramRow >= 0: keeps each voice's buffer (Resource) or sequence (DeviceArray) alive
    bool resourceDirty = false;
    std::shared_ptr<ConvolverState> conv;
    // seq / seq2 / sparseq / sparseq2 (Core.h:411-466, Seq2.h:39-84, SparSeq.h:40-124, SparSeq2.h:20-56)
    std::shared_ptr<DeviceArray> seqData;
    uint32_t seqGen = 0, loopGen = 0;
    bool seqHold = false, seqLoop = true, follow = false;
    uint64_t seqOffset = 0;
    int32_t loopStart = -1, loopEnd = -1, interpolate = 0;
    double tickIntervalSamples = 0.0;
    int64_t intervalSamps = 0;       // metro (wasm/Metro.h:24-34)
    // event side (SURVEY.md §8f N4).  Ring positions that evolve identically for every voice of the group are mirrored
    // on the host: scope's MultiChannelRingBuffer read/write positions (MultiChannelRingBuffer.h:36-96), metro's
    // eventFlag/lastOut (Metro.h:47-52).  capture's relayBuffer (Capture.h:62-72) is a host vector per voice.
    uint32_t scopeR = 0, scopeW = 0;
    bool metroFlag = false; float metroLastOut = 0.0f;
    std::vector<std::vector<float>> relay;
    std::vector<float> window;       // fft: Blackman-Harris window of the current size (wasm/FFT.h:49-62)
};

struct Program {
    std::vector<uint32_t> code;
    std::vector<uint32_t> stateMap;
    std::vector<uint32_t> paramMap;       // shared-memory parameter row i+1 <- global row paramMap[i]
    int nOps = 0;
    int nStateRows = 0;
    int nSlots = 1;
    int nDelayBuf = 0;           // OP_DELAY ops (aux1 = 1 + the index of the op's read-window buffer, LaunchParams::nDelayBuf)
    int nIn = 0;
    bool usesHostInputs = false;
    std::vector<int32_t> rootIds;         // root index -> node id
    std::vector<int32_t> nodeIds;         // every node referenced (gc liveness)
    uint32_t* dCode = nullptr;
    uint32_t* dStateMap = nullptr;
    uint32_t* dParamMap = nullptr;
    bool planOnly = false;
    // warp pipeline of a one-voice program (LaunchParams::pipeW ...): filled by compile() when the program was cut
    int pipeW = 1, pipeRingBase = 0, pipeDepth = 1;
    uint32_t pipeCode[MAX_PIPE] = {0, 0, 0, 0};
    unsigned short pipeState[MAX_PIPE + 1] = {0, 0, 0, 0, 0}, pipeSrow[MAX_PIPE] = {0, 0, 0, 0};
    // K1 stages: stage k interprets code[stages[k].codeOffset ...]; after it the convolvers of that stage run (K3)
    struct Conv { int32_t node; float* in; float* out; int inChannel; };   // inChannel >= 0: K3 reads host input channel inChannel directly (no staging copy)
    struct Stage { uint32_t codeOffset = 0; std::vector<Conv> convolves; bool empty = false; };   // empty: no K1 work in this stage
    std::vector<Stage> stages;
    // `convolve -> root`: the last stage would only reload the convolver's output and apply the root — K3 does that in its epilogue
    // (convolve.h ConvEpilogue) and the stage's K1 launch is skipped.  fusedConvStage < 0: not fused.
    int fusedConvStage = -1, fusedConvIndex = 0, fusedRoot = 0;
    std::vector<float*> blockBuffers;     // [Vpad][blockSize] HBM buffers carrying values across stages
    std::vector<std::shared_ptr<DeviceArray>> pinned;   // device arrays the code points at
    struct EvNode { int32_t node; int root; };
    std::vector<EvNode> evNodes;          // event-emitting nodes in render order (GraphRenderSequence.h:189-198 walks nodeList)
    std::vector<int32_t> dynNodes;        // LaunchParams::dyn[i] belongs to node dynNodes[i]
    bool hasCustom = false;               // uses a registered device node type: only a specialised kernel can run it
    std::shared_ptr<SpecJob> specJob;     // K1 being / having been specialised for this program (option "specialize"); the interpreter runs until it is loaded
    const float* stagedTable = nullptr; int stagedTableFloats = 0;   // the wavetable K1 stages into shared memory with TMA (first `table` node that fits)
    ~Program();
};

struct Group {
    int v0 = 0, nv = 0, Vpad = 0;
    int tileWidth = 0;                    // L, fixed at first compile
    std::unordered_map<int32_t, Node> nodes;
    std::set<int32_t> currentRoots;
    float* dRows = nullptr;
    int rowsCap = 0, rowsUsed = 0;
    std::map<std::string, float*> tapShared;
    std::shared_ptr<Program> pending, active;
    bool codeDirty = false;               // a property that is baked into the program changed: recompile at the next process()
    std::vector<std::shared_ptr<Program>> superseded;   // queued but never run (rseqQueue, Runtime.h:133,277-285): still pin their nodes for gc
    int nTiles() const { return tileWidth ? (nv + tileWidth - 1) / tileWidth : 0; }
};

struct EngineOptions {
    int tileWidth = 0;            // 0 = choose per group from the voice count
    int warpsPerCta = 0;          // 0 = choose
    int targetTiles = 2048;       // shrink the tile width until about this many warps exist (4096 voices -> L = 2)
    bool targetTilesSet = false;  // the option was given explicitly: no automatic choice (see Engine::midRangeDense)
    int niter = 0;                // 0 = default elements-per-lane per tile; 4 selects the T = 4 variant for L = 32
    bool batchGroups = true;      // launch all single-stage voice groups of one tile geometry together
    bool fuseChains = true;       // fold runs of element-wise nodes into one OP_CHAIN
    int specialize = 0;           // spec_host.h: NVRTC-compile K1 against each small single-stage program; 1 = on the compile-queue thread
                                  // (the interpreter serves meanwhile), 2 = wait for the compiler at COMMIT (benchmarks, parity runs)
    int specializeMaxWords = 512; // programs longer than this keep the interpreter (compile time grows with the unrolled program)
    bool fuseConvRoot = true;     // `convolve -> root`: root gain + per-voice output + partial mix in K3's epilogue, no K1 launch for the last stage
    int pipelineStages = 3;       // one-voice groups in the many-groups launch: cut the program into this many pipeline stages, one warp each
                                  // (render_groups_pipe_kernel; 0 / 1 = off).  Bit-identical to one warp per graph; on an H100, BASELINE
                                  // config 5 takes 0.66 ms per block at 3 stages against 0.71 at 4 and 0.73 unpipelined — per-op time grows
                                  // with the number of resident warps, so the gain is far from the stage count (DESIGN.md section 4)
    int specMinBlocks = 0;        // > 0: specialised kernels of the narrow geometries (1 < L < 32) are compiled for this many CTAs per SM (8 = 64 registers)
    bool specializeStrict = false; // a failed specialisation is an error (COMMIT returns 7 / process -1) instead of a silent stay on the interpreter
    bool specOpprof = false;      // specialised kernels carry the per-opcode cycle counters (-DEB_OPPROF; tools/spec_opprof.py); profiling only
};

class Engine {
public:
    Engine(double sampleRate, int blockSize, int numVoices, int device);
    ~Engine();

    int applyInstructions(int voiceBegin, int voiceEnd, const char* json, size_t len);
    int setPropertyPerVoice(int32_t nodeId, const char* key, const double* values, int voiceBegin, int count);
    // Instruction-stream ingestion at scale (SURVEY.md §8f N2).  applyBinary: the SAME instruction stream in the binary encoding
    // documented in include/elem_b200.h (no text to parse: ids are int32, numbers float64, strings length-prefixed), decoded into the
    // same in-memory batch and run through the same interpreter — identical semantics and return codes.  setConstTable: a per-voice
    // property TABLE, values[p][count] float32 row-major -> `value` of const node nodeIds[p] for voices [voiceBegin, voiceBegin +
    // count): nProps copies straight from the caller's table, no per-value conversion, no JSON.
    int applyBinary(int voiceBegin, int voiceEnd, const void* data, size_t bytes);
    int setConstTable(const int32_t* nodeIds, int nProps, const float* values, int voiceBegin, int count);
    // Per-voice `path` of a convolve or sample node: voice voiceBegin+i convolves with / plays the shared resource names[index[i]] from
    // the next block on, restarting from silence like a [3, nodeId, "path", name] batch on that voice alone — but the voice group is not
    // cut: the group's K3 state holds one IR per channel (convolve.h), a sample node reads its buffer from per-voice parameter rows.
    // Everything is checked before anything changes.
    int setPathPerVoice(int32_t nodeId, const char* const* names, int numNames, const int32_t* index, int voiceBegin, int count);
    // Per-voice `seq` of a seq, seq2, sparseq or sparseq2 node: voice voiceBegin+i gets the JSON value seqs[index[i]] from its next block
    // on, like a [3, nodeId, "seq", seqs[index[i]]] batch on that voice alone — but the voice group is not cut: the node reads each voice's
    // sequence from four per-voice parameter rows.  Each distinct text is parsed and uploaded once.  Everything is checked before
    // anything changes.
    int setSeqPerVoice(int32_t nodeId, const char* const* seqs, int numSeqs, const int32_t* index, int voiceBegin, int count);
    int addSharedResource(const char* name, const float* const* chans, size_t nCh, size_t nSamples);
    void pruneSharedResources();
    std::vector<std::string> listSharedResources() const;
    int gc(int voice, std::vector<int32_t>& pruned);
    // Voices voices[0..count) (runtime-global, any order, repeats allowed) restart as fresh instances from the next block on: state rows
    // at their creation values (rand / once replayed from their shadow rows), their lanes of every tile buffer and their convolver
    // regions zeroed, pending readouts and capture relays dropped.  One K6 launch, stream-ordered; no group is cut, nothing compiled.
    int resetVoices(const int32_t* voices, size_t count);
    // Runtime::reset(): every sample node of every voice sends noteOff to both readers (Sample.h:78-81), stream-ordered.
    void reset();

    // Runtime::process shape: planar host buffers; inputs broadcast to every voice; out = mix bus.
    int process(const float* const* in, size_t nIn, float* const* out, size_t nOut, size_t numSamples, const int64_t* sampleTime = nullptr);
    // Voice-major host buffers: in[voice][nIn][n] (may be null), out[voice][nOut][n] (may be null), mix (may be null).
    int processVoices(const float* in, size_t nIn, float* outVoices, float* mix, size_t nOut, size_t numSamples);
    // Device-resident: no host I/O, no synchronisation; used for throughput timing and by processVoices/process.
    int enqueueBlock(size_t nIn, size_t nOut, size_t numSamples, bool perVoiceIn, bool materialise, bool mix, bool allReduce = false);
    int synchronize();
    // Offline rendering (BASELINE config 5: minutes of audio per graph, nobody listening): numBlocks blocks of every voice, per-voice
    // output, no mix bus, no host round trip per block — blocks are enqueued back to back, the kernels write straight into chunk buffers
    // of `chunkBlocks` blocks ([voice][nOut][chunk] on the device), and finished chunks travel to hostOut[voice][nOut][numBlocks *
    // blockSize] on a copy stream while the next chunk renders.  The reference does the same job with OfflineRenderer.process in a loop.
    int renderOffline(size_t nOut, size_t numBlocks, float* hostOut, size_t chunkBlocks);
    // OfflineRenderer.process(inputs, outputs) (js/packages/offline-renderer/index.ts:87-133): ceil(numSamples / blockSize) full blocks
    // through the same chunk loop, with inputs (shared in[c][numSamples] or per-voice inVoices[voice][nIn][numSamples], zero past
    // numSamples) going up through chunk buffers too, and the mix bus (mixOut[c][numSamples]) and / or per-voice outputs
    // (voicesOut[voice][nOut][numSamples]) coming back, truncated to numSamples.  Block k of the mix is what process() returns for the same
    // block; sampleTime: as process()'s, for the first block (block k gets *sampleTime + k * blockSize).
    int processOffline(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                       size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime);
    // processOffline that also delivers, for block k of the call, cb(k, type, event JSON, user) for every event that
    // processQueuedEvents(vb, ve) would deliver right after the k-th of the equivalent process() calls (ve < 0: all voices).  A K5 launch
    // after each block logs what that poll reads and applies its side effects on the device; the log travels with the chunk's outputs and
    // is replayed through the live poll's formatter after the chunk is scattered, so callbacks lag the render by up to two chunks.
    typedef void (*BlockEventFn)(size_t block, const char* type, const char* json, void* user);
    int processOfflineEvents(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                             size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime, int vb, int ve,
                             BlockEventFn cb, void* user);

    // Cross-GPU mix bus (SURVEY.md §8e): peerExport() allocates this rank's exchange buffer and returns its CUDA IPC handle
    // (64 bytes); peerAttach() maps the buffers of all ranks (handles = world x 64 bytes, in rank order).  Afterwards
    // enqueueBlock(..., allReduce = true) leaves the sum over all ranks in the mix bus of every rank (K4, kernels.h).
    int peerExport(void* handleOut64);
    int peerAttach(int rank, int world, const void* handles);
    int peerStatus();   // 0 = ok, 1 = a peer did not answer within the spin bound
    int setOption(const char* key, double value);
    // Runtime::registerNodeType (Runtime.h:105-106,480-487) for a fused-kernel engine: a new node type is DEVICE code — the body of
    //   float node(float* s /* numState persistent floats per voice, zero-initialised */, const float* in /* numInputs samples */, float sr)
    // as CUDA C++ text, evaluated once per sample.  It is compiled (NVRTC) into the kernel specialised for every render program that
    // uses the type; numState = 0 makes it element-wise (all lanes), otherwise it runs in the lane that owns the voice.  Returns
    // NodeTypeAlreadyExists (4) for a builtin or already registered name, like the reference.
    int registerNodeType(const char* type, int numInputs, int numState, const char* body);
    bool hasNodeType(const char* type) const;
    void setStream(cudaStream_t s);
    float* mixDevicePtr() { return dMix_; }
    float* voiceOutDevicePtr() { return dOutVoice_; }
    float* voiceInDevicePtr(size_t nIn);
    float* sharedInDevicePtr(size_t nIn);
    std::string lastError() const { Lock lk(mu_); return lastError_; }
    int numVoices() const { return numVoices_; }
    int blockSize() const { return blockSize_; }
    uint64_t kernelLaunches() const { Lock lk(mu_); return launches_; }
    uint64_t resetBytesWritten() const { Lock lk(mu_); return resetBytes_; }
    // The int64 sample clock handed to nodes through BlockContext::userData (wasm/Main.cpp:206-217, Metro.h:44,
    // SampleTime.h:19).  process() takes it from *userData when given; otherwise the engine counts samples itself.
    // Runtime::processQueuedEvents (Runtime.h:64,438-446): events of the voices [vb, ve); cb(type, event JSON, voice).
    typedef void (*EventFn)(const char* type, const char* json, int voice, void* user);
    int processQueuedEvents(int vb, int ve, EventFn cb, void* user);
    // The poll of one meter / snapshot node over voices [vb, vb + count) into arrays (events_host.cpp): a / b / fresh[i] for voice vb + i,
    // a and b written only where fresh[i] = 1 (meter: min / max; snapshot: the value, b unused; b may be null).  The side effects and the
    // rules of processQueuedEvents for that node and those voices.  device: the arrays are device memory and the work is only enqueued;
    // otherwise the stream is synchronised and the arrays are host memory.  Everything is checked before anything changes.
    int pollReadouts(int32_t nodeId, int vb, int count, float* a, float* b, uint8_t* fresh, bool device);
    // processOffline that also reads, after every block k, what pollReadouts(nodeIds[j], vb, count, ...) would read there, in node order:
    // host arrays a / b / fresh [numNodes][numBlocks][count].  Event nodes not listed are not polled.
    int processOfflineReadouts(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                               size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime,
                               const int32_t* nodeIds, int numNodes, int vb, int count, float* a, float* b, uint8_t* fresh);
    // The registered type name of node `nodeId` in the voice group containing `voice` ("" when there is none).
    std::string nodeType(int voice, int32_t nodeId) const;
    void setCurrentTime(int64_t t) { Lock lk(mu_); sampleTime_ = t; }
    int64_t currentTime() const { Lock lk(mu_); return sampleTime_; }
    // Sum of the device durations (ms) of the K1 render kernels launched since the last call, measured with
    // CUDA events recorded on the launching stream (option "time_kernels" = 1). Synchronises the stream.
    double takeKernelTimeMs(uint64_t* count);
    // K3 time/count gathered by the same takeKernelTimeMs() call
    double lastConvolveTimeMs(uint64_t* count) const { Lock lk(mu_); if (count) *count = lastKindCount_[2]; return lastKindMs_[2]; }
    // per kernel kind (0 = K1 render, 1 = K2 mix reduce, 2 = K3 convolve, 3 = K4 mix exchange): summed ms and launch counts of the same call
    void lastKernelTimes(double ms[4], uint64_t counts[4]) const { Lock lk(mu_); for (int i = 0; i < 4; ++i) { ms[i] = lastKindMs_[i]; counts[i] = lastKindCount_[i]; } }
    // A cross-GPU barrier on the render stream (K4 with an empty payload): returns once every rank's stream has reached it.
    int peerBarrier();
    std::string describe() const;
    // Runtime::snapshot() (Runtime.h:110,490-499): {"0x<node id, 8 hex digits>": {props...}, ...} of the voice group containing `voice`
    // (per-voice capable props report the value last set for the group's highest addressed voice, like any other prop the last write).
    std::string snapshot(int voice) const;
    // The encoded render program (program.h) of the voice group containing `voice` — the newest compiled one.  Introspection:
    // tests, and the input of per-program kernel specialisation (DESIGN.md §8).
    std::vector<uint32_t> programWords(int voice) const;
    // Compile (not load, not run) the specialised K1 of the voice group containing `voice`: returns the cubin size or -1, the
    // NVRTC log in `log`.  Works without a GPU (NVRTC is a pure compiler): the CPU test-suite uses it.
    long specializeDryRun(int voice, std::string& log);
    // Adds the per-opcode counters of the loaded specialised kernels compiled with option spec_opprof (each kernel once) to out128.
    bool specOpprofRead(unsigned long long* out128, bool reset);

private:
    // Threading contract of the boundary (Runtime.h:133,204,277-285: one control thread + one render thread, concurrently): every
    // public entry point takes this lock for its host-side work.  process()/processVoices() hold it only while they ENQUEUE the block
    // (tens of microseconds) and wait for the GPU without it, so the control thread works while a block renders; a control call
    // holds it while it mutates the node table / compiles (NVRTC never runs under it in "specialize" = 1 mode).  Recursive because
    // public methods call each other.
    mutable std::recursive_mutex mu_;
    typedef std::lock_guard<std::recursive_mutex> Lock;
    bool planDryRun_ = false;     // plan-only engines: enqueueBlock runs ALL its host logic and skips only the CUDA calls (thread-safety tests)
    double sr_;
    int blockSize_, numVoices_, device_;
    int smCount_ = 132;           // SMs of the device (queried; plan-only engines assume an H100 SXM)
    cudaStream_t stream_ = nullptr;
    bool ownStream_ = true;
    EngineOptions opt_;
    std::vector<std::unique_ptr<Group>> groups_;
    std::map<std::string, std::shared_ptr<Resource>> resources_;
    IrBank irBank_;                       // convolver IR spectra, one set per resource however many channels use it
    struct CustomType { std::string name, body; int nIn = 0, nState = 0; };
    std::vector<CustomType> customTypes_;
    std::string customSource() const;     // the generated device text of all registered types (part of the specialisation key)
    std::string lastError_;
    uint64_t launches_ = 0;
    int64_t sampleTime_ = 0;
    bool timeKernels_ = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timed_[4], eventPool_;   // timed_[kind]: K1, K2, K3, K4 pairs since takeKernelTimeMs()
    double lastKindMs_[4] = {0, 0, 0, 0}; uint64_t lastKindCount_[4] = {0, 0, 0, 0};   // K1, K2, K3, K4 of the latest takeKernelTimeMs()
    std::pair<cudaEvent_t, cudaEvent_t> timedBegin();
    void timedEnd(std::pair<cudaEvent_t, cudaEvent_t> ev, int kind);

    // I/O staging
    float* dMix_ = nullptr;          // [max(MAX_OUT, widest nOut so far)][blockSize]
    float* dMixScratch_ = nullptr;   // K2 group sums [MIX_REDUCE_MAX_GROUPS][MAX_OUT][blockSize]
    unsigned int* dMixTickets_ = nullptr;
    float* dPartial_ = nullptr; size_t partialFloats_ = 0;
    float* dOutVoice_ = nullptr; size_t outVoiceFloats_ = 0;
    float* dInVoice_ = nullptr; size_t inVoiceFloats_ = 0;
    float* dInShared_ = nullptr; size_t inSharedFloats_ = 0;
    float* hPinned_ = nullptr; size_t pinnedFloats_ = 0;
    // Host delivery of the mix bus (kernels.h HostDeliver): mapped pinned [mixFloats_] floats + the sequence word behind them.
    // process() arms it for the block it enqueues and polls the word instead of D2H copy + stream synchronize.
    float* hMixHost_ = nullptr; float* dMixHostAlias_ = nullptr;
    volatile uint32_t* hMixFlag_ = nullptr; uint32_t* dMixFlagAlias_ = nullptr;
    unsigned int* dDeliverDone_ = nullptr;
    uint32_t deliverSeq_ = 0;
    bool hostDeliver_ = true, processAllReduce_ = true;   // options "host_deliver", "process_allreduce"
    bool deliverArmed_ = false, deliverLaunched_ = false;
    HostDeliver takeDeliver();
    void allocMixHost();
    // Offline chunk buffers, kept across calls: two on the device (rendered into / uploaded to back to back), two pinned on the host
    struct OfflineBuf { float* dev[2] = {nullptr, nullptr}; float* pinned[2] = {nullptr, nullptr}; size_t devFloats[2] = {0, 0}, pinnedFloats[2] = {0, 0}; };
    OfflineBuf offOut_, offIn_, offMix_;  // per-voice outputs [voice][nOut][C * bs], inputs [nIn][C * bs] or [voice][nIn][C * bs], mix [nOut][C * bs]
    OfflineBuf offLog_;                   // event log of the chunk's blocks, packed (EventLog)

    // A poll (processQueuedEvents) in two halves.  planPoll walks the polled event nodes and takes the decisions that are the same for every
    // voice of a group — whether a scope / fft window is read and where, the metro flag — advancing the host mirrors; emitPoll reads what
    // the item needs from a PollSource (the device now, or a block's logged record) and turns it into events, with the capture relays.
    struct PollItem {
        Group* g = nullptr; Node* n = nullptr;
        int b = 0, e = 0;                 // group-relative voices
        bool fire = false;                // scope / fft: a window is read; metro: the flag was up
        uint32_t r = 0, size = 0;         // scope / fft: read position, window length
        int nch = 0;                      // scope / fft: ring channels read
        size_t logOff = 0;                // offline: the item's record in the chunk's event log (words)
    };
    struct PollSource;
    struct DeviceSource;
    struct LogSource;
    template <class F> int forEachPolled(int vb, int ve, bool queued, F&& f);
    int planPoll(int vb, int ve, std::vector<PollItem>& items);
    int emitPoll(const PollItem& it, PollSource& src, EventFn cb, void* user);
    size_t pollRecordWords(const PollItem& it) const;   // the item's record in the event log
    int captureConsumed(const PollItem& it, bool clearReady);
    // The per-block event log of an offline render: the plans of the blocks of the two chunks in flight and their records' extent.
    struct EventLog {
        int vb = 0, ve = 0;
        BlockEventFn cb = nullptr; void* user = nullptr;
        size_t blockWords = 0;            // bound on one block's records
        std::vector<std::vector<PollItem>> blocks[2];
        size_t used[2] = {0, 0};
    };
    // Array polls (pollReadouts, processOfflineReadouts).  A node's record holds [count] words of a, [count] of b, then count fresh bytes.
    int readoutTargets(int32_t nodeId, int vb, int count, std::vector<VoiceTarget>& out);   // the checks of one node (graph_host.cpp)
    static size_t readoutWords(int count) { return 2 * (size_t) count + ((size_t) count + 3) / 4; }
    typedef std::set<std::pair<const Group*, int32_t>> PolledSet;   // (group, node) pairs a poll reaches
    int readoutPolled(int vb, int ve, PolledSet& out);
    // K5 items of one node's poll into device arrays a, b (null: not written), fresh; appended to `batch`, launched when full.  A group
    // whose (group, node) pair is not in `polled` reports nothing and keeps its queue.
    int readoutEnqueue(int32_t nodeId, const std::vector<VoiceTarget>& targets, const PolledSet& polled, uint32_t* a, uint32_t* b,
                       uint8_t* fresh, EventLogBatch& batch);
    int flushEventLog(EventLogBatch& batch);
    struct ReadoutLog {
        std::vector<int32_t> nodes;
        std::vector<std::vector<VoiceTarget>> targets;
        int vb = 0, count = 0;
        float* a = nullptr; float* b = nullptr; uint8_t* fresh = nullptr;
        size_t numBlocks = 0;
        PolledSet polled;                 // the walk of the latest block
        size_t blockWords() const { return nodes.size() * readoutWords(count); }
    };
    int readoutBlock(ReadoutLog& ro, int slot, size_t inChunk);
    void readoutScatter(const ReadoutLog& ro, const uint32_t* rec, size_t block);   // one block's records into the caller's arrays
    uint32_t* dReadout_ = nullptr; size_t readoutCap_ = 0;      // pollReadouts in host mode: the device staging buffer (words)
    uint32_t* hReadout_ = nullptr; size_t readoutPinned_ = 0;   // and its pinned host copy
    int offlineArgs(const float* const* in, size_t nIn, const float* inVoices, float* voicesOut, size_t nOut);
    int eventLogBegin(EventLog& log);
    int eventLogBlock(EventLog& log, int slot, size_t inChunk);
    int eventLogReplay(EventLog& log, int slot, size_t firstBlock);
    int offlineLoop(const float* const* in, size_t nIn, const float* inVoices, float* const* mixOut, float* voicesOut,
                    size_t nOut, size_t numSamples, size_t chunkBlocks, const int64_t* sampleTime, EventLog* log = nullptr,
                    ReadoutLog* ro = nullptr);
    // Where a block's I/O lives: rows of `pitch` floats, the block in column `col` of each.  Device-resident calls pass the engine's own
    // buffers (pitch blockSize, column 0), offline blocks their chunk slots.
    struct BlockIO {
        size_t nIn = 0, nOut = 0, numSamples = 0;
        bool perVoiceIn = false, allReduce = false;
        const float* in = nullptr; int inPitch = 0;    // [nIn] or [voice][nIn] rows (null without inputs)
        float* voiceOut = nullptr; int outPitch = 0;   // [voice][nOut] rows; null: per-voice outputs are not materialised
        float* mix = nullptr; int mixPitch = 0;        // [nOut] rows; null: no mix
        int col = 0;
        // The steady-state key: the cached descriptors hold the input and output base pointers and pitches; the column and the mix rows
        // are kernel arguments of every block (K1's many-groups launches, K2, K2w), so they may differ.
        bool sameSteadyKey(const BlockIO& o) const {
            return nIn == o.nIn && nOut == o.nOut && numSamples == o.numSamples && perVoiceIn == o.perVoiceIn && allReduce == o.allReduce &&
                   in == o.in && inPitch == o.inPitch && voiceOut == o.voiceOut && outPitch == o.outPitch && !mix == !o.mix;
        }
    };
    int enqueueBlock(const BlockIO& io);
    int walkGroups(const BlockIO& io);
    struct BatchBuffers { LaunchParams* dDescs = nullptr; int* dTileStart = nullptr; size_t capDescs = 0, capTiles = 0; std::vector<char> lastDescs; };
    std::map<int, BatchBuffers> batch_;   // per tile width
    // Steady-state fast path for engines made of many batched voice groups (BASELINE config 5: 1250 graphs): when the last block found
    // every group steady — no queued program, nothing dirty, all root fades settled, no event mirrors to advance — and the call has the
    // same shape, the next block re-launches the cached buckets (the descriptors on the device are still right; the sample clock is a
    // kernel argument) without walking the groups.  Any instruction batch, gc, option or resource change invalidates it.
    struct SteadyBucket { int L, nGroups, totalTiles, maxSlots, maxState, maxParams, wpc, pipeStages, key, smemOut; };
    static constexpr int PIPE_BUCKET = 1000;   // bucket key = tile width (+ PIPE_BUCKET for pipelined one-voice programs)
    std::vector<SteadyBucket> steadyBuckets_;
    bool steadyValid_ = false;
    BlockIO steadyIO_;
    int steadyTiles_ = 0;                 // tiles of the last walk: K2's partial rows
    // Wide mix bus (nOut > MAX_OUT_CHANNELS, DESIGN.md section 3): each voice group writes compact partial rows for the channels its
    // roots aim at only (mix channels, ascending), per-voice outputs go to a compact [voice][mix channel] buffer and are scattered to
    // [voice][nOut]; K2w reduces each channel over its own row list.  Rebuilt by every slow pass; the device copies are re-uploaded
    // only when they change, so the steady-state fast path relaunches K2w on them as they stand.
    struct WidePlan {
        std::vector<int> rows;            // CSR row lists of the channels, concatenated in channel order
        std::vector<WideSeg> segs;        // K2w segments
        std::vector<int> dstRow;          // compact per-voice output row -> row of [voice][nOut]
        int nScratch = 0;                 // scratch / ticket rows of the channels with more than one tile group
        int* dRows = nullptr; size_t capRows = 0;
        WideSeg* dSegs = nullptr; size_t capSegs = 0;
        int* dDst = nullptr; size_t capDst = 0;
        std::vector<int> upRows, upDst; std::vector<char> upSegs;   // what the device copies hold
        int nSmall = 0;                   // segs[0, nSmall) have fewer than WIDE_BIG_ROWS rows
        // the per-voice output buffer is zero outside outZeroRows (rows of [voice][outZeroNOut]) since its last clear
        bool outZeroValid = false; size_t outZeroNOut = 0; std::vector<int> outZeroRows;
    } wide_;
    float* dWideScratch_ = nullptr; unsigned int* dWideTickets_ = nullptr; size_t wideScratchFloats_ = 0, wideTicketCount_ = 0;
    float* dOutCompact_ = nullptr; size_t outCompactFloats_ = 0;
    size_t mixFloats_ = 0;                // dMix_ and the mapped host-delivery buffer hold this many floats
    int uploadWidePlan();
    int launchWide(const BlockIO& io);
    // the mix channels of a program: distinct channels in [0, nOut) of all its roots, running or fading, ascending
    std::vector<int> mixChannels(const Group& g, const Program& p, size_t nOut) const;

    // K6 (resetVoices): the reset plans of the groups a call touches, as last uploaded, and the call's voice list and runs
    std::vector<char> resetPlanUp_;
    char* dResetPlan_ = nullptr; size_t resetPlanCap_ = 0;
    int* dResetCall_ = nullptr; size_t resetCallCap_ = 0;
    uint64_t resetBytes_ = 0;            // bytes the reset launches wrote so far (from the plans)

    // K4 state
    void* dExchange_ = nullptr; size_t exchangeBytes_ = 0; size_t exchangeFlagOffset_ = 0, exchangeOwnOffset_ = 0;
    PeerMix peer_{}; bool peerAttached_ = false; uint32_t peerEpoch_ = 0; int* dPeerStatus_ = nullptr;
    std::vector<void*> peerMapped_;

    bool planOnly_ = false;
    bool cuda(cudaError_t e, const char* what);
    cudaError_t dmalloc(void** p, size_t bytes);
    void dfree(void* p);
    cudaError_t dmemset(void* p, int v, size_t bytes);
    cudaError_t dmemcpy(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind);
    cudaError_t dmemcpySync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind);
    cudaError_t dzeroBlock(float* p, int pitch, size_t rows);   // the first blockSize floats of `rows` rows of `pitch` floats
    // Grow a device allocation (pinned: page-locked host memory) holding cap elements to at least n, allocating n * slack: drains the
    // stream, drops the old contents, zeroes the new memory on request.  false (p null, cap 0) when the allocation fails.
    template <typename T> bool grow(T*& p, size_t& cap, size_t n, const char* what, bool zero = false, size_t slack = 1, bool pinned = false);
    void dsync();
    void dsetdev();
    int fail(int code, const std::string& msg) { lastError_ = msg; return code; }

    // instruction interpreter (Runtime.h:170-433)
    int applyToGroup(Group& g, const std::vector<Value>& batch, int vb, int ve);
    int applyBatch(int vb, int ve, const std::vector<Value>& batch);
    int createNode(Group& g, const Value& id, const Value& type);
    int appendChild(Group& g, const Value& parent, const Value& child, const Value& chan);
    int setProperty(Group& g, const Value& id, const Value& key, const Value& val, int vb, int ve);
    template <class KindOk> int voiceTargets(int32_t nodeId, int vb, int count, KindOk kindOk, const char* kindError, std::vector<VoiceTarget>& out);
    int activateRoots(Group& g, const Value& roots);
    int nodeSetProperty(Group& g, Node& n, const std::string& key, const Value& val, int vb, int ve);
    bool isValueOnlyBatch(const std::vector<Value>& batch, int vb, int ve);
    int splitGroupsAt(int v);
    // 8192 <= voices < 131072 with specialised kernels: twice the warps (about 4096) from narrow-geometry kernels compiled for 8 CTAs per
    // SM (64 registers) — on an H100 6-9 % faster than ~2048 warps at 110 registers (16 384 and 65 536 voices)
    bool midRangeDense(int nv) const { return opt_.specialize > 0 && !opt_.targetTilesSet && opt_.tileWidth == 0 && opt_.specMinBlocks == 0 && nv >= 8192; }

    // storage
    int allocRows(Group& g, int count, bool evenAlign, int& row);
    int fillRow(Group& g, int row, int vb, int ve, float value);
    int fillRowBits(Group& g, int row, int vb, int ve, uint32_t bits);
    int ensureResourceOnDevice(Resource& r);
    int writeColumns(Group& g, int row, int rows, int vb, int cnt, const void* words, const char* what);
    int assignVoiceArrays(Group& g, Node& n, const std::vector<VoiceArray>& arrs, const int32_t* index, int vb, int ve, const uint32_t* gen = nullptr);
    int assignSampleBuffers(Group& g, Node& n, const std::vector<std::shared_ptr<Resource>>& res, const int32_t* index, int vb, int ve);
    int uploadArray(std::shared_ptr<DeviceArray>& out, const void* data, size_t bytes, size_t count);
    void retireArrays(std::vector<std::shared_ptr<const void>>&& arrs);
    // arrays no voice reads any more (voiceArrays), each batch released once the stream has passed its event (retireArrays)
    std::deque<std::pair<cudaEvent_t, std::vector<std::shared_ptr<const void>>>> retiredArrays_;

    // compile (Runtime.h:521-577 + GraphRenderSequence.h:107-187)
    int compile(Group& g, int nIn, std::shared_ptr<Program>& out);
    void traverse(Group& g, std::set<int32_t>& visited, std::vector<int32_t>& order, int32_t n);
    int chooseTileWidth(int nv) const;
    friend struct Compiler;
};

} // namespace eb
