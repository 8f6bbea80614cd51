/* elem_b200.h — C ABI of the H100-native Elementary render engine (libelem_b200.so).
 *
 * Drop-in boundary for ONE path of elemaudio/elementary: elem::Runtime<float> — applyInstructions() /
 * process() / gc() / shared resources — with the per-block graph walk executed by a fused sm_90a kernel for
 * thousands of independent voices (graph instances) at once.  Every entry point below replaces the method of
 * the reference class cited next to it (paths relative to the reference tree); the embind surface of
 * wasm/Main.cpp:374-390 was the model.  Plain pointers and sizes only; the library owns all device memory and
 * nothing device-side crosses this ABI except where a function says "device pointer".
 *
 * Conventions
 *   - return value: 0 = Ok, 1..8 = elem::ReturnCode (runtime/elem/Types.h:51-60), negative = engine failure
 *     (-1 CUDA error, -2 bad argument); elem_b200_last_error() gives the text.
 *   - exceptions never cross the ABI: malformed JSON, which makes the reference throw (runtime/elem/JSON.h:
 *     146-154, Value.h:89-92), returns 8 (InvalidInstructionFormat).
 *   - threading: one control thread for everything except elem_b200_process*, which may run on one other
 *     thread — the same contract as the reference (Runtime.h:329-332).
 *   - audio buffers are planar, non-interleaved float32, borrowed for the duration of the call;
 *     numSamples <= blockSize (Runtime.h:51-57).
 *   - a "voice" is one independent instance of the reference Runtime: its own node table, state and outputs.
 *     There is NO CPU fallback: without a CUDA device elem_b200_create returns NULL.
 */
#ifndef ELEM_B200_H
#define ELEM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct elem_b200_runtime elem_b200_runtime;

/* Output channels of elem_b200_process / _process_voices / _enqueue_block / _process_offline (the mix bus past 8 channels is compact, see process). */
#define ELEM_B200_MAX_OUT_CHANNELS 4096

/* Runtime<float>::Runtime(double sampleRate, int blockSize)  — runtime/elem/Runtime.h:44,158-166.
 * New here: numVoices independent instances living on CUDA device `device`. */
elem_b200_runtime* elem_b200_create(double sampleRate, int blockSize, int numVoices, int device);
void elem_b200_destroy(elem_b200_runtime* rt);

/* Runtime::applyInstructions(js::Array const&) — Runtime.h:48,170-218 — fed with the JSON text the JS
 * reconciler emits (cli/Benchmark.cpp:40-43 does parseJSON + applyInstructions).  The batch is applied to
 * every voice in [voiceBegin, voiceEnd) (voiceEnd < 0 = all).  A batch consisting only of SET_PROPERTY on
 * per-voice capable props (const.value, rand.seed) may address any sub-range. */
int elem_b200_apply_instructions(elem_b200_runtime* rt, int voiceBegin, int voiceEnd, const char* json, size_t len);

/* Instruction-stream ingestion at scale (what runtime/elem/JSON.h:17-156 costs when there are a million voices).
 * BINARY BATCH FORMAT — the same instruction stream (core/index.ts:43-49, Runtime.h:115-121), same semantics, same return codes:
 *   little-endian, unaligned:  u32 magic 'EB2I' (0x49324245)  u32 version = 1  u32 numInstructions, then per instruction  u8 opcode:
 *     0 CREATE_NODE     i32 id, u16 len, type bytes
 *     2 APPEND_CHILD    i32 parent, i32 child, i32 childOutputChannel
 *     3 SET_PROPERTY    i32 id, u16 len, key bytes, u8 valueType: 0 null | 1 bool (u8) | 2 number (f64) | 3 string (u32 len, bytes)
 *                                                         | 4 float array (u32 n, f32[n]) | 5 any other value as JSON text (u32 len, bytes)
 *     4 ACTIVATE_ROOTS  u32 n, i32 ids[n]
 *     5 COMMIT_UPDATES
 * elementary_b200.el.encode_binary() writes it from the list form. */
int elem_b200_apply_binary(elem_b200_runtime* rt, int voiceBegin, int voiceEnd, const void* data, size_t bytes);

/* Per-voice property TABLE: values[p][i] (float32, row-major, numProps rows of `count`) -> the `value` prop of const node nodeIds[p]
 * for voice voiceBegin+i.  One device copy per row straight from the caller's table: a million voices x a dozen per-voice constants
 * are a dozen copies, not a dozen million JSON numbers.  Equivalent to the [[3,nodeIds[p],"value",values[p][i]]] batches.
 * Returns -2 for a voice range out of bounds or a negative numProps, NodeNotFound (2) when a voice group in the range lacks one of
 * the nodes, InvalidPropertyType (5) when one is not a const.  All of it is checked before anything changes: a failed call changes
 * nothing. */
int elem_b200_set_const_table(elem_b200_runtime* rt, const int32_t* nodeIds, int numProps, const float* values, int voiceBegin, int count);

/* Vectorised SET_PROPERTY: values[i] -> voice voiceBegin+i; equivalent to `count` single-voice
 * [[3,nodeId,key,values[i]]] batches (Runtime.h:316-333) without `count` JSON parses.  Per-voice capable: const `value`,
 * rand `seed`, sample `startOffset` and `stopOffset`; any other node or key returns InvalidPropertyType (5), a sample offset
 * whose (int) is negative InvalidPropertyValue (6).  All of it is checked before anything changes: a failed call changes nothing. */
int elem_b200_set_property_per_voice(elem_b200_runtime* rt, int32_t nodeId, const char* key,
                                     const double* values, int voiceBegin, int count);

/* Per-voice impulse response of a `convolve` node (ConvolutionNode::setProperty("path"), wasm/Convolve.h:34-56), or per-voice
 * buffer of a `sample` node (SampleNode::setProperty("path"), Sample.h:27-36).
 * voice voiceBegin+i gets the `path` names[index[i]]; same result as `count` single-voice
 * [[3, nodeId, "path", names[index[i]]]] batches, except that no voice group is cut.
 * A names table plus a per-voice index, like elem_b200_set_const_table: a million voices choose among K IRs without a million strings.
 * Each addressed voice restarts from silence at the next process/enqueue_block, even on an unchanged name: a fresh convolver, or
 * fresh sample readers (currentReader and the trigger's last value are kept); the other voices are untouched.  Each resource's
 * partition spectra are computed once, however many voices use it; a resource any sample voice plays stays alive across
 * elem_b200_prune_shared_resources.
 * Returns -2 for a voice range out of bounds or an index outside [0, numNames), NodeNotFound (2) when a voice group in the range
 * lacks the node, InvalidPropertyType (5) when the node is neither a convolve nor a sample, InvalidPropertyValue (6) when a name is not a shared
 * resource.  All of it is checked before anything changes: a failed call changes nothing. */
int elem_b200_set_path_per_voice(elem_b200_runtime* rt, int32_t nodeId, const char* const* names, int numNames,
                                 const int32_t* index, int voiceBegin, int count);

/* Per-voice sequence of a `seq`, `seq2`, `sparseq` or `sparseq2` node (their setProperty("seq"), Core.h:447-466, Seq2.h:60-84,
 * SparSeq.h:102-124, SparSeq2.h:39-56).  seqs[k] is the JSON text of one `seq` value, as [3, nodeId, "seq", value] carries it; voice
 * voiceBegin+i gets seqs[index[i]].  Same result as `count` single-voice [[3, nodeId, "seq", seqs[index[i]]]] batches, except that no
 * voice group is cut: the node reads each voice's sequence from per-voice parameter rows.  Each addressed voice takes its sequence at
 * its next block as its own Runtime would, even an unchanged one (seq: index wrapped and hold value reloaded; sparseq: hold index
 * re-found; sparseq2: previous / next event reset); the other voices are untouched.  Each distinct seqs[k] is parsed and uploaded once,
 * however many voices use it.  A later whole-group [3, nodeId, "seq", v] gives every voice of the group v; voice resets keep a voice's
 * sequence; snapshot() reports the value set for the group's highest addressed voice.
 * Returns -2 for a voice range out of bounds or an index outside [0, numSeqs), NodeNotFound (2) when a voice group in the range lacks
 * the node, InvalidPropertyType (5) when the node is not one of the four, and for a seqs[k] what [3, nodeId, "seq", seqs[k]] returns
 * on that node (5 for a non-array, 8 for a malformed entry), 8 for text that is not JSON.  All of it is checked before anything
 * changes: a failed call changes nothing. */
int elem_b200_set_seq_per_voice(elem_b200_runtime* rt, int32_t nodeId, const char* const* seqs, int numSeqs,
                                const int32_t* index, int voiceBegin, int count);

/* Voices voices[0..count) restart as fresh instances: each renders from its next block on what a Runtime newly
 * created and given this runtime's instruction history would render. Props are replayed as last set for that voice.
 * Stream-ordered: applied between the previous and the next block, with no host synchronisation. No voice group is
 * cut, nothing is recompiled, and snapshot() and the groups and programs in describe() do not change.
 * Indices are runtime-global and may be unsorted or repeated; one outside [0, numVoices) returns -2 and nothing changes;
 * count == 0 launches nothing.  Call it from the control thread, like elem_b200_set_property_per_voice.
 * Shared by a voice group, so not restarted: root fades, the scope / fft window positions, the metro flag, the sample clock and
 * the convolver's partition phase — a reset voice's convolver is a fresh one fed zeros since the last 512-sample partition
 * boundary, as after elem_b200_set_path_per_voice.  No reference method: the equivalent of constructing a new Runtime for
 * that voice. */
int elem_b200_reset_voices(elem_b200_runtime* rt, const int32_t* voices, size_t count);
/* Bytes the voice resets of this runtime have written so far, counted from their plans (state cells, buffer lanes, convolver
 * regions). */
uint64_t elem_b200_reset_bytes_written(elem_b200_runtime* rt);

/* Runtime::process(in, nIn, out, nOut, numSamples, userData) — Runtime.h:51-57,275-290.
 * `in` channels are broadcast to every voice; out[c] receives the MIX BUS: the sum over all voices of what
 * each voice's Runtime would have written to its out[c].  Host buffers; the H2D copy of the inputs and the hand-over of the
 * result (stored into mapped host memory by the kernel that finishes the mix bus; the call returns when its sequence word
 * arrives) are inside the call.  With peers attached (elem_b200_peer_attach) the sum runs over the voices of ALL ranks and every
 * rank must make the call for every block.
 * userData: NULL, or — as every reference host passes it (wasm/Main.cpp:206-215) — a pointer to the int64 sample
 * time of the block's first sample, read by the `time` and `metro` nodes (wasm/SampleTime.h:19, Metro.h:44).
 * With NULL the engine keeps the clock itself (+= numSamples per call, like wasm/Main.cpp:217).
 * OUTPUT CHANNELS: nOut <= 4096 (ELEM_B200_MAX_OUT_CHANNELS); more returns -2.  A root aimed outside [0, nOut) does not run and its
 * nodes keep their state, as in the reference.  Up to 8 channels the mix is K2's fixed summation tree over all tiles (DESIGN.md §4).
 * Past 8 the mix bus is compact: each voice group writes partial rows only for the channels its roots aim at, and channel c is K2's
 * tree over its own rows — the groups that write c in engine order, their tiles in order (K2w, DESIGN.md §3-4); still deterministic
 * run to run.  Past 8 channels peers may not be attached with the cross-GPU sum requested (-2). */
int elem_b200_process(elem_b200_runtime* rt, const float* const* in, size_t nIn,
                      float* const* out, size_t nOut, size_t numSamples, void* userData);

/* ElementaryAudioProcessor::setCurrentTime — wasm/Main.cpp:232-241: (re)set the engine-kept sample clock. */
void elem_b200_set_current_time(elem_b200_runtime* rt, int64_t sampleTime);
int64_t elem_b200_current_time(elem_b200_runtime* rt);

/* Voice-major variant for per-voice I/O and parity tests: in = [voice][nIn][numSamples] or NULL,
 * outVoices = [voice][nOut][numSamples] or NULL, mix = [nOut][numSamples] or NULL (all host memory).
 * nOut <= 4096 with the mix order of elem_b200_process; past 8 channels a voice's channels that none of its roots aim at are zero. */
int elem_b200_process_voices(elem_b200_runtime* rt, const float* in, size_t nIn,
                             float* outVoices, float* mix, size_t nOut, size_t numSamples);

/* Offline rendering (what js/packages/offline-renderer does with process() in a loop; BASELINE config 5): numBlocks full blocks of every
 * voice, per-voice output hostOut[voice][nOut][numBlocks * blockSize] (host memory, nOut <= 8), no inputs, no mix bus.  Blocks are enqueued back to
 * back with no host synchronisation in between; outputs are written by the kernels into device chunk buffers of chunkBlocks blocks
 * (0 = default 8; fewer when a chunk buffer would pass 256 MiB) and copied out on a second stream while the next chunk renders. */
int elem_b200_render_offline(elem_b200_runtime* rt, size_t nOut, size_t numBlocks, float* hostOut, size_t chunkBlocks);

/* OfflineRenderer.process(inputs, outputs) — js/packages/offline-renderer/index.ts:87-133: render a whole signal in one call, with inputs,
 * through the chunk loop of elem_b200_render_offline (no host round trip per block).  All buffers are host memory.
 *   in         nIn planar channels of numSamples, broadcast to every voice (as elem_b200_process), or NULL;
 *   inVoices   per-voice inputs [voice][nIn][numSamples] (as elem_b200_process_voices), or NULL — not both with `in`;
 *   mixOut     nOut planar channels of numSamples: the MIX BUS, or NULL;
 *   voicesOut  per-voice outputs [voice][nOut][numSamples], or NULL.
 * BLOCKS: ceil(numSamples / blockSize) FULL blocks, like the reference's offline renderer; input samples past numSamples are zero and the
 *   outputs are truncated to numSamples.  A second call continues at the next block boundary.  numSamples == 0 renders nothing.
 * BITS: block k of the mix is, bit for bit, what elem_b200_process returns for the same zero-padded block of inputs (the same summation
 *   tree: K2 up to 8 channels, K2w past 8); per-voice outputs are those of elem_b200_process_voices.
 * OUTPUT CHANNELS: the mix takes nOut <= 4096 (ELEM_B200_MAX_OUT_CHANNELS) with the channel rules of elem_b200_process (a channel no
 *   running root aims at is +0.0); per-voice outputs nOut <= 8.  With voicesOut == NULL nothing per-voice is materialised or copied.
 * SAMPLE CLOCK: userData NULL lets the engine clock run on; a pointer to an int64 t0 gives block k the time t0 + k * blockSize, as if
 *   elem_b200_process had been called with that userData for each block.
 * EVENTS are not polled inside the call: afterwards the event queues hold what as many elem_b200_process calls would have left
 *   (elem_b200_process_offline_events delivers them block by block).
 * Blocks go through chunk buffers of chunkBlocks blocks (0 = default 8; fewer when a chunk buffer would pass 256 MiB): chunk k + 1's
 *   inputs are uploaded and chunk k - 1's outputs copied out while chunk k renders.  The engine lock is held for the whole call.
 * Returns -2, before rendering anything, when both `in` and `inVoices` are given, when nIn > 0 comes without an input pointer, when
 *   nOut is 0 or above its limit, and with peers attached while the cross-GPU sum of process() is on ("process_allreduce" = 1): the
 *   offline mix is not summed across GPUs. */
int elem_b200_process_offline(elem_b200_runtime* rt, const float* const* in, size_t nIn, const float* inVoices,
                              float* const* mixOut, float* voicesOut, size_t nOut, size_t numSamples, size_t chunkBlocks, void* userData);

/* elem_b200_process_offline with every block's events, as OfflineRenderer.process does when it polls after each block
 * (js/packages/offline-renderer/index.ts:104-132).  Arguments, blocks, chunks, sample clock, outputs and errors are those of
 * elem_b200_process_offline, and the outputs are bit for bit what it returns: logging events does not change the audio.
 * EVENTS: for block k of this call (0-based), cb(k, type, jsonEvent, user) receives the events, in the same order and with the same text,
 *   that elem_b200_process_queued_events_range(rt, voiceBegin, voiceEnd, ...) would deliver right after the k-th of the equivalent
 *   elem_b200_process calls (voiceEnd < 0: all voices; voiceBegin == voiceEnd: none).  After each block a kernel copies what that poll reads
 *   (meter / snapshot readouts, the capture samples written since the last poll, scope / fft windows when one is due) into an event log that
 *   travels down with the chunk's outputs, and applies the poll's effects on the device (queues drained, capture read positions moved).
 *   The chunk size shrinks so that two logs stay within 256 MiB each, like the other chunk buffers.
 * DELIVERY: in block order, on the calling thread, before the call returns; up to two chunks after the block rendered.  The engine lock is
 *   held throughout, so cb must not call into the runtime.
 * STATE AFTERWARDS: queues, scope / fft read positions, capture relays and the metro flag are what the process() + poll-per-block loop
 *   leaves; voices outside [voiceBegin, voiceEnd) keep what un-polled process() calls leave them, with the group-wide scope / fft / metro
 *   rule of elem_b200_process_queued_events_range.  Capture samples that wait in the ring when the call starts are read into the relay
 *   first (reported with the next relay), so a backlog within one block of the ring's 2^k capacity keeps samples the live poll would lose.
 * Returns -2, before rendering anything, where elem_b200_process_offline does, for cb == NULL, and for a voice range outside
 *   [0, numVoices] or with voiceEnd < voiceBegin. */
typedef void (*elem_b200_block_event_cb)(size_t block, const char* type, const char* jsonEvent, void* user);
int elem_b200_process_offline_events(elem_b200_runtime* rt, const float* const* in, size_t nIn, const float* inVoices,
                                     float* const* mixOut, float* voicesOut, size_t nOut, size_t numSamples,
                                     size_t chunkBlocks, void* userData, int voiceBegin, int voiceEnd,
                                     elem_b200_block_event_cb cb, void* user);

/* elem_b200_process_offline with every block's meter / snapshot readouts as arrays (see elem_b200_poll_readouts) instead of events.
 * Arguments, blocks, chunks, sample clock, outputs and their errors are those of elem_b200_process_offline, and the audio is bit for bit
 * what it returns.
 * READOUTS: a, b, fresh are host arrays [numNodes][numBlocks][count], numBlocks = ceil(numSamples / blockSize).  Entry [j][k][i] is what
 *   elem_b200_poll_readouts(rt, nodeIds[j], voiceBegin, count, ...) would write for voice voiceBegin + i right after the k-th of the
 *   equivalent elem_b200_process calls, the listed nodes polled in the order given: a and b only where fresh is 1; b may be NULL.
 *   After each block a K5 launch writes every listed node's readouts into a record that travels down with the chunk's outputs; the chunk
 *   size shrinks so that two of these logs stay within 256 MiB each.  Event nodes not listed are not polled: their queues end as un-polled
 *   elem_b200_process calls leave them.  The engine lock is held for the whole call.
 * Returns, before rendering anything, what elem_b200_process_offline returns, and -2 for numNodes < 1, a node id listed twice, count < 1,
 *   a NULL `a` or `fresh` or a voice range outside [0, numVoices); NodeNotFound (2) and InvalidPropertyType (5) per node as
 *   elem_b200_poll_readouts returns them.  No reference method: the reference has no voice axis. */
int elem_b200_process_offline_readouts(elem_b200_runtime* rt, const float* const* in, size_t nIn, const float* inVoices,
                                       float* const* mixOut, float* voicesOut, size_t nOut, size_t numSamples,
                                       size_t chunkBlocks, void* userData,
                                       const int32_t* nodeIds, int numNodes, int voiceBegin, int count,
                                       float* a, float* b, uint8_t* fresh);

/* Device-resident stepping for throughput measurement and pipelines that keep audio in HBM: enqueue one block
 * on the engine's stream (no host copies, no synchronisation).  flags: 1 = read per-voice inputs from
 * elem_b200_voice_in_device(), 2 = materialise per-voice outputs, 4 = produce the mix bus, 8 = (with 4, after
 * elem_b200_peer_attach) sum the mix bus over all ranks in place — every rank ends with the mix of the whole voice set (nOut <= 8).
 * nOut <= 4096 with the channel rules and mix order of elem_b200_process. */
int elem_b200_enqueue_block(elem_b200_runtime* rt, size_t nIn, size_t nOut, size_t numSamples, int flags);
int elem_b200_synchronize(elem_b200_runtime* rt);
/* Device pointer [nOut][blockSize] holding the mix of the last enqueued block (at least [8][blockSize]).  The buffer grows the first
 * time a wider nOut is used, so the pointer may MOVE then: fetch it again after a call with a larger nOut than before. */
float* elem_b200_mix_device(elem_b200_runtime* rt);
float* elem_b200_voice_out_device(elem_b200_runtime* rt);              /* device pointer [voice][nOut][blockSize]; may move like the mix */
float* elem_b200_voice_in_device(elem_b200_runtime* rt, size_t nIn);   /* device pointer [voice][nIn][blockSize] */
float* elem_b200_shared_in_device(elem_b200_runtime* rt, size_t nIn);  /* device pointer [nIn][blockSize] */
void elem_b200_set_stream(elem_b200_runtime* rt, void* cudaStream);    /* run on a caller-owned cudaStream_t */

/* The one collective of the path (SURVEY.md §8e, no reference equivalent: the reference has no voice axis): voices are
 * sharded over one process per GPU, and the per-rank mix buses are summed by our own kernel over NVLink/NVSwitch peer
 * memory.  elem_b200_peer_export writes this rank's 64-byte CUDA IPC handle; the caller gathers the handles of all ranks
 * (any transport: torch.distributed.all_gather_object, MPI, a file) and passes them, in rank order, to
 * elem_b200_peer_attach (world <= 8, one box).  elem_b200_peer_status: 0 = ok, 1 = a peer did not answer in time. */
int elem_b200_peer_export(elem_b200_runtime* rt, void* handleOut64);
int elem_b200_peer_attach(elem_b200_runtime* rt, int rank, int world, const void* handles);
int elem_b200_peer_status(elem_b200_runtime* rt);
/* A cross-GPU barrier enqueued on the render stream (the exchange kernel with an empty payload): the stream passes it once the
 * streams of all attached ranks have reached theirs.  Lets a host line the GPUs up before a timed region without a host-side
 * collective.  No-op (0) without attached peers. */
int elem_b200_peer_barrier(elem_b200_runtime* rt);

/* Runtime::addSharedResource(name, unique_ptr<SharedResource>) — Runtime.h:83,462-465;
 * AudioBufferResource copies the samples (AudioBufferResource.h:13-24).  Returns 1 on success, 0 when the
 * name already exists (SharedResource.h:44-46). */
int elem_b200_add_shared_resource(elem_b200_runtime* rt, const char* name,
                                  const float* const* channels, size_t numChannels, size_t numSamples);
/* Runtime::pruneSharedResources() — Runtime.h:89,468-471 */
void elem_b200_prune_shared_resources(elem_b200_runtime* rt);
/* Runtime::getSharedResourceMapKeys() — Runtime.h:94,474-477.  Writes up to `cap` bytes of '\n'-separated
 * names, returns the number of resources. */
int elem_b200_list_shared_resources(elem_b200_runtime* rt, char* buf, size_t cap);

/* Runtime::gc() — Runtime.h:76,221-272.  Collects for the voice group containing `voice`; writes up to `cap`
 * pruned node ids (ascending), returns how many were pruned. */
int elem_b200_gc(elem_b200_runtime* rt, int voice, int32_t* ids, size_t cap);
/* Runtime::reset() — Runtime.h:70,449-458: as in the reference, only `sample` nodes react: both readers of every voice get noteOff
 * (they fade out over 10 ms).  Stream-ordered: applied between the previous and the next block. */
void elem_b200_reset(elem_b200_runtime* rt);
/* Runtime::processQueuedEvents(cb) — Runtime.h:64,438-446; relayed like wasm/Main.cpp:220-231.  For every root
 * sub-sequence whose root is active, every event node in render order (GraphRenderSequence.h:189-198): `meter`
 * {min,max,source}, `snapshot` {source,data}, `scope` {source,data:[[..],..]}, `capture` {source,data:[..]}
 * (runtime/elem/builtins/Analyzers.h, Capture.h), `fft` {source,data:{real,imag}} (wasm/FFT.h:90-131) and `metro` {source}
 * (wasm/Metro.h:58-66).  One callback per voice
 * that has something to report; jsonEvent is the reference's event object as JSON text plus a "voice" key.  Call it
 * from the control thread between blocks (it synchronises the stream). */
typedef void (*elem_b200_event_cb)(const char* type, const char* jsonEvent, void* user);
void elem_b200_process_queued_events(elem_b200_runtime* rt, elem_b200_event_cb cb, void* user);
/* Same, restricted to the voices [voiceBegin, voiceEnd) (voiceEnd < 0 = all): at a million voices nobody wants a
 * million meter callbacks per block.  Per-voice queues (meter, snapshot, capture) of the other voices keep their contents;
 * the ring windows of scope / fft and the metro flag are shared by a voice group (their positions are identical for every
 * voice), so a poll that reaches a group consumes that window for the whole group. */
int elem_b200_process_queued_events_range(elem_b200_runtime* rt, int voiceBegin, int voiceEnd, elem_b200_event_cb cb, void* user);

/* The poll of one `meter` or `snapshot` node over the voices [voiceBegin, voiceBegin + count), into arrays instead of one JSON event per
 * voice; index i is voice voiceBegin + i, across every voice group of the range.
 *   meter     a[i] = min, b[i] = max;   snapshot  a[i] = the latched value, b is never written.  b may be NULL.
 *   fresh[i]  1 exactly when elem_b200_process_queued_events_range over the same voices, called now, would deliver an event of this node
 *             for that voice (the sequence the last process() used, an active root, a queue not pushed a multiple of 32 times since its
 *             last drain); a[i] and b[i] are written only then, as the float32 bits of the readout (a non-finite value too, where the
 *             JSON text has null).
 * Side effects: those of that poll on this node and these voices — the queues under an active root are drained — and nothing else, so
 * a later JSON poll sees nothing from the voices drained here, and the reverse.
 * flags 0: host arrays; the call synchronises the render stream.  ELEM_B200_READOUT_DEVICE: device arrays on the runtime's device; the
 * work is enqueued on the runtime's stream and the call returns without synchronising (order reads after it with elem_b200_synchronize
 * or through elem_b200_set_stream), so a loop of elem_b200_enqueue_block + this call has no host round trip per block.
 * Returns -2 for a voice range out of bounds, count < 0, or a NULL `a` or `fresh` with count > 0; NodeNotFound (2) when a voice group
 * in the range lacks the node; InvalidPropertyType (5) when it is not a meter or snapshot (or a meter in one group and a snapshot in
 * another); 0 and nothing launched for count == 0; -1 on a plan-only runtime.  All of it is checked before anything changes.  A
 * control-thread call, like elem_b200_process_queued_events.  No reference method: the reference has no voice axis. */
#define ELEM_B200_READOUT_DEVICE 1
int elem_b200_poll_readouts(elem_b200_runtime* rt, int32_t nodeId, int voiceBegin, int count,
                            float* a, float* b, uint8_t* fresh, int flags);

/* Tuning and introspection (no reference equivalent).  Keys: "tile_width" (1..32 voices per warp, 0 = auto), "warps_per_cta",
 * "target_tiles", "niter" (sample-tile variant: 4 = 128-sample one-voice tiles), "batch_groups", "fuse_chains",
 * "specialize" (per-program NVRTC kernels: 0 off, 1 compile in the background while the interpreter serves, 2 wait at COMMIT),
 * "specialize_max_words", "specialize_strict", "pipeline_stages" (warp pipeline of one-voice groups, default 4, 0 = off),
 * "fuse_conv_root" (root + mix in the convolver's epilogue, default 1), "host_deliver" (process(): the finishing kernel stores the
 * mix bus into mapped host memory, default 1), "process_allreduce" (process() sums over the attached peers, default 1),
 * "time_kernels" (event pairs around every kernel launch), "plan_dry_run" (plan-only engines).  Geometry options must be set before
 * the first COMMIT of a voice group.  Returns -2 for an unknown key. */
int elem_b200_set_option(elem_b200_runtime* rt, const char* key, double value);
/* Runtime::registerNodeType(type, NodeFactoryFn) — Runtime.h:105-106,480-487 (the plug-in / operator interface of GraphNode.h:20-96).
 * In a fused-kernel engine a new node type is DEVICE code: `cudaBody` is the body of
 *     float node(float* s, const float* in, const float sr)
 * as CUDA C++ text, evaluated once per sample: in[0..numInputs) are this sample's input values (children in order), s[0..numStateFloats)
 * the node's persistent per-voice state (zero-initialised, GraphNode members in the reference), sr the sample rate; the return value is
 * the node's output sample.  numStateFloats = 0 declares the node element-wise.  The body is compiled by NVRTC into the kernel
 * specialised for every render program that uses the type (COMMIT returns 7 with the compiler log in elem_b200_last_error if it does
 * not compile).  Like the reference: 4 (NodeTypeAlreadyExists) for a builtin or already registered name; nodes of the type lacking
 * inputs render zeros; instructions naming an unregistered type return 1.  elem_b200_has_node_type: 1 if `type` is builtin or registered. */
int elem_b200_register_node_type(elem_b200_runtime* rt, const char* type, int numInputs, int numStateFloats, const char* cudaBody);
int elem_b200_has_node_type(elem_b200_runtime* rt, const char* type);

/* Runtime::snapshot() — Runtime.h:110,490-499: the node table of the voice group containing `voice` as JSON text
 * {"0x<node id as 8 hex digits>": {<props>}, ...} (nodeIdToHex, Types.h:16-27; props as they were last set, GraphNode.h:60-64,130).
 * Returns the bytes needed including the terminating NUL; writes at most cap. */
int elem_b200_snapshot(elem_b200_runtime* rt, int voice, char* buf, size_t cap);
/* The type name of node `nodeId` ("meter", "snapshot", ...) in the voice group containing `voice` — what snapshot() does not carry, and
 * what tells a caller of elem_b200_poll_readouts whether `a` / `b` are min / max or a snapshot's value.  Writes up to `cap` bytes
 * including the terminating NUL, returns the name's length + 1, or 0 when that group has no such node.  No reference method. */
int elem_b200_node_type(elem_b200_runtime* rt, int voice, int32_t nodeId, char* buf, size_t cap);

/* JSON description of voice groups and compiled programs; returns bytes needed.  "steady": the next block of the same shape relaunches
 * cached work without walking the groups.  Per group, "mix_channels": the non-negative root channels of the program the last block
 * rendered (before the first block, of the queued one) — its mix channels for any nOut past 8 are those below nOut. */
int elem_b200_describe(elem_b200_runtime* rt, char* buf, size_t cap);
/* The encoded render program (32-bit words, elementary_b200/csrc/program.h) of the voice group containing `voice`; writes up to
 * `cap` words, returns the program length.  Introspection only (tests; input of per-program kernel specialisation). */
int elem_b200_program_words(elem_b200_runtime* rt, int voice, uint32_t* buf, size_t cap);
/* EXPERIMENTAL (option "specialize" = 1, off by default; DESIGN.md §8): K1 compiled at run time by NVRTC against the render
 * program of a voice group as a compile-time constant.  This entry point only COMPILES the specialised kernel of the group
 * containing `voice` (no GPU needed) and returns the cubin size, or -1 with the compiler log in logBuf. */
long elem_b200_specialize_dry_run(elem_b200_runtime* rt, int voice, char* logBuf, size_t cap);
/* A/B builds of the library compiled with -DEB_OPPROF (tools/opprof.py) only: cycles (out128[2*op]) and dispatch counts
 * (out128[2*op+1]) per opcode of the K1 interpreter since the last reset; the product library writes zeros.  Engine option
 * "spec_opprof" = 1 compiles the same counters into the specialised kernels (any library build); theirs are added in.  No reference counterpart:
 * this is what the pipeline cost model of the host compiler is calibrated against.  Returns 0, or -1 on a CUDA error. */
int elem_b200_debug_opprof(elem_b200_runtime* rt, unsigned long long* out128, int reset);
/* Number of CUDA kernels this runtime has launched so far. */
uint64_t elem_b200_kernel_launches(elem_b200_runtime* rt);
/* With option "time_kernels" = 1 every K1 render-kernel launch is bracketed by CUDA events on the launching
 * stream; this returns the summed device time (ms) of the launches since the previous call and their count.
 * Synchronises the stream. */
double elem_b200_take_kernel_time_ms(elem_b200_runtime* rt, uint64_t* count);
/* Same for the K3 convolver launches, as gathered by the most recent elem_b200_take_kernel_time_ms() call. */
double elem_b200_last_convolve_time_ms(elem_b200_runtime* rt, uint64_t* count);
/* Per kernel kind, as gathered by the most recent elem_b200_take_kernel_time_ms() call: ms[4] / counts[4] = summed device ms and
 * launch counts of K1 (render), K2 (mix reduce; K2w past 8 output channels), K3 (convolver), K4 (cross-GPU mix exchange). */
void elem_b200_last_kernel_times(elem_b200_runtime* rt, double* ms4, uint64_t* counts4);
const char* elem_b200_last_error(elem_b200_runtime* rt);
/* ReturnCode::describe — runtime/elem/Types.h:62-85 */
const char* elem_b200_describe_return_code(int code);
/* Number of CUDA devices visible (0 = the library cannot run here). */
int elem_b200_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* ELEM_B200_H */
