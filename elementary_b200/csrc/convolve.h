// convolve.h — K3: partitioned-FFT convolver for the `convolve` node (device side in convolve_kernel.cu).
//
// Reference: ConvolutionNode (wasm/Convolve.h:23-92) wraps fftconvolver::TwoStageFFTConvolver(head 512, tail 4096)
// (wasm/FFTConvolver/TwoStageFFTConvolver.cpp:74-220, FFTConvolver.cpp:85-204).  Whatever its internal staging, that
// object computes — with zero latency and for any call length — the plain linear convolution of the input stream
// with the impulse response (after dropping trailing taps with |h| < 1e-6, FFTConvolver.cpp:94-98).  Here the same
// convolution is evaluated as ONE uniformly partitioned frequency-domain delay line per channel (partition 512,
// FFT 1024, S = ceil(irLen/512) partitions), the structure of the reference's head stage applied to the whole IR:
// no 8192-point tail bursts, identical work every block, spectra streamed once per block.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace eb {

constexpr int CONV_BLOCK = 512;          // partition / head block size (Convolve.h:49: init(512, 4096, ...))
constexpr int CONV_FFT = 1024;           // segment size 2*B (FFTConvolver.cpp:107)
constexpr int CONV_BINS = 513;           // ComplexSize(1024)
constexpr int CONV_PACKED_BINS = 512;    // stored spectra: bin 0 = (Re X[0], Re X[512]) — both bins are purely real
constexpr int CONV_CH_PER_CTA = 2;       // channels sharing one pass over the IR spectra

// The partition spectra of one impulse response after trimming (FFTConvolver.cpp:94-98): the engine's own copy, computed once
// per shared resource however many convolvers and channels use it, freed when the last of them lets go.
struct IrSpectra {
    int partitions = 0;                  // S_v (0: the IR trimmed to nothing — silence)
    float2* dH = nullptr;                // [S_v][512] (packed)
    bool planOnly = false;
    ~IrSpectra();
};

// Spectra by resource object.  Resources are immutable and nodes hold them by shared_ptr, so the object is the key; an entry whose
// resource died (pruned) may meet a new resource at the same address, which is why the owner is checked too.
class IrBank {
public:
    std::shared_ptr<IrSpectra> acquire(const void* key, const std::weak_ptr<const void>& owner, const float* ir, size_t irLen,
                                       bool planOnly, cudaStream_t stream, std::string& err);
    size_t live() const;                 // entries some convolver still uses
private:
    struct Entry { std::weak_ptr<const void> owner; std::weak_ptr<IrSpectra> spectra; };
    std::map<const void*, Entry> entries_;
};

// Per-channel descriptor of the per-channel-IR form of K3.
struct ConvChannel { const float2* H; int S; int pad; };

struct ConvolverState {
    int partitions = 0;                  // R: slots of the input spectra ring = the largest S_v of the group's channels
    int nv = 0;                          // channels (voices of the group)
    int cur = 0;                         // FDL slot of the block being filled (decrements per block: FFTConvolver.cpp:200)
    int fill = 0;                        // samples already in the current partition's input buffer (:157-162)
    float2* dFdl = nullptr;              // [nv][R][512] input spectra ring (frequency-domain delay line)
    float2* dYpre = nullptr;             // [nv][512]  sum over the older partitions, valid while fill > 0 (:168-177)
    float* dOverlap = nullptr;           // [nv][512]
    float* dInBuf = nullptr;             // [nv][512]
    float2* dTw = nullptr;               // [512] exp(-2*pi*i*m/1024)
    // impulse responses: chIr[c] = the spectra channel c convolves with; irs = the distinct ones, in order of first use
    std::vector<std::shared_ptr<IrSpectra>> chIr, irs;
    int maxS = 0;                        // largest S_v in use (0: every channel is silent)
    // per-channel form (more than one distinct IR): descriptors [nv] and work units [ceil(nv/2)] {c0, c1 (-1: none), max S, same IR}
    ConvChannel* dChan = nullptr;
    int4* dUnits = nullptr;
    std::vector<std::pair<cudaEvent_t, void*>> retired;   // rings replaced by a larger one, freed once the stream has passed the event
    bool planOnly = false;
    ~ConvolverState();
    bool perChannel() const { return irs.size() > 1; }
    size_t bytesPerChannel() const { return (size_t) partitions * CONV_PACKED_BINS * 8 + CONV_PACKED_BINS * 8 + 2 * CONV_BLOCK * 4; }
};

// Build the device state for `nv` channels sharing one impulse response (the bank entry of resource `key`). Returns false and
// fills `err` on failure.
bool convolver_init(ConvolverState& st, IrBank& bank, const void* key, const std::weak_ptr<const void>& owner, const float* ir, size_t irLen,
                    int nv, bool planOnly, cudaStream_t stream, std::string& err);

// Channels [c0, c0 + n) start over (zero input history: a fresh TwoStageFFTConvolver, Convolve.h:45-51) on spectra `h[i]`; the ring
// grows (keeping every channel's most recent spectra, in order) when an IR is longer than any before.  Stream-ordered.
bool convolver_assign(ConvolverState& st, int c0, int n, const std::vector<std::shared_ptr<IrSpectra>>& h, cudaStream_t stream, std::string& err);

// What one channel owns of the state, voice-major: base + c * bytesPerChannel.  convolver_assign zeroes these regions of the channels
// that restart; a voice reset (K6, Engine::resetVoices) zeroes them on the device.
struct ConvRegion { void* base; size_t bytesPerChannel; };
std::vector<ConvRegion> convolver_channel_regions(const ConvolverState& st);

// Copy of channels [c0, c0+n) of `src` (same IRs, same position in the partition cycle) — used when a voice group is cut.
bool convolver_clone_range(const ConvolverState& src, int c0, int n, ConvolverState& dst, cudaStream_t stream, std::string& err);
// Keep only the first n channels (the other half of a cut): the unit table and descriptors are rebuilt, the storage stays.
bool convolver_truncate(ConvolverState& st, int n, cudaStream_t stream, std::string& err);

// Root + mix fused behind the inverse transform (graph_host.cpp sets it when the convolver's output feeds nothing but the graph's root,
// the `convolve -> root` shape of a reverb send: BASELINE config 4).  The kernel then applies the root's gain fade exactly like K1's
// OP_ROOT does (Core.h:66-78, GainFade.h:56-72: g = clamp(gain0 + step * sampleIndex) while fading, the target otherwise), writes the
// per-voice output and this channel's row of the per-tile partial mix (one-voice tiles: row = channel) — the K1 launch that would only
// have re-read the block and multiplied it disappears, and the convolver's own output buffer is not written at all.
struct ConvEpilogue {
    bool active = false;
    bool running = true;             // the root's sub-sequence runs this block (else: silence, like the skipped segment in K1)
    float gain0 = 1.0f, step = 0.0f, target = 1.0f;
    int channel = 0;                 // the root's output channel
    int nOut = 1, blockSize = 512;
    float* mixPartial = nullptr;     // [tileBase + channel][nOut][blockSize] or null
    int tileBase = 0;
    float* outVoice = nullptr;       // [voice0 + channel][nOut][outStride] (+ outOffset) or null
    int voice0 = 0, outStride = 512, outOffset = 0;
};

// Convolve `n` more samples (n <= 512 - st.fill) of every channel: in is [channel][inStride] (inStride 0 = one input shared by
// all channels), out is [channel][outStride]; the samples of this call start at `offset`.  Advances st.fill / st.cur.
cudaError_t convolver_process_chunk(ConvolverState& st, const float* in, int inStride, float* out, int outStride, int offset, int n, cudaStream_t stream,
                                    const ConvEpilogue& epi = ConvEpilogue{});

// Ring growth on the stream: dst[c][i] = src[c][(cur + i) mod oldR] for i < oldR (newest first), zeros for oldR <= i < newR.
cudaError_t convolver_relayout(float2* dst, const float2* src, int nv, int oldR, int newR, int cur, cudaStream_t stream);

// Algorithmic HBM bytes of one full 512-sample block for one channel (DESIGN.md §4 K3).
inline size_t convolver_algorithmic_bytes_per_channel_block(int partitions) {
    return (size_t) 2 * CONV_BLOCK * 4                         // input read + output write
         + (size_t) (partitions - 1) * CONV_PACKED_BINS * 8    // older input spectra read
         + (size_t) CONV_PACKED_BINS * 8                       // newest spectrum written
         + (size_t) 2 * CONV_BLOCK * 4;                        // overlap read + write
}

} // namespace eb
