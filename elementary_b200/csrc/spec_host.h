// spec_host.h — per-program specialisation of K1 at run time (DESIGN.md §4 "K1, specialised").
//
// render_kernel.cu is compiled a second time, by NVRTC, with the render program of one voice group as a compile-time constant
// (EB_SPEC_PROGRAM, see the #ifdef in render_tile): the interpreter's per-op bodies are reused verbatim, dispatch and operand
// decoding fold away.  libnvrtc and libcuda are opened with dlopen, so the library has no load-time dependency on either.
//
// The device sources NVRTC compiles are the ones THIS library was built from: spec_sources.S embeds render_kernel.cu,
// render_ops.inc, program.h, kernels.h and rtc_compat.h into the shared object at build time, so a specialised kernel can never
// disagree with the host about LaunchParams or the opcode numbering, and an installed .so needs no csrc/ directory next to it.
//
// Threading: all compilations of a process run on ONE worker thread fed by a queue (a thousand voice groups never become a
// thousand NVRTC threads), results are cached by (program words with device pointers masked, tile geometry, device), so the two
// halves of a split group — or every rank-local engine of one process — share one compilation.  Jobs are owned jointly by the
// queue, the cache and the programs that asked for them; dropping a Program on the render thread never waits for the compiler.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "program.h"

namespace eb {

struct SpecKernel {
    void* module = nullptr;      // CUmodule (lives as long as the process: cached kernels are never unloaded)
    void* function = nullptr;    // CUfunction of render_block_kernel<NITER, LOGL> specialised for one program
    std::vector<char> cubin;
    std::string loweredName;     // mangled name of the kernel inside the cubin
    int numRegs = 0, localBytes = 0;   // filled by specialise_load (cuFuncGetAttribute): reported by describe()
    std::string opprofName;      // -DEB_OPPROF builds: mangled name of the per-opcode counter array g_opprof
    unsigned long long opprofPtr = 0;  // its device address once loaded
};

// Step 1 — pure compilation (NVRTC only; thread safe, needs no CUDA context, works without a GPU): K1 for (tileWidth,
// niterOverride) against `code` (one single-stage program).  Fills out.cubin / out.loweredName.
// minBlocks > 0: CTAs per SM the narrow geometries (1 < L < 32) are compiled for (8 = 64 registers); opprof: compile the per-opcode
// cycle counters in (-DEB_OPPROF, read with specialise_opprof_read).
bool specialise_compile(const std::vector<uint32_t>& code, int tileWidth, int niterOverride, const std::string& customSource, SpecKernel& out, std::string& log,
                        int minBlocks = 0, bool opprof = false);
// Step 2 — on a thread whose CUDA context is current: load the cubin and resolve the kernel (milliseconds).
bool specialise_load(SpecKernel& k, std::string& log);

// A compilation request.  state: 0 queued / compiling, 1 compiled (cubin ready, not loaded), 2 loaded, -1 failed (log says why).
struct SpecJob {
    std::atomic<int> state{0};
    SpecKernel kernel;
    std::string log;             // written by the worker before state leaves 0, by the loader before it leaves 1
    std::mutex loadMutex;        // two engines sharing a cached job must not both load it
    std::vector<uint32_t> code;
    std::string customSource;
    int tileWidth = 0, niterOverride = 0, minBlocks = 0;
    bool opprof = false;
};
// Queue (or find in the cache) the specialisation of `code` for a tile geometry on `device`.  Never blocks on the compiler.
// customSource: device text of the registered node types the program may use (Engine::customSource; empty = none) — compiled in front of the kernel.
std::shared_ptr<SpecJob> specialise_request(const std::vector<uint32_t>& code, int tileWidth, int niterOverride, int device, const std::string& customSource,
                                            int minBlocks = 0, bool opprof = false);
// A loaded kernel compiled with opprof: adds its counters (out128[2 * op] cycles, [2 * op + 1] dispatches, op 63 = whole sample loop of a
// warp) to out128, optionally zeroing them.  A kernel without counters adds nothing.
bool specialise_opprof_read(const SpecKernel& k, unsigned long long* out128, bool reset);
// Block until the job has left state 0 (used by option "specialize" = 2 and by tests).
void specialise_wait(SpecJob& job);
// Render thread: load a compiled job (state 1 -> 2 / -1).  Returns the state afterwards.
int specialise_ensure_loaded(SpecJob& job);

// cuLaunchKernel of a specialised kernel with the same launch geometry the built-in instantiation would get.
cudaError_t specialise_launch(const SpecKernel& k, const LaunchParams& P, int grid, int threads, size_t smem, int perWarpFloats, cudaStream_t stream);

// The part of a program the specialised kernel is compiled against: everything up to and including the first OP_END, with the
// device-pointer words of every header zeroed (the kernel reads those from the copy of the program in memory).
std::vector<uint32_t> specialise_key_words(const std::vector<uint32_t>& code);

}  // namespace eb
