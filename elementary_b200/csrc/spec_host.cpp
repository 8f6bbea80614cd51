// spec_host.cpp — see spec_host.h.
#include "spec_host.h"

#include <cuda.h>
#include <dlfcn.h>
#include <nvrtc.h>

#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <sstream>
#include <thread>

#include "kernels.h"

// The device sources this library was built from (spec_sources.S, .incbin): NUL-terminated texts.
extern "C" {
extern const char eb_src_render_kernel_cu[];
extern const char eb_src_render_ops_inc[];
extern const char eb_src_program_h[];
extern const char eb_src_kernels_h[];
extern const char eb_src_rtc_compat_h[];
}

namespace eb {

namespace {

struct Api {
    bool nvrtcOk = false, driverOk = false;
    std::string nvrtcErr, driverErr;
    decltype(&nvrtcCreateProgram) createProgram = nullptr;
    decltype(&nvrtcDestroyProgram) destroyProgram = nullptr;
    decltype(&nvrtcAddNameExpression) addNameExpression = nullptr;
    decltype(&nvrtcCompileProgram) compileProgram = nullptr;
    decltype(&nvrtcGetProgramLogSize) getLogSize = nullptr;
    decltype(&nvrtcGetProgramLog) getLog = nullptr;
    decltype(&nvrtcGetCUBINSize) getCubinSize = nullptr;
    decltype(&nvrtcGetCUBIN) getCubin = nullptr;
    decltype(&nvrtcGetLoweredName) getLoweredName = nullptr;
    decltype(&cuModuleLoadData) moduleLoadData = nullptr;
    decltype(&cuModuleUnload) moduleUnload = nullptr;
    decltype(&cuModuleGetFunction) moduleGetFunction = nullptr;
    decltype(&cuFuncSetAttribute) funcSetAttribute = nullptr;
    decltype(&cuFuncGetAttribute) funcGetAttribute = nullptr;
    decltype(&cuLaunchKernel) launchKernel = nullptr;
    decltype(&cuGetErrorString) getErrorString = nullptr;
    decltype(&cuModuleGetGlobal) moduleGetGlobal = nullptr;   // optional: only opprof kernels use it
};

template <typename F>
bool sym(void* h, const char* name, F& f) {
    f = reinterpret_cast<F>(dlsym(h, name));
    return f != nullptr;
}

// Both halves are resolved exactly once, each under its own std::call_once: a handle is never visible before every entry
// point behind it is, whichever thread (compile worker, render thread) gets there first.
Api& api() {
    static Api a;
    return a;
}
std::once_flag g_nvrtcOnce, g_driverOnce;
void waitForCompilerAtExit();   // below: registered with atexit once NVRTC is loaded

bool loadNvrtc(std::string& log) {
    Api& a = api();
    std::call_once(g_nvrtcOnce, [&a]() {
        void* h = nullptr;
        for (const char* n : {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12"}) {
            h = dlopen(n, RTLD_NOW | RTLD_LOCAL);
            if (h) break;
        }
        if (!h) { a.nvrtcErr = "libnvrtc not found (dlopen)"; return; }
        a.nvrtcOk = sym(h, "nvrtcCreateProgram", a.createProgram) && sym(h, "nvrtcDestroyProgram", a.destroyProgram) &&
                    sym(h, "nvrtcAddNameExpression", a.addNameExpression) && sym(h, "nvrtcCompileProgram", a.compileProgram) &&
                    sym(h, "nvrtcGetProgramLogSize", a.getLogSize) && sym(h, "nvrtcGetProgramLog", a.getLog) &&
                    sym(h, "nvrtcGetCUBINSize", a.getCubinSize) && sym(h, "nvrtcGetCUBIN", a.getCubin) &&
                    sym(h, "nvrtcGetLoweredName", a.getLoweredName);
        if (!a.nvrtcOk) { a.nvrtcErr = "libnvrtc lacks a required entry point"; dlclose(h); }
        // A process that exits while the (detached) compile-queue thread is inside nvrtcCompileProgram tears NVRTC's own statics down
        // under it (segfault / "realloc(): invalid pointer" at exit).  Registered HERE — after NVRTC's static initialisers have run —
        // the handler runs BEFORE their destructors and simply waits for the compile in flight; no further job is started.
        else std::atexit(waitForCompilerAtExit);
    });
    if (!a.nvrtcOk) log = a.nvrtcErr;
    return a.nvrtcOk;
}

bool loadDriver(std::string& log) {
    Api& a = api();
    std::call_once(g_driverOnce, [&a]() {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!h) { a.driverErr = "libcuda.so.1 not found (no CUDA driver on this machine)"; return; }
        a.driverOk = sym(h, "cuModuleLoadData", a.moduleLoadData) && sym(h, "cuModuleUnload", a.moduleUnload) &&
                     sym(h, "cuModuleGetFunction", a.moduleGetFunction) && sym(h, "cuFuncSetAttribute", a.funcSetAttribute) &&
                     sym(h, "cuFuncGetAttribute", a.funcGetAttribute) && sym(h, "cuLaunchKernel", a.launchKernel) &&
                     sym(h, "cuGetErrorString", a.getErrorString);
        if (!a.driverOk) { a.driverErr = "libcuda lacks a required entry point"; dlclose(h); }
        else sym(h, "cuModuleGetGlobal_v2", a.moduleGetGlobal);
    });
    if (!a.driverOk) log = a.driverErr;
    return a.driverOk;
}

std::string cuErr(CUresult r) {
    const char* s = nullptr;
    if (api().getErrorString && api().getErrorString(r, &s) == CUDA_SUCCESS && s) return std::string(s) + " (CUresult " + std::to_string((int) r) + ")";
    return "CUresult " + std::to_string((int) r);
}

// ---- the compile queue: one worker thread per process, started on first use, detached (it owns the queue through a shared_ptr,
// so nothing has to be joined or torn down in a static destructor) ----
struct Queue {
    std::mutex m;
    std::condition_variable cv, done;
    std::deque<std::shared_ptr<SpecJob>> jobs;
    std::map<std::string, std::shared_ptr<SpecJob>> cache;
    bool workerStarted = false;
    bool busy = false;          // the worker is inside specialise_compile
    bool quitting = false;      // the process is exiting: the worker starts nothing new
};
std::shared_ptr<Queue> queue() {
    static std::shared_ptr<Queue> q = std::make_shared<Queue>();
    return q;
}

void workerLoop(std::shared_ptr<Queue> q) {
    for (;;) {
        std::shared_ptr<SpecJob> job;
        {
            std::unique_lock<std::mutex> lk(q->m);
            q->cv.wait(lk, [&] { return !q->jobs.empty() || q->quitting; });
            if (q->quitting) return;
            job = q->jobs.front();
            q->jobs.pop_front();
            q->busy = true;
        }
        std::string log;
        const bool ok = specialise_compile(job->code, job->tileWidth, job->niterOverride, job->customSource, job->kernel, log, job->minBlocks, job->opprof);
        {
            std::lock_guard<std::mutex> lk(q->m);
            job->log = log;
            job->state.store(ok ? 1 : -1, std::memory_order_release);
            q->busy = false;
        }
        q->done.notify_all();
    }
}

void waitForCompilerAtExit() {
    auto q = queue();
    std::unique_lock<std::mutex> lk(q->m);
    q->quitting = true;
    q->cv.notify_all();
    q->done.wait(lk, [&] { return !q->busy; });
}

}  // namespace

std::vector<uint32_t> specialise_key_words(const std::vector<uint32_t>& code) {
    std::vector<uint32_t> out;
    size_t pc = 0;
    while (pc + OP_HEADER_WORDS <= code.size()) {
        const uint32_t w0 = code[pc];
        const size_t n = OP_HEADER_WORDS + ((w0 >> 8) & 0xFF);
        if (pc + n > code.size()) break;
        const size_t at = out.size();
        out.insert(out.end(), code.begin() + (long) pc, code.begin() + (long) (pc + n));
        out[at + 4] = 0; out[at + 5] = 0;     // device pointer: read from memory by the kernel, never a constant
        pc += n;
        if ((w0 & 0xFF) == OP_END) break;
    }
    return out;
}

bool specialise_compile(const std::vector<uint32_t>& codeIn, int tileWidth, int niterOverride, const std::string& customSource, SpecKernel& out, std::string& log,
                        int minBlocks, bool opprof) {
    if (!loadNvrtc(log)) return false;
    Api& a = api();
    const std::vector<uint32_t> code = specialise_key_words(codeIn);
    if (code.empty()) { log = "empty program"; return false; }

    std::ostringstream hdr;   // the program as a constant: what EB_SPEC_PROGRAM / EB_SPEC_CODE stand for in render_tile
    hdr << "#pragma once\n#include \"rtc_compat.h\"\nnamespace eb {\n__device__ constexpr uint32_t EB_SPEC_CODE[] = {";
    for (size_t i = 0; i < code.size(); ++i) hdr << (i ? "," : "") << "0x" << std::hex << code[i] << "u";
    hdr << "};\nconstexpr int EB_SPEC_CODE_LEN = " << std::dec << code.size() << ";\n}\n#define EB_SPEC_PROGRAM 1\n";
    hdr << customSource;      // bodies of the registered node types (OP_CUSTOM), if any
    const std::string hdrText = hdr.str();
    const char* hdrSrc[] = {hdrText.c_str(), eb_src_render_ops_inc, eb_src_program_h, eb_src_kernels_h, eb_src_rtc_compat_h};
    const char* hdrNames[] = {"eb_spec_program.h", "render_ops.inc", "program.h", "kernels.h", "rtc_compat.h"};

    nvrtcProgram prog = nullptr;
    if (a.createProgram(&prog, eb_src_render_kernel_cu, "render_kernel.cu", 5, hdrSrc, hdrNames) != NVRTC_SUCCESS) { log = "nvrtcCreateProgram failed"; return false; }
    int logl = 0;
    for (int l = tileWidth; l > 1; l >>= 1) ++logl;
    const int niter = render_niter_for(tileWidth, niterOverride);
    const std::string name = "eb::render_block_kernel<" + std::to_string(niter) + ", " + std::to_string(logl) + ">";
    a.addNameExpression(prog, name.c_str());
    const char* const opprofExpr = "&eb::g_opprof";
    if (opprof) a.addNameExpression(prog, opprofExpr);
    const std::string mb = "-DEB_NARROW_MINBLOCKS=" + std::to_string(minBlocks > 0 ? minBlocks : 4);
    const char* opts[] = {"--std=c++20", "--gpu-architecture=sm_90a", "--fmad=false", "-lineinfo", "-default-device",
                          "--pre-include=eb_spec_program.h", "-diag-suppress=186,68,179,177", mb.c_str(), "-DEB_OPPROF"};
    const int nOpts = (int) (sizeof(opts) / sizeof(opts[0])) - (opprof ? 0 : 1);
    const nvrtcResult rc = a.compileProgram(prog, nOpts, opts);
    size_t n = 0;
    a.getLogSize(prog, &n);
    if (n > 1) { log.resize(n); a.getLog(prog, &log[0]); }
    bool ok = rc == NVRTC_SUCCESS;
    std::string lowered;
    if (ok) {
        size_t sz = 0;
        ok = a.getCubinSize(prog, &sz) == NVRTC_SUCCESS && sz > 0;
        if (ok) { out.cubin.resize(sz); ok = a.getCubin(prog, out.cubin.data()) == NVRTC_SUCCESS; }
        const char* ln = nullptr;
        if (ok && a.getLoweredName(prog, name.c_str(), &ln) == NVRTC_SUCCESS && ln) lowered = ln; else ok = false;
        const char* pn = nullptr;
        if (ok && opprof) { if (a.getLoweredName(prog, opprofExpr, &pn) == NVRTC_SUCCESS && pn) out.opprofName = pn; else ok = false; }
    }
    a.destroyProgram(&prog);
    if (!ok) { if (log.empty()) log = "NVRTC compilation failed"; return false; }
    out.loweredName = lowered;
    return true;
}

bool specialise_load(SpecKernel& k, std::string& log) {
    if (k.function) return true;
    if (k.cubin.empty() || k.loweredName.empty()) { log = "nothing compiled"; return false; }
    if (!loadDriver(log)) return false;
    Api& a = api();
    CUmodule mod = nullptr;
    CUfunction fn = nullptr;
    CUresult r = a.moduleLoadData(&mod, k.cubin.data());
    if (r != CUDA_SUCCESS) { log = "cuModuleLoadData failed: " + cuErr(r); return false; }
    r = a.moduleGetFunction(&fn, mod, k.loweredName.c_str());
    if (r != CUDA_SUCCESS) { a.moduleUnload(mod); log = "cuModuleGetFunction failed for " + k.loweredName + ": " + cuErr(r); return false; }
    a.funcGetAttribute(&k.numRegs, CU_FUNC_ATTRIBUTE_NUM_REGS, fn);
    a.funcGetAttribute(&k.localBytes, CU_FUNC_ATTRIBUTE_LOCAL_SIZE_BYTES, fn);
    if (!k.opprofName.empty()) {
        CUdeviceptr p = 0;
        size_t bytes = 0;
        r = a.moduleGetGlobal ? a.moduleGetGlobal(&p, &bytes, mod, k.opprofName.c_str()) : CUDA_ERROR_NOT_FOUND;
        if (r != CUDA_SUCCESS) { a.moduleUnload(mod); log = "cuModuleGetGlobal failed for the opprof counters: " + cuErr(r); return false; }
        k.opprofPtr = (unsigned long long) p;
    }
    k.module = mod;
    k.function = fn;
    return true;
}

std::shared_ptr<SpecJob> specialise_request(const std::vector<uint32_t>& code, int tileWidth, int niterOverride, int device, const std::string& customSource,
                                            int minBlocks, bool opprof) {
    // Load NVRTC (and so register waitForCompilerAtExit) on THIS thread, before any job can reach the worker: loaded lazily by the
    // worker, a process that queues a job and exits at once could start exiting before the handler exists, and the worker would then
    // run NVRTC while its statics are torn down.  A load failure is reported by the job itself.
    {
        std::string ignored;
        loadNvrtc(ignored);
    }
    auto q = queue();
    const std::vector<uint32_t> key = specialise_key_words(code);
    std::string k(reinterpret_cast<const char*>(key.data()), key.size() * sizeof(uint32_t));
    k += "|c" + customSource + "|L" + std::to_string(tileWidth) + "|n" + std::to_string(render_niter_for(tileWidth, niterOverride)) + "|d" + std::to_string(device) + "|b" + std::to_string(minBlocks) + "|p" + (opprof ? "1" : "0");
    std::lock_guard<std::mutex> lk(q->m);
    auto it = q->cache.find(k);
    if (it != q->cache.end() && it->second->state.load(std::memory_order_acquire) >= 0) return it->second;
    auto job = std::make_shared<SpecJob>();
    job->code = key;
    job->customSource = customSource;
    job->tileWidth = tileWidth;
    job->niterOverride = niterOverride;
    job->minBlocks = minBlocks;
    job->opprof = opprof;
    q->cache[k] = job;
    q->jobs.push_back(job);
    if (!q->workerStarted) {
        q->workerStarted = true;
        std::thread(workerLoop, q).detach();
    }
    q->cv.notify_one();
    return job;
}

void specialise_wait(SpecJob& job) {
    auto q = queue();
    std::unique_lock<std::mutex> lk(q->m);
    q->done.wait(lk, [&] { return job.state.load(std::memory_order_acquire) != 0; });
}

int specialise_ensure_loaded(SpecJob& job) {
    int st = job.state.load(std::memory_order_acquire);
    if (st != 1) return st;
    std::lock_guard<std::mutex> lk(job.loadMutex);
    st = job.state.load(std::memory_order_acquire);
    if (st != 1) return st;
    std::string log;
    const bool ok = specialise_load(job.kernel, log);
    if (!ok) job.log = log;
    job.state.store(ok ? 2 : -1, std::memory_order_release);
    return ok ? 2 : -1;
}

bool specialise_opprof_read(const SpecKernel& k, unsigned long long* out128, bool reset) {
    if (!k.opprofPtr) return true;
    unsigned long long buf[128];
    void* dev = reinterpret_cast<void*>((uintptr_t) k.opprofPtr);   // unified addressing: the module's global as a runtime-API pointer
    if (cudaMemcpy(buf, dev, sizeof buf, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    for (int i = 0; i < 128; ++i) out128[i] += buf[i];
    return !reset || cudaMemset(dev, 0, sizeof buf) == cudaSuccess;
}

cudaError_t specialise_launch(const SpecKernel& k, const LaunchParams& P, int grid, int threads, size_t smem, int perWarpFloats, cudaStream_t stream) {
    Api& a = api();
    if (!k.function || !a.launchKernel) return cudaErrorInvalidDeviceFunction;
    CUfunction fn = static_cast<CUfunction>(k.function);
    CUresult r = a.funcSetAttribute(fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int) smem);
    if (r != CUDA_SUCCESS) { std::fprintf(stderr, "elem_b200: cuFuncSetAttribute(smem=%zu) on a specialised kernel: %s\n", smem, cuErr(r).c_str()); return cudaErrorInvalidValue; }
    LaunchParams params = P;
    int perWarp = perWarpFloats;
    void* args[] = {&params, &perWarp};
    r = a.launchKernel(fn, (unsigned) grid, 1, 1, (unsigned) threads, 1, 1, (unsigned) smem, reinterpret_cast<CUstream>(stream), args, nullptr);
    if (r == CUDA_SUCCESS) return cudaSuccess;
    std::fprintf(stderr, "elem_b200: cuLaunchKernel of a specialised kernel failed: %s\n", cuErr(r).c_str());
    switch (r) {   // keep the cause: the caller reports cudaGetErrorString of what comes back
        case CUDA_ERROR_INVALID_VALUE: return cudaErrorInvalidValue;
        case CUDA_ERROR_OUT_OF_MEMORY: return cudaErrorMemoryAllocation;
        case CUDA_ERROR_LAUNCH_OUT_OF_RESOURCES: return cudaErrorLaunchOutOfResources;
        case CUDA_ERROR_INVALID_HANDLE: return cudaErrorInvalidResourceHandle;
        case CUDA_ERROR_INVALID_CONTEXT: return cudaErrorDeviceUninitialized;
        default: return cudaErrorLaunchFailure;
    }
}

}  // namespace eb
