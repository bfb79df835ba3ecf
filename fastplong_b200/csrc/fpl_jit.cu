// Run-time specialisation of the adapter+quality scan (k_scan_jit, source in fpl_scan_jit_src.h): NVRTC compiles it
// for sm_90a with the two adapter strings and the option flags as constants, the driver API loads and launches it.
// Modules are cached per (device, specialisation) for the life of the process.
#include <cuda.h>
#include <cuda_runtime.h>
#include <nvrtc.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <mutex>
#include <functional>
#include <string>
#include <vector>
#include "fpl_device.cuh"
#include "fpl_jit.h"
#include "fpl_scan_jit_src.h"
#include "fpl_scan_jit2_src.h"

#include <dlfcn.h>

namespace {
struct Cached { CUmodule mod; CUfunction fn; };
std::mutex g_mu;
std::map<std::string, Cached> g_cache;

// The driver library is resolved lazily: libfplgpu.so must stay loadable on a machine without a GPU driver
// (build check, symbol test), where only fpl_create() fails.
struct Driver {
    CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
    CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
    CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream,
                             void**, void**) = nullptr;
    CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
    bool ok = false;
    Driver() {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        ModuleLoadData = (decltype(ModuleLoadData))dlsym(h, "cuModuleLoadData");
        ModuleGetFunction = (decltype(ModuleGetFunction))dlsym(h, "cuModuleGetFunction");
        LaunchKernel = (decltype(LaunchKernel))dlsym(h, "cuLaunchKernel");
        GetErrorString = (decltype(GetErrorString))dlsym(h, "cuGetErrorString");
        ok = ModuleLoadData && ModuleGetFunction && LaunchKernel && GetErrorString;
    }
};
Driver& driver() { static Driver d; return d; }

// ---- version 2: the match counter of one adapter as straight-line CUDA source ----
// A streaming 3:2 compressor: every letter's match vector (one funnel shift of the letter's mask of this lane and of
// its neighbour) is pushed at weight 1; as soon as a weight holds three vectors a full adder turns them into one
// vector of that weight and a carry that is pushed at the next weight.  What is left at the end (at most two vectors
// per weight) is rippled upwards.  Every full adder removes one vector, so an adapter of n letters costs about
// n - log2(n) of them (25 for 30 letters) and at most three vectors per weight are ever live.
std::string gen_counter(int which, const char* adapter) {
    const int alen = (int)strlen(adapter);
    int amax_bits = 0;
    while ((1 << amax_bits) <= alen) amax_bits++;        // planes this adapter's count needs
    std::string out = "__device__ __forceinline__ void count_matches_" + std::to_string(which) +
                      "(const Masks& m, uint32_t (&c)[NPL]) {\n";
    std::vector<std::vector<std::string>> buf(12);
    int tmp = 0;
    auto fresh = [&] { return std::string("t") + std::to_string(which) + "_" + std::to_string(tmp++); };
    std::function<void(const std::string&, int)> push = [&](const std::string& v, int w) {
        buf[w].push_back(v);
        if (buf[w].size() == 3) {
            const std::string sname = fresh(), cname = fresh();
            out += "    FA(" + sname + ", " + cname + ", " + buf[w][0] + ", " + buf[w][1] + ", " + buf[w][2] + ")\n";
            buf[w].clear();
            buf[w].push_back(sname);
            push(cname, w + 1);
        }
    };
    for (int i = 0; i < alen; i++) {
        const char L = adapter[i];
        const int w = i >> 5, sh = i & 31;
        const std::string base = std::string("m.") + L;
        const std::string v = sh == 0 ? base + "[" + std::to_string(w) + "]"
                                      : "FS(" + base + "[" + std::to_string(w) + "], " + base + "[" + std::to_string(w + 1) + "], " + std::to_string(sh) + ")";
        const std::string name = fresh();
        out += "    const uint32_t " + name + " = " + v + ";\n";
        push(name, 0);
    }
    for (int w = 0; w < 11; w++) {
        if (buf[w].size() == 2) {
            const std::string sname = fresh(), cname = fresh();
            out += "    HA(" + sname + ", " + cname + ", " + buf[w][0] + ", " + buf[w][1] + ")\n";
            buf[w].clear();
            buf[w].push_back(sname);
            push(cname, w + 1);
        }
    }
    out += "#pragma unroll\n    for (int b = 0; b < NPL; b++) c[b] = 0u;\n";
    for (int w = 0; w < 11; w++)
        if (!buf[w].empty()) out += "    if constexpr (" + std::to_string(w) + " < NPL) c[" + std::to_string(w) + "] = " + buf[w][0] + ";\n";
    out += "}\n";
    (void)amax_bits;
    return out;
}

std::string scan_source_v2(const char* a0, const char* a1) {
    std::string src = kScanJit2Source;
    const std::string marker = "//@@COUNTERS@@";
    const size_t at = src.find(marker);
    src.replace(at, marker.size(), gen_counter(0, a0) + gen_counter(1, a1));
    return src;
}
}  // namespace

// development aid (tools/jit_check.py): the source text NVRTC would be given for these adapters
extern "C" const char* fpl_jit_debug_source(const char* a0, const char* a1) {
    static std::string keep;
    keep = scan_source_v2(a0, a1);
    return keep.c_str();
}

int fpl_jit_build_scan(int device, const char* a0, const char* a1, bool doAdapters, bool doCounts, bool doCplx, bool doQhist,
                       int qq, FplJitKernel* out, char* err, size_t errlen) {
    out->fn = nullptr;
    out->qhist = false;
    std::string defs;
    if (!doAdapters) { a0 = ""; a1 = ""; }
    const bool v1 = getenv("FPL_JIT_V1") != nullptr;       // the round-1 kernel, kept for A/B measurements
    if (v1) doQhist = false;                                // (version 1 has no histograms)
    defs += std::string("#define FPL_A0 \"") + a0 + "\"\n";
    defs += std::string("#define FPL_A1 \"") + a1 + "\"\n";
    defs += "#define FPL_ALEN0 " + std::to_string(strlen(a0)) + "\n";
    defs += "#define FPL_ALEN1 " + std::to_string(strlen(a1)) + "\n";
    defs += std::string("#define FPL_JIT_VERSION ") + (v1 ? "1" : "2") + "\n";
    defs += std::string("#define FPL_DO_ADAPTERS ") + (doAdapters ? "true" : "false") + "\n";
    defs += std::string("#define FPL_DO_COUNTS ") + (doCounts ? "true" : "false") + "\n";
    defs += std::string("#define FPL_DO_CPLX ") + (doCplx ? "true" : "false") + "\n";
    defs += std::string("#define FPL_DO_QHIST ") + (doQhist ? "true" : "false") + "\n";
    defs += "#define FPL_QQ " + std::to_string(qq & 0x7f) + "\n";
    const char* mb = getenv("FPL_JIT_MINBLOCKS");   // occupancy knob (registers per thread); 8 (64 registers) on H100: 6/8/10 blocks -> 15.1/15.0/23.2 ms (profiles/README.md)
    defs += std::string("#define FPL_MINBLOCKS ") + (mb && atoi(mb) > 0 ? std::to_string(atoi(mb)) : std::string("8")) + "\n";
    const std::string key = std::to_string(device) + "|" + defs;
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_cache.find(key);
    if (it != g_cache.end()) { out->fn = (void*)it->second.fn; out->qhist = doQhist; return 0; }

    const std::string src = defs + (v1 ? std::string(kScanJitSource) : scan_source_v2(a0, a1));
    nvrtcProgram prog;
    if (nvrtcCreateProgram(&prog, src.c_str(), "fpl_scan_jit.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) {
        snprintf(err, errlen, "nvrtcCreateProgram failed");
        return -1;
    }
    const char* opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo"};
    nvrtcResult rc = nvrtcCompileProgram(prog, 3, opts);
    if (rc != NVRTC_SUCCESS) {
        size_t n = 0;
        nvrtcGetProgramLogSize(prog, &n);
        std::vector<char> log(n + 1, 0);
        nvrtcGetProgramLog(prog, log.data());
        snprintf(err, errlen, "NVRTC: %s: %.300s", nvrtcGetErrorString(rc), log.data());
        nvrtcDestroyProgram(&prog);
        return -1;
    }
    size_t n = 0;
    nvrtcGetCUBINSize(prog, &n);
    std::vector<char> cubin(n);
    nvrtcGetCUBIN(prog, cubin.data());
    nvrtcDestroyProgram(&prog);
    // the runtime API has already made the device's primary context current (cudaSetDevice + allocations in fpl_create)
    Cached c;
    if (!driver().ok) { snprintf(err, errlen, "libcuda.so.1 not loadable"); return -1; }
    CUresult cr = driver().ModuleLoadData(&c.mod, cubin.data());
    if (cr == CUDA_SUCCESS) cr = driver().ModuleGetFunction(&c.fn, c.mod, "k_scan_jit");
    if (cr != CUDA_SUCCESS) {
        const char* s = nullptr;
        driver().GetErrorString(cr, &s);
        snprintf(err, errlen, "loading the JIT module failed: %s", s ? s : "?");
        return -1;
    }
    g_cache[key] = c;
    out->fn = (void*)c.fn;
    out->qhist = doQhist;
    return 0;
}

int fpl_jit_launch_scan(const FplJitKernel* k, const DevBatch& b, ReadState* st, cudaStream_t stream) {
    if (b.n_reads == 0) return 0;
    const uint8_t* seq = b.seq;
    const uint8_t* qual = b.qual;
    const int64_t* offsets = b.offsets;
    int64_t n = b.n_reads;
    // `one` is the multiplier of the IMADs that must stay IMADs (an add the compiler cannot see through stays on the
    // FMA pipe); version 1 ignores the extra argument.  The histogram inputs (qhist) ride in the ReadState (k_trim).
    unsigned one = 1;
    void* args[] = {(void*)&seq, (void*)&qual, (void*)&offsets, (void*)&st, (void*)&n, (void*)&one};
    // one CTA per read: the hardware scheduler balances the gamma-distributed read lengths better than persistent CTAs
    // walking the reads round-robin.
    CUresult cr = driver().LaunchKernel((CUfunction)k->fn, (unsigned)b.n_reads, 1, 1, 128, 1, 1, 0, (CUstream)stream, args, nullptr);
    return cr == CUDA_SUCCESS ? 0 : -1;
}
