// TEST INFRASTRUCTURE: <cuda_runtime.h> for the emulated build of libfplgpu (tests/simt_emu.py: build_library).  Device memory
// is host memory, streams run synchronously, events are timestamps; kernels run under the SIMT emulator (../emu_cuda.h).
#pragma once
#include "../emu_cuda.h"
#include <time.h>

enum cudaError_t { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNotReady = 600 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct EmuEvent { double t; };
typedef EmuEvent* cudaEvent_t;
static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated runtime error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int d) { return d == 0 ? cudaSuccess : cudaErrorInvalidValue; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
// cudaMalloc does not zero memory: EMU_MALLOC_FILL=<byte> fills every allocation with that byte (default 0), so that a kernel or
// host path leaning on fresh allocations being zero shows up.  emu::live_allocs counts the cudaMalloc / cudaMallocHost blocks not
// yet freed; emu::fail_alloc_in = k > 0 makes the k-th allocation from now fail, once (emu_core.cpp: emu_live_allocs, emu_fail_alloc).
namespace emu { extern long long live_allocs, fail_alloc_in; }
static inline void* emu_alloc(size_t n) {
    if (emu::fail_alloc_in > 0 && --emu::fail_alloc_in == 0) return nullptr;
    static const char* f = getenv("EMU_MALLOC_FILL");
    void* p = malloc(n ? n : 1);
    if (p) { memset(p, f ? (int)strtol(f, nullptr, 0) : 0, n ? n : 1); emu::live_allocs++; }
    return p;
}
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { *p = (T*)emu_alloc(n); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <class T> static inline cudaError_t cudaMallocHost(T** p, size_t n) { *p = (T*)emu_alloc(n); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFree(void* p) { if (p) { emu::live_allocs--; free(p); } return cudaSuccess; }
static inline cudaError_t cudaFreeHost(void* p) { if (p) { emu::live_allocs--; free(p); } return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind,
                                            cudaStream_t = nullptr) {
    for (size_t r = 0; r < height; r++) memmove((char*)d + r * dpitch, (const char*)s + r * spitch, width);
    return cudaSuccess;
}
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline double emu_now_ms() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new EmuEvent{0}; return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = new EmuEvent{0}; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = emu_now_ms(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t - a->t); return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }

// ---- host forms of the PTX wrappers (their definitions are cut out of fpl_device.cuh / fpl_stats.cu) ----
static inline uint32_t shared_addr(const void* p) { return emu::to_shared(p); }
static inline void red_shared_add(uint32_t a, uint32_t v) { *(uint32_t*)emu::from_shared(a) += v; }
template <int IMM> static inline void red_shared_add_imm(uint32_t a, uint32_t v) { *(uint32_t*)emu::from_shared(a + (uint32_t)IMM) += v; }
static inline uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {       // prmt.b32, default mode
    const uint64_t src = ((uint64_t)b << 32) | a;
    uint32_t d = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t c = (sel >> (4 * i)) & 0xF;
        uint32_t byte = (uint32_t)(src >> (8 * (c & 7))) & 0xFF;
        if (c & 8) byte = (byte & 0x80) ? 0xFF : 0x00;
        d |= byte << (8 * i);
    }
    return d;
}
static inline uint4 lds128(uint32_t a) { uint4 v; memcpy(&v, emu::from_shared(a), 16); return v; }
static inline uint32_t lds32(uint32_t a) { uint32_t v; memcpy(&v, emu::from_shared(a), 4); return v; }
namespace emu {      // cp.async / mbarrier emulation (emu_ptx.cpp)
void cp_async(uint32_t dst, const void* src, int n, int size);
void cp_commit();
void cp_wait(int n_pending);
void mbar_init(uint32_t bar);
void mbar_expect(uint32_t bar, uint32_t bytes);
void mbar_wait(uint32_t bar, uint32_t parity);
void bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar);
}  // namespace emu
static inline void cp_async16(uint32_t dst, const void* src, int n) { emu::cp_async(dst, src, n, 16); }
static inline void cp_async4(uint32_t dst, const void* src, int n) { emu::cp_async(dst, src, n, 4); }
static inline void cp_async_commit() { emu::cp_commit(); }
template <int N> static inline void cp_async_wait() { emu::cp_wait(N); }
static inline void mbar_init(uint32_t bar, uint32_t) { emu::mbar_init(bar); }
static inline void mbar_expect_tx(uint32_t bar, uint32_t bytes) { emu::mbar_expect(bar, bytes); }
static inline void mbar_wait(uint32_t bar, uint32_t parity) { emu::mbar_wait(bar, parity); }
static inline void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) { emu::bulk(dst, src, bytes, bar); }
