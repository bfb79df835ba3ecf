// TEST INFRASTRUCTURE: <cuda_runtime.h> for the emulated build of libfplgpu (tests/simt_emu.py: build_library).  Device memory
// is host memory, streams run synchronously, events are timestamps; kernels run under the SIMT emulator (../emu_cuda.h).
#pragma once
#include "../emu_cuda.h"
#include <time.h>

enum cudaError_t { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorInvalidResourceHandle = 400,
                   cudaErrorNotReady = 600 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct EmuEvent;
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
// Streams and events are ids that are never reused, kept by emu_core.cpp (an event with its timestamp): emu_live_handles counts the
// live ones; emu::fail_handle_in = k > 0 makes the k-th creation from now fail, once, and write EMU_POISON as the handle
// (emu_fail_handle); a call that gets a handle that is not live (poison, destroyed) fails and counts in emu_bad_handles.  The null
// stream is the default stream.
enum { EMU_STREAM = 1, EMU_EVENT = 2, EMU_TIMING_EVENT = 3 };
#define EMU_POISON ((void*)0xBADBAD0)
namespace emu {
void* handle_new(int kind);             // nullptr: this creation fails
double* handle(const void* h);          // the live handle's timestamp; nullptr (and counted) when h is not live
bool handle_free(const void* h);
}  // namespace emu
template <class H> static inline cudaError_t emu_create(H* h, int kind) {
    void* p = emu::handle_new(kind);
    *h = (H)(p ? p : EMU_POISON);
    return p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline bool emu_stream_ok(cudaStream_t s) { return !s || emu::handle(s); }
#define EMU_CHECK_STREAM(s) do { if (!emu_stream_ok(s)) return cudaErrorInvalidResourceHandle; } while (0)
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t st = nullptr) {
    EMU_CHECK_STREAM(st);
    if (n) memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind,
                                            cudaStream_t st = nullptr) {
    EMU_CHECK_STREAM(st);
    for (size_t r = 0; r < height; r++) memmove((char*)d + r * dpitch, (const char*)s + r * spitch, width);
    return cudaSuccess;
}
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st = nullptr) {
    EMU_CHECK_STREAM(st);
    if (n) memset(d, v, n);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { return emu_create(s, EMU_STREAM); }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { return emu_create(s, EMU_STREAM); }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { return s && emu::handle_free(s) ? cudaSuccess : cudaErrorInvalidResourceHandle; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t s) { EMU_CHECK_STREAM(s); return cudaSuccess; }
static inline double emu_now_ms() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { return emu_create(e, EMU_TIMING_EVENT); }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned flags) {
    return emu_create(e, flags & cudaEventDisableTiming ? EMU_EVENT : EMU_TIMING_EVENT);
}
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { return emu::handle_free(e) ? cudaSuccess : cudaErrorInvalidResourceHandle; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s = nullptr) {
    double* t = emu::handle(e);
    EMU_CHECK_STREAM(s);
    if (!t) return cudaErrorInvalidResourceHandle;
    *t = emu_now_ms();
    return cudaSuccess;
}
static inline cudaError_t cudaEventSynchronize(cudaEvent_t e) { return emu::handle(e) ? cudaSuccess : cudaErrorInvalidResourceHandle; }
static inline cudaError_t cudaEventQuery(cudaEvent_t e) { return emu::handle(e) ? cudaSuccess : cudaErrorInvalidResourceHandle; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
    const double *ta = emu::handle(a), *tb = emu::handle(b);
    if (!ta || !tb) return cudaErrorInvalidResourceHandle;
    *ms = (float)(*tb - *ta);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned = 0) {
    const bool ok = emu::handle(e) != nullptr;
    EMU_CHECK_STREAM(s);
    return ok ? cudaSuccess : cudaErrorInvalidResourceHandle;
}
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
