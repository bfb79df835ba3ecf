// Ownership of CUDA resources for the host side of the library: DevBuf<T> owns one cudaMalloc allocation and frees it when it
// goes, and its growth methods are the library's only allocation policies.  Kernels and the by-value descriptors (DevBatch,
// EmitSource, ReportCurves, HtmlText, MergeSrc) take the raw pointer.  Growth returns the CUDA error, so each module keeps
// its own way of reporting it.  Streams, events and pinned host blocks have owners of their own (Owned, at the end).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <memory>
#include <type_traits>
#include <utility>

// a CUDA call in a function that reports into the caller's (err, errlen) buffer
#define FPL_CK_ERR(call)                                                                                         \
    do {                                                                                                       \
        cudaError_t e_ = (call);                                                                               \
        if (e_ != cudaSuccess) { snprintf(err, errlen, "%s failed: %s", #call, cudaGetErrorString(e_)); return -1; } \
    } while (0)

#define FPL_FIRST_BYTES (1 << 16)       // first capacity of a doubling buffer

template <class T>
class DevBuf {
public:
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept { swap(o); }
    DevBuf& operator=(DevBuf&& o) noexcept { DevBuf(std::move(o)).swap(*this); return *this; }
    ~DevBuf() { reset(); }

    operator T*() const { return p_; }
    T* get() const { return p_; }
    int64_t bytes() const { return bytes_; }
    void swap(DevBuf& o) noexcept { std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); }
    void reset() {
        if (p_) cudaFree(p_);
        p_ = nullptr; bytes_ = 0;
    }

    // Room for n elements, contents discarded: the byte capacity doubles, from first_bytes or from what it is, until it
    // covers them.  Geometric, so the wait of cudaFree is rare.
    cudaError_t grow(int64_t n, int64_t first_bytes = FPL_FIRST_BYTES) {
        const int64_t need = (int64_t)sizeof(T) * n;
        return need <= bytes_ ? cudaSuccess : alloc(doubled(need, first_bytes));
    }
    // Room for exactly n elements when it holds fewer, contents discarded.
    cudaError_t grow_exact(int64_t n) {
        const int64_t need = (int64_t)sizeof(T) * n;
        return need <= bytes_ ? cudaSuccess : alloc(need);
    }
    // grow(n), the first `keep` elements kept: copied on stream s, which is synchronised before the old block is freed.  On
    // failure the buffer is as it was.
    cudaError_t grow_keep(int64_t n, int64_t keep, cudaStream_t s, int64_t first_bytes = FPL_FIRST_BYTES) {
        const int64_t need = (int64_t)sizeof(T) * n;
        if (need <= bytes_) return cudaSuccess;
        DevBuf nb;
        cudaError_t e = nb.alloc(doubled(need, first_bytes));
        if (e == cudaSuccess && keep) e = cudaMemcpyAsync(nb.p_, p_, sizeof(T) * keep, cudaMemcpyDeviceToDevice, s);
        if (e == cudaSuccess && p_) e = cudaStreamSynchronize(s);
        if (e == cudaSuccess) swap(nb);
        return e;                       // nb frees the old block, or the new one
    }

private:
    int64_t doubled(int64_t need, int64_t first_bytes) const {
        int64_t c = bytes_ ? bytes_ : first_bytes;
        while (c < need) c *= 2;
        return c;
    }
    cudaError_t alloc(int64_t n_bytes) {
        reset();
        cudaError_t e = cudaMalloc(&p_, (size_t)n_bytes);
        if (e == cudaSuccess) bytes_ = n_bytes;
        else p_ = nullptr;
        return e;
    }
    T* p_ = nullptr;
    int64_t bytes_ = 0;
};

// cub's two-phase call: call(nullptr, bytes) asks for the temporary storage, `tmp` grows (DevBuf::grow) to that + 256,
// call(tmp, bytes) runs.  call: (void* d_temp, size_t& bytes) -> cudaError_t.
template <class F>
cudaError_t cub_call(DevBuf<uint8_t>& tmp, F&& call, int64_t first_bytes = FPL_FIRST_BYTES) {
    size_t bytes = 0;
    cudaError_t e = call(nullptr, bytes);
    if (e == cudaSuccess) e = tmp.grow((int64_t)bytes + 256, first_bytes);
    if (e == cudaSuccess) e = call(tmp.get(), bytes);
    return e;
}

// A unique_ptr whose deleter releases the handle H, handed to CUDA calls as the raw handle (as DevBuf hands out its pointer).
// The create_* calls below give an owner its handle only when the creation succeeded.
template <class H, class Release>
struct Owned : std::unique_ptr<std::remove_pointer_t<H>, Release> {
    operator H() const { return this->get(); }
};
struct StreamRelease { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct EventRelease { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct PinnedRelease { void operator()(void* p) const { cudaFreeHost(p); } };
using Stream = Owned<cudaStream_t, StreamRelease>;
using Event = Owned<cudaEvent_t, EventRelease>;
template <class T> using PinnedHost = Owned<T*, PinnedRelease>;

// a non-blocking stream
inline cudaError_t create_stream(Stream& s) {
    cudaStream_t h;
    cudaError_t e = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking);
    if (e == cudaSuccess) s.reset(h);
    return e;
}
// timing: an event cudaEventElapsedTime can read; otherwise one that only orders work (cudaEventDisableTiming)
inline cudaError_t create_event(Event& ev, bool timing) {
    cudaEvent_t h;
    cudaError_t e = timing ? cudaEventCreate(&h) : cudaEventCreateWithFlags(&h, cudaEventDisableTiming);
    if (e == cudaSuccess) ev.reset(h);
    return e;
}
// n elements of pinned host memory
template <class T>
cudaError_t create_pinned(PinnedHost<T>& p, size_t n) {
    T* h;
    cudaError_t e = cudaMallocHost(&h, sizeof(T) * n);
    if (e == cudaSuccess) p.reset(h);
    return e;
}
