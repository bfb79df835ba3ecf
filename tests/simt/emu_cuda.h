// TEST INFRASTRUCTURE: a small SIMT emulator so that the CPU suite can EXECUTE the kernels of libfplgpu (their source text,
// preprocessed by tests/simt_emu.py) against the oracle.  One OS thread; every CUDA thread of a block is a fiber (ucontext);
// a warp-level or block-level collective (__shfl_*_sync, __ballot_sync, __reduce_*_sync, __syncwarp, __syncthreads) parks the
// fiber until every live thread of the warp / block has arrived, then hands all of them the gathered values.  That is the
// contract the kernels rely on (full masks, convergent call sites); a collective that not all live lanes reach is reported
// as a deadlock instead of returning garbage.  Device memory is host memory; atomics are plain operations (one OS thread);
// __shared__ variables become function-local statics (one block runs at a time).  Timing, caches, bank conflicts, memory
// ordering between warps are NOT modelled: this checks what the code computes, not how fast or how safely it races.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <limits.h>
#include <ucontext.h>
#include <functional>
#include <type_traits>
#include <vector>

struct uint3 { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint4 { uint32_t x, y, z, w; };
struct uint2 { uint32_t x, y; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 v = {x, y, z, w}; return v; }
static inline uint2 make_uint2(uint32_t x, uint32_t y) { uint2 v = {x, y}; return v; }
typedef void* cudaStream_t;

#define __device__
#define __global__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __shared__ static
#define __constant__ static
#define __grid_constant__
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

extern uint3 emu_threadIdx, emu_blockIdx;
extern dim3 emu_blockDim, emu_gridDim;
#define threadIdx emu_threadIdx
#define blockIdx emu_blockIdx
#define blockDim emu_blockDim
#define gridDim emu_gridDim

namespace emu {
struct Group {             // a warp or a block: the live threads that must all reach a collective
    uint64_t slot[1024], res[1024];
    unsigned long long in_lo = 0;      // (warp) bit mask of the lanes that took part
    unsigned res_mask = 0;
    int arrived = 0, alive = 0;
    unsigned gen = 0;
};
void yield();
void note_progress();      // a waiting fiber's condition may have changed without a collective completing (mbarrier emulation)
Group& warp();
Group& block();
int lane();
int tid_in_block();
// deposit v, wait for the group, return the group's generation result (res[], res_mask valid until the next collective)
Group& collect(Group& g, int index, uint64_t v);
void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body);
void note_launch(const char* call);     // counts a launch under its kernel's name (emu_core.cpp: emu_launches)
extern long long collectives;
extern unsigned long long block_serial;      // counts the blocks run so far (per-thread emulation state resets on a new block)
extern uint8_t* dynamic_smem;          // `extern __shared__` of the running kernel
// 32-bit "shared window" addresses (what cvta.to.shared yields on the device): a 16 MB window per region of host memory
uint32_t to_shared(const void* p);
void* from_shared(uint32_t a);
}  // namespace emu

// ---- warp collectives (full masks only: the kernels never pass anything else) ----
template <class T> static inline uint64_t emu_bits(T v) { uint64_t b = 0; memcpy(&b, &v, sizeof(T)); return b; }
template <class T> static inline T emu_unbits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
#define EMU_FULL(mask) do { if ((mask) != 0xffffffffu) { fprintf(stderr, "emu: partial mask %x\n", (unsigned)(mask)); abort(); } } while (0)

template <class T> static inline T __shfl_sync(unsigned mask, T v, int src) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), emu_bits(v));
    return emu_unbits<T>(g.res[src & 31]);
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned d) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), emu_bits(v));
    const int l = emu::lane();
    return l >= (int)d ? emu_unbits<T>(g.res[l - d]) : v;
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned d) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), emu_bits(v));
    const int l = emu::lane();
    return l + (int)d < 32 ? emu_unbits<T>(g.res[l + d]) : v;
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int x) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), emu_bits(v));
    return emu_unbits<T>(g.res[(emu::lane() ^ x) & 31]);
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), pred ? 1u : 0u);
    unsigned b = 0;
    for (int i = 0; i < 32; i++) if ((g.res_mask >> i & 1u) && g.res[i]) b |= 1u << i;
    return b;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), pred ? 1u : 0u);
    for (int i = 0; i < 32; i++) if ((g.res_mask >> i & 1u) && !g.res[i]) return 0;
    return 1;
}
static inline void __syncwarp(unsigned mask = 0xffffffffu) { EMU_FULL(mask); emu::collect(emu::warp(), emu::lane(), 0); }
template <class T, class F> static inline T emu_reduce(unsigned mask, T v, F f) {
    EMU_FULL(mask);
    emu::Group& g = emu::collect(emu::warp(), emu::lane(), emu_bits(v));
    bool first = true;
    T acc = v;
    for (int i = 0; i < 32; i++) if (g.res_mask >> i & 1u) { T x = emu_unbits<T>(g.res[i]); acc = first ? x : f(acc, x); first = false; }
    return acc;
}
static inline int __reduce_add_sync(unsigned m, int v) { return emu_reduce(m, v, [](int a, int b) { return (int)((unsigned)a + (unsigned)b); }); }
static inline unsigned __reduce_add_sync(unsigned m, unsigned v) { return emu_reduce(m, v, [](unsigned a, unsigned b) { return a + b; }); }
static inline int __reduce_min_sync(unsigned m, int v) { return emu_reduce(m, v, [](int a, int b) { return a < b ? a : b; }); }
static inline unsigned __reduce_min_sync(unsigned m, unsigned v) { return emu_reduce(m, v, [](unsigned a, unsigned b) { return a < b ? a : b; }); }
static inline int __reduce_max_sync(unsigned m, int v) { return emu_reduce(m, v, [](int a, int b) { return a > b ? a : b; }); }
static inline unsigned __reduce_max_sync(unsigned m, unsigned v) { return emu_reduce(m, v, [](unsigned a, unsigned b) { return a > b ? a : b; }); }
static inline unsigned __reduce_or_sync(unsigned m, unsigned v) { return emu_reduce(m, v, [](unsigned a, unsigned b) { return a | b; }); }
static inline unsigned __reduce_and_sync(unsigned m, unsigned v) { return emu_reduce(m, v, [](unsigned a, unsigned b) { return a & b; }); }
// ---- block collectives ----
static inline void __syncthreads() { emu::collect(emu::block(), emu::tid_in_block(), 0); }
static inline int __syncthreads_count(int pred) {
    emu::Group& g = emu::collect(emu::block(), emu::tid_in_block(), pred ? 1u : 0u);
    int n = 0;
    for (unsigned i = 0; i < emu_blockDim.x; i++) n += g.res[i] != 0;     // exited threads left 0 behind
    return n;
}

// ---- scalar intrinsics ----
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i); return r; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)(((((unsigned long long)hi) << 32) | lo) >> (sh & 31)); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)((((((unsigned long long)hi) << 32) | lo) << (sh & 31)) >> 32); }
static inline unsigned __dp4a(unsigned a, unsigned b, unsigned c) { for (int i = 0; i < 4; i++) c += ((a >> (8 * i)) & 0xFFu) * ((b >> (8 * i)) & 0xFFu); return c; }
static inline int __dp4a(int a, int b, int c) { for (int i = 0; i < 4; i++) c += (int)(int8_t)((unsigned)a >> (8 * i)) * (int)(int8_t)((unsigned)b >> (8 * i)); return c; }
static inline unsigned __dp4a(unsigned a, unsigned b, int c) { return __dp4a(a, b, (unsigned)c); }
template <class A, class B> static inline typename std::common_type<A, B>::type min(A a, B b) { typedef typename std::common_type<A, B>::type T; return (T)a < (T)b ? (T)a : (T)b; }
template <class A, class B> static inline typename std::common_type<A, B>::type max(A a, B b) { typedef typename std::common_type<A, B>::type T; return (T)a > (T)b ? (T)a : (T)b; }
// ---- atomics (one OS thread: plain read-modify-write, old value returned) ----
template <class T, class U> static inline T atomicAdd(T* p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicSub(T* p, U v) { T o = *p; *p = (T)(o - (T)v); return o; }
template <class T, class U> static inline T atomicOr(T* p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> static inline T atomicAnd(T* p, U v) { T o = *p; *p = (T)(o & (T)v); return o; }
template <class T, class U> static inline T atomicMin(T* p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMax(T* p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicExch(T* p, U v) { T o = *p; *p = (T)v; return o; }
template <class T, class U, class V> static inline T atomicCAS(T* p, U cmp, V v) { T o = *p; if (o == (T)cmp) *p = (T)v; return o; }

// KERNEL<<<grid, block, smem, stream>>>(args) is rewritten by tests/simt_emu.py into EMU_LAUNCH(grid, block, smem, KERNEL(args))
#define EMU_LAUNCH(grid, block, smem, ...) \
    (emu::note_launch(#__VA_ARGS__), emu::launch(dim3(grid), dim3(block), (size_t)(smem), [&]() { __VA_ARGS__; }))
