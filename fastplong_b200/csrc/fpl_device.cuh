// Shared device-side definitions for libfplgpu.so (sm_90a).  See DESIGN.md for the kernel map.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fplgpu.h"

#define FPL_NUM_SMS 132      // H100 SXM: the grid caps of the grid-stride kernels are multiples of it

#define FPL_WINDOW 200       // AdapterTrimmer WINDOW (src/adaptertrimmer.cpp:169,239)
#define FPL_PATTERN_LEN 16   // AdapterTrimmer PATTERN_LEN (:170,240)

// Kernel parameter block: the options POD + device tables built once per context.
struct DevParams {
    fpl_options opt;
    int n_adapters;
    const uint8_t* adapters;  // [n][FPL_MAX_ADAPTER_LEN] adapter bytes
    const int* alen;          // [n]
    const uint4* peq;         // [n][256]: 128-bit match mask of the whole adapter for every byte value
    const uint32_t* peq16;    // [n][2][256]: [0] = match masks of the first plen chars, [1] = of the last plen chars
    const uint32_t* acode;    // [n][4]: 2-bit codes ((byte>>1)&3 at bit 2i) lo/hi + position mask lo/hi; mask == 0: not ACGT-only or > 32 bp
    short thr[FPL_MAX_ADAPTER_LEN + 1];  // thr(n) = (int)round(ed_max*n), tabulated on the host with libm round
    const int* pf_order;      // [n - 2]: the FASTA adapters' indices sorted by pre-filter width class (<= 32 bp, <= 64 bp, longer)
    const unsigned long long* peq_long;  // [n][256][peq_words]: match masks of adapters longer than 128 bp (else nullptr)
    int peq_words;            // 64-bit words per mask in peq_long
    int small_adapters;       // size class of -s / -e: 0 both <= 32 bp, 1 both <= 64 bp, 2 any (k_trim<CLS>)
    int fasta_class;          // the same for the FASTA adapters (k_trim_fasta<CLS>)
    uint32_t one;             // 1: the multiplier of the IMADs that must stay on the FMA pipe (an add the compiler cannot fold)
    unsigned long long* qstripes;   // k_scan_jit's histogram sums (k_trim hands the address on in the ReadState), else nullptr
};

// Device view of a packed batch.
struct DevBatch {
    const uint8_t* seq;
    const uint8_t* qual;
    const int64_t* offsets;
    const int32_t* lens;
    int64_t n_reads;
};

// Per-read state handed from kernel to kernel (SoA would save little: it is 64 B/read, ~0.4% of the payload).
struct ReadState {
    int32_t lo, len;          // r1 window after trimAndCut / polyX / adapter trims
    uint32_t alive;           // 0 if dropped by trimAndCut
    uint32_t pad;             // k_scan_jit with the quality histograms: the read's median quality char
    unsigned long long best[2];   // middle-adapter scan: (minHamming << 32) | pos, ~0ull = no position scanned
    int32_t lowq, nn, totalq, diff;  // passFilter counts over the window
    int32_t reserved[4];      // k_scan_jit with the quality histograms: [0] the window's median quality char (out);
                              // [1] the read's length, [2..3] DevParams::qstripes (in, written by k_trim)
};

// A segment to be fed to the Stats kernels: absolute byte offset into the batch buffers + length (0 = skip).
struct StatSeg {
    int64_t off;
    int32_t len;
    int32_t read;   // owning read (for writing the median back), -1 = none
    int32_t slot;   // 0/1: which seg_median_qual slot, 2 = pre_median_qual
    int32_t pad;
};

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// Shared-memory reduction (no return value) on a 32-bit shared-window address: avoids the generic-address
// conversion the compiler emits around atomicAdd(&smem[i], v) and never needs a convergence barrier.
__device__ __forceinline__ void red_shared_add(uint32_t saddr, uint32_t v) {
    asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t shared_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ int warp_incl_scan(int v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane_id() >= d) v += t;
    }
    return v;
}

// Myers/Hyyro bit-parallel Levenshtein, global alignment, with the m-bit pattern held in the TOP m bits of the word:
// the last row's horizontal deltas are then bit 31 of HP / HN (one shift each to count them) and the bits below the
// pattern stay inert (VP = VN = 0, HP = all ones there; the +1 that enters row 0 comes in at bit 0 of the word and the
// ones below the pattern carry it up).  Left shifts are multiplies (IMAD pipe).  9 logic-pipe ops per column.
struct Myers32 {
    uint32_t VP, VN, accP, accN;
    __device__ __forceinline__ void init(int m) {
        VP = m >= 32 ? 0xFFFFFFFFu : ~(0xFFFFFFFFu >> m);
        VN = 0; accP = 0; accN = 0;
    }
    // Eq: match mask of this text byte, already in the top m bits
    __device__ __forceinline__ void column(uint32_t Eq) {
        const uint32_t Xv = Eq | VN;
        const uint32_t Xh = (((Eq & VP) + VP) ^ VP) | Eq;
        uint32_t HP = VN | ~(Xh | VP);
        uint32_t HN = VP & Xh;
        accP += HP >> 31;
        accN += HN >> 31;
        asm("mad.lo.u32 %0, %1, 2, 1;" : "=r"(HP) : "r"(HP));
        asm("mad.lo.u32 %0, %1, 2, 0;" : "=r"(HN) : "r"(HN));
        VP = HN | ~(Xv | HP);
        VN = HP & Xv;
    }
    __device__ __forceinline__ int score(int m) const { return m + (int)accP - (int)accN; }
};
// table word -> top-aligned match mask of pattern bits [shift, shift + m)
__device__ __forceinline__ uint32_t myers_eq_top(uint32_t w, int shift, int m) {
    uint32_t e = w >> shift, d;
    const uint32_t mul = m >= 32 ? 1u : (1u << (32 - m));
    asm("mad.lo.u32 %0, %1, %2, 0;" : "=r"(d) : "r"(e), "r"(mul));
    return d;
}

// Two distances at once, one per half-warp (lanes 0-15: problem 0, lanes 16-31: problem 1), each with n <= 32 text bytes
// and an m <= 32 bit pattern; a half whose `on` is false idles through the same instructions.  Every lane returns its
// own half's distance.  Must be called by all 32 lanes.
__device__ __forceinline__ int myers32_halves(const uint8_t* text, int n, const uint4* peq, int m, bool on) {
    const int lane = threadIdx.x & 31, hl = lane & 15, base = lane & 16;
    uint32_t e0 = 0, e1 = 0;            // match masks of text bytes hl and hl + 16
    if (on && hl < n) e0 = myers_eq_top(__ldg(&peq[text[hl]].x), 0, m);
    if (on && hl + 16 < n) e1 = myers_eq_top(__ldg(&peq[text[hl + 16]].x), 0, m);
    const int nmax = max(__shfl_sync(0xffffffffu, on ? n : 0, 0), __shfl_sync(0xffffffffu, on ? n : 0, 16));
    Myers32 M;
    M.init(m);
    for (int i = 0; i < nmax; i++) {
        const uint32_t Eq = __shfl_sync(0xffffffffu, i < 16 ? e0 : e1, base + (i & 15));
        if (i < n) M.column(Eq);
    }
    return M.score(m);
}

// myers32 for a whole warp that wants ONE distance (n <= 32 text bytes): lane i fetches the match mask of text byte i,
// so the two dependent loads per column happen once, side by side, instead of n times in a row; every lane then runs
// the recurrence on shuffled masks and returns the same value.  Must be called by all 32 lanes.
__device__ __forceinline__ int myers32_warp(const uint8_t* text, int n, const uint4* peq, int shift, int m) {
    if (m == 0) return n;
    if (n == 0) return m;
    const int lane = threadIdx.x & 31;
    uint32_t mine = 0;
    if (lane < n) mine = myers_eq_top(__ldg(&peq[text[lane]].x), shift, m);
    Myers32 M;
    M.init(m);
    for (int i = 0; i < n; i++) M.column(__shfl_sync(0xffffffffu, mine, i));
    return M.score(m);
}

// Levenshtein distance (Myers/Hyyro bit-parallel, global), pattern = adapter bits [shift, shift+m) with
// shift+m <= 32, text = n read bytes.  Exact, == edit_distance() of src/editdistance.cpp:100-126.
__device__ __forceinline__ int myers32(const uint8_t* text, int n, const uint4* peq, int shift, int m) {
    if (m == 0) return n;
    if (n == 0) return m;
    Myers32 M;
    M.init(m);
#pragma unroll 4
    for (int i = 0; i < n; i++) M.column(myers_eq_top(__ldg(&peq[text[i]].x), shift, m));
    return M.score(m);
}

// Levenshtein distance for adapters longer than 128 bp: Myers/Hyyro in 64-bit blocks with the horizontal delta carried
// from block to block (global distance: +1 enters the first block in every column).  Pattern = adapter bits
// [shift, shift + m), m <= FPL_MAX_ADAPTER_LEN; exact, == edit_distance() of src/editdistance.cpp:100-126 (which switches
// to its own multi-block form at 64 bp and to a plain DP beyond 640).  One call per lane; rare, not tuned.
static __device__ __noinline__ int myers_long(const uint8_t* text, int n, const unsigned long long* peq, int words, int shift, int m) {
    if (m == 0) return n;
    if (n == 0) return m;
    constexpr int MAXB = FPL_MAX_ADAPTER_LEN / 64;
    unsigned long long VP[MAXB], VN[MAXB];
    const int nb = (m + 63) >> 6;
    const int lastbits = m - 64 * (nb - 1);
    for (int b = 0; b < nb; b++) { VP[b] = ~0ull; VN[b] = 0; }
    if (lastbits < 64) VP[nb - 1] = (1ull << lastbits) - 1;
    const unsigned long long lasttop = 1ull << (lastbits - 1);
    const int w0 = shift >> 6, sh = shift & 63;
    int score = m;
    for (int i = 0; i < n; i++) {
        const unsigned long long* e = peq + (size_t)text[i] * words;
        int hin = 1;
        for (int b = 0; b < nb; b++) {
            unsigned long long Eq = __ldg(&e[w0 + b]) >> sh;
            if (sh && w0 + b + 1 < words) Eq |= __ldg(&e[w0 + b + 1]) << (64 - sh);
            const bool last = b == nb - 1;
            if (last && lastbits < 64) Eq &= (1ull << lastbits) - 1;
            const unsigned long long Pv = VP[b], Mv = VN[b];
            const unsigned long long Xv = Eq | Mv;
            if (hin < 0) Eq |= 1ull;
            const unsigned long long Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
            unsigned long long Ph = Mv | ~(Xh | Pv);
            unsigned long long Mh = Pv & Xh;
            const unsigned long long top = last ? lasttop : (1ull << 63);
            const int hout = (Ph & top) ? 1 : (Mh & top) ? -1 : 0;
            Ph <<= 1; Mh <<= 1;
            if (hin < 0) Mh |= 1ull; else if (hin > 0) Ph |= 1ull;
            VP[b] = Mh | ~(Xv | Ph);
            VN[b] = Ph & Xv;
            if (last && lastbits < 64) { VP[b] &= (1ull << lastbits) - 1; VN[b] &= (1ull << lastbits) - 1; }
            hin = hout;
        }
        score += hin;
    }
    return score;
}

