// k_scan_fast: bit-sliced version of the per-base "adapter + quality" pass (same contract as k_scan in fpl_scan.cu,
// selected by the host when both -s/-e adapters are non-empty, ACGT-only and <= 128 bp).
//
// Data layout per warp-tile: 32 lanes x 32 consecutive bytes (two 16-byte vector loads per lane, coalesced).
//   1. each lane turns its 32 sequence bytes into five 32-bit bit-planes (bits 0..4 of every byte; one
//      AND + IMAD + funnel-shift per word per plane) and checks (b & 0xE0) == 0x40 for all of them (0x40..0x5F:
//      every upper-case letter).  Under that check the planes decide exactly which bytes are A, C, G, T (plane V),
//      their 2-bit code (HI = bit 1, LO = bit 2) and which are 'N'.  Lanes holding any other byte take a per-byte path.
//   2. adapter letter a_i matches read position p+i iff V & (HI == h_i) & (LO == l_i) there: three funnel shifts by
//      the static amount i (shared by both adapters) and two LOP3 whose third operands h_i / l_i come straight from
//      the constant bank (ScanPlan.hm / lm), statically indexed because the loop over i is fully unrolled;
//   3. the alen one-bit match vectors are summed per position with carry-save adders (3:2 compressors are two LOP3
//      each, Harley-Seal blocks of 8) into a bit-sliced match counter; H(p) = alen - matches(p);
//   4. a bit-sliced arg-max (MSB-first candidate narrowing) gives each lane its best position of the tile; the
//      first arg-min of the whole read falls out of a (H << 32 | pos) min-reduction (strict '<' of
//      src/adaptertrimmer.cpp:148 == smallest position among equal H).
// Quality bytes: sum via dp4a, #(q < qualified) via one SWAR compare per word; N count = popcount of the N plane;
// the complexity count compares each word with itself shifted by one byte.
#include "fpl_device.cuh"
#include "fpl_scanplan.h"
#include "fpl_scan.h"

#define SF_WARPS 4
#define SF_THREADS (SF_WARPS * 32)

namespace {

// carry-save adder: (h, l) = a + b + c per bit position (two LOP3)
#define CSA(h, l, a, b, c)                       \
    do {                                         \
        const uint32_t a_ = (a), b_ = (b), c_ = (c); \
        l = a_ ^ b_ ^ c_;                        \
        h = (a_ & b_) | (c_ & (a_ | b_));        \
    } while (0)

__device__ __forceinline__ uint32_t plane_nibble(uint32_t w, uint32_t mask, uint32_t mul) { return (w & mask) * mul; }

// exact per-byte "non-zero" flags in bit 7 of every byte
__device__ __forceinline__ uint32_t nz7(uint32_t d) { return (((d & 0x7f7f7f7fu) + 0x7f7f7f7fu) | d) & 0x80808080u; }

struct LaneSeq { uint32_t w[8]; };

__device__ __forceinline__ void load32(const uint8_t* p, bool ok, LaneSeq& s) {
    if (ok) {
        const uint4* v = reinterpret_cast<const uint4*>(p);
        uint4 a = __ldg(v), b = __ldg(v + 1);
        s.w[0] = a.x; s.w[1] = a.y; s.w[2] = a.z; s.w[3] = a.w;
        s.w[4] = b.x; s.w[5] = b.y; s.w[6] = b.z; s.w[7] = b.w;
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) s.w[k] = 0;
    }
}

// bit-sliced counter of matches for one adapter
template <int NPL>
struct Counter {
    uint32_t ones, twos, fours, hi[NPL > 3 ? NPL - 3 : 1];
    __device__ __forceinline__ void clear() {
        ones = twos = fours = 0;
#pragma unroll
        for (int b = 0; b < NPL - 3; b++) hi[b] = 0;
    }
    __device__ __forceinline__ void add8(const uint32_t (&x)[8]) {
        uint32_t twosA, twosB, foursA, foursB, eight;
        CSA(twosA, ones, ones, x[0], x[1]);
        CSA(twosB, ones, ones, x[2], x[3]);
        CSA(foursA, twos, twos, twosA, twosB);
        CSA(twosA, ones, ones, x[4], x[5]);
        CSA(twosB, ones, ones, x[6], x[7]);
        CSA(foursB, twos, twos, twosA, twosB);
        CSA(eight, fours, fours, foursA, foursB);
        uint32_t carry = eight;
#pragma unroll
        for (int b = 0; b < NPL - 3; b++) {
            const uint32_t t = hi[b] & carry;
            hi[b] ^= carry;
            carry = t;
        }
    }
    __device__ __forceinline__ uint32_t plane(int b) const { return b == 0 ? ones : b == 1 ? twos : b == 2 ? fours : hi[b - 3]; }
    // lane-local arg-max over the positions in `valid`, first position on ties
    __device__ __forceinline__ void argmax(uint32_t valid, int64_t pos0, int& bestM, int64_t& bestPos) const {
        if (!valid) return;
        uint32_t cand = valid;
        int val = 0;
#pragma unroll
        for (int b = NPL - 1; b >= 0; b--) {
            const uint32_t t = cand & plane(b);
            if (t) { cand = t; val |= 1 << b; }
        }
        if (val > bestM) { bestM = val; bestPos = pos0 + (__ffs(cand) - 1); }
    }
};

}  // namespace

template <int NPL, int HL>
__global__ void __launch_bounds__(SF_THREADS, 6)
k_scan_fast(const __grid_constant__ DevParams P, const __grid_constant__ ScanPlan plan, DevBatch b,
            ReadState* __restrict__ st) {
    __shared__ unsigned long long sh64[2][SF_WARPS];
    __shared__ int sh32[4][SF_WARPS];
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const int64_t r = blockIdx.x;
    const ReadState s = st[r];
    if (!s.alive) return;
    const int len = s.len;
    const int64_t start = b.offsets[r] + s.lo;            // absolute byte offset of the window
    const int pre = (int)(start & 15);                    // bytes between the 16-byte aligned base and the window
    const uint8_t* sbase = b.seq + (start - pre);
    const uint8_t* qbase = b.qual + (start - pre);
    const int alen0 = P.alen[0], alen1 = P.alen[1];
    const bool doAdapters = P.opt.adapter_enabled != 0;
    const bool doCounts = (P.opt.qual_filter_enabled || P.opt.length_filter_enabled);
    const bool doCplx = P.opt.complexity_enabled != 0;
    const uint32_t qq4 = (uint32_t)(P.opt.qualified_qual & 0x7f) * 0x01010101u;
    const int np0 = (doAdapters && alen0 <= len) ? len - alen0 : 0;
    const int np1 = (doAdapters && alen1 <= len) ? len - alen1 : 0;
    const int amax = max(alen0, alen1);
    const int step = (32 - HL) * 32;                      // bytes advanced per warp-tile
    const int total = pre + len;                          // bytes from the aligned base to the window end

    int bestM0 = -1, bestM1 = -1;
    int64_t bestP0 = 0, bestP1 = 0;
    int lowq_ge = 0, nn = 0, totalq = 0, diff = 0, nbytes = 0;

    for (int64_t t0 = (int64_t)wid * step; t0 < total; t0 += (int64_t)SF_WARPS * step) {
        const int64_t a0 = t0 + 32 * lane;                // this lane's first byte (relative to the aligned base)
        const bool inrange = a0 < total && a0 + 32 > pre;
        LaneSeq sq;
        load32(sbase + a0, inrange, sq);
        // ---- alphabet check + bit planes ----
        uint32_t bad = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) bad |= (sq.w[k] & 0xE0E0E0E0u) ^ 0x40404040u;
        uint32_t V, HI, LO, NM;
        if (bad == 0) {
            uint32_t B0 = 0, B1 = 0, B2 = 0, B3 = 0, B4 = 0;
#pragma unroll
            for (int k = 7; k >= 0; k--) {
                const uint32_t w = sq.w[k];
                B0 = __funnelshift_l(plane_nibble(w, 0x01010101u, 0x10204080u), B0, 4);
                B1 = __funnelshift_l(plane_nibble(w, 0x02020202u, 0x08102040u), B1, 4);
                B2 = __funnelshift_l(plane_nibble(w, 0x04040404u, 0x04081020u), B2, 4);
                B3 = __funnelshift_l(plane_nibble(w, 0x08080808u, 0x02040810u), B3, 4);
                B4 = __funnelshift_l(plane_nibble(w, 0x10101010u, 0x01020408u), B4, 4);
            }
            // bytes are 010 b4 b3 b2 b1 b0:  A 00001  C 00011  G 00111  T 10100  N 01110
            V = ~B3 & ((~B4 & B0 & (B1 | ~B2)) | (B4 & B2 & ~B1 & ~B0));
            HI = B1; LO = B2;
            NM = B3 & B2 & B1 & ~B0 & ~B4;
        } else {
            V = HI = LO = NM = 0;
            for (int j = 0; j < 32; j++) {
                const uint32_t ch = (sq.w[j >> 2] >> (8 * (j & 3))) & 0xFFu;
                const uint32_t bit = 1u << j;
                if (ch == 'A' || ch == 'C' || ch == 'G' || ch == 'T') {
                    V |= bit;
                    if (ch & 2u) HI |= bit;
                    if (ch & 4u) LO |= bit;
                }
                if (ch == 'N') NM |= bit;
            }
        }
        // ---- window masks for this lane: which of its 32 bytes are inside the window / are scan positions ----
        const int64_t p_first = a0 - pre;                 // window position of bit 0
        const bool mine = lane < 32 - HL;                 // halo lanes are re-processed by the next tile
        uint32_t inwin = 0, v0 = 0, v1 = 0;
        if (mine && inrange) {
            // bits j with 0 <= p_first + j < n  (p_first > -32 here because the lane is in range)
            const uint32_t from0 = p_first >= 0 ? 0xFFFFFFFFu : (0xFFFFFFFFu << (int)(-p_first));
            auto range_mask = [&](int n) -> uint32_t {
                const int64_t hi = (int64_t)n - p_first;   // bits below hi are < n
                const uint32_t upto = hi >= 32 ? 0xFFFFFFFFu : hi <= 0 ? 0u : ((1u << (int)hi) - 1u);
                return upto & from0;
            };
            inwin = range_mask(len);
            v0 = range_mask(np0);
            v1 = range_mask(np1);
        }
        // ---- passFilter counts ----
        if (inwin && doCounts) {
            LaneSeq qv;
            load32(qbase + a0, true, qv);
            if (inwin == 0xFFFFFFFFu) {
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const uint32_t q = qv.w[k];
                    totalq = (int)__dp4a(q, 0x01010101u, (unsigned)totalq);
                    lowq_ge += __popc(((q | 0x80808080u) - qq4) & 0x80808080u);   // bit7: q >= qualified
                }
                nbytes += 32;
            } else {
                for (int j = 0; j < 32; j++)
                    if (inwin >> j & 1u) {
                        const int q = (int)((qv.w[j >> 2] >> (8 * (j & 3))) & 0xFFu);
                        totalq += q;
                        lowq_ge += (q & 0x7f) >= (int)(qq4 & 0x7f);
                        nbytes++;
                    }
            }
            nn += __popc(NM & inwin);
        }
        if (doCplx) {   // warp-uniform: pairs (i, i+1), i < len-1; byte 31's partner is the next lane's first byte
            const uint32_t nxt = __shfl_down_sync(0xffffffffu, sq.w[0], 1);
            if (inwin) {
                uint32_t pm = inwin;
                const int64_t last = (int64_t)len - 1 - p_first;   // bit index of the window's last byte
                if (last >= 0 && last < 32) pm &= ~(1u << last);
                if (pm == 0xFFFFFFFFu) {
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const uint32_t w = sq.w[k], w2 = k < 7 ? sq.w[k + 1] : nxt;
                        diff += __popc(nz7(w ^ __funnelshift_r(w, w2, 8)));
                    }
                } else {
                    for (int j = 0; j < 32; j++)
                        if (pm >> j & 1u) {
                            const uint32_t c0 = (sq.w[j >> 2] >> (8 * (j & 3))) & 0xFFu;
                            const uint32_t w2 = (j + 1) < 32 ? sq.w[(j + 1) >> 2] : nxt;
                            const uint32_t c1 = (w2 >> (8 * ((j + 1) & 3))) & 0xFFu;
                            diff += c0 != c1;
                        }
                }
            }
        }
        // ---- Hamming scans ----
        if (doAdapters) {
            // planes of this lane's word and of the HL following words (neighbour lanes; the last HL lanes of the tile
            // read wrapped garbage, their results are masked out by `mine`)
            uint32_t PV[HL + 1], P1[HL + 1], P2[HL + 1];
            PV[0] = V; P1[0] = HI; P2[0] = LO;
#pragma unroll
            for (int w = 1; w <= HL; w++) {
                PV[w] = __shfl_down_sync(0xffffffffu, V, w);
                P1[w] = __shfl_down_sync(0xffffffffu, HI, w);
                P2[w] = __shfl_down_sync(0xffffffffu, LO, w);
            }
            Counter<NPL> c0, c1;
            c0.clear(); c1.clear();
#pragma unroll
            for (int i0 = 0; i0 < HL * 32; i0 += 8) {
                if (i0 < amax) {                           // warp-uniform
                    uint32_t sv[8], s1[8], s2[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int i = i0 + j, w = i >> 5, sh = i & 31;
                        sv[j] = __funnelshift_r(PV[w], PV[w + 1], sh);
                        s1[j] = __funnelshift_r(P1[w], P1[w + 1], sh);
                        s2[j] = __funnelshift_r(P2[w], P2[w + 1], sh);
                    }
#pragma unroll
                    for (int k = 0; k < 2; k++) {
                        const int alen = k ? alen1 : alen0;
                        if (i0 < alen) {                   // warp-uniform
                            uint32_t x[8];
                            if (i0 + 8 <= alen) {
#pragma unroll
                                for (int j = 0; j < 8; j++) {
                                    const uint32_t u = sv[j] & ~(s1[j] ^ plan.hm[k][i0 + j]);
                                    x[j] = u & ~(s2[j] ^ plan.lm[k][i0 + j]);
                                }
                            } else {                       // last block of an adapter whose length is not a multiple of 8
#pragma unroll
                                for (int j = 0; j < 8; j++) {
                                    const uint32_t u = sv[j] & ~(s1[j] ^ plan.hm[k][i0 + j]);
                                    x[j] = u & ~(s2[j] ^ plan.lm[k][i0 + j]) & plan.vm[k][i0 + j];
                                }
                            }
                            if (k) c1.add8(x); else c0.add8(x);
                        }
                    }
                }
            }
            c0.argmax(v0, p_first, bestM0, bestP0);
            c1.argmax(v1, p_first, bestM1, bestP1);
        }
    }
    // ---- block reduction ----
    unsigned long long k0 = bestM0 >= 0 ? (((unsigned long long)(unsigned)(alen0 - bestM0) << 32) | (unsigned)bestP0) : ~0ull;
    unsigned long long k1 = bestM1 >= 0 ? (((unsigned long long)(unsigned)(alen1 - bestM1) << 32) | (unsigned)bestP1) : ~0ull;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        unsigned long long o0 = __shfl_xor_sync(0xffffffffu, k0, d), o1 = __shfl_xor_sync(0xffffffffu, k1, d);
        k0 = o0 < k0 ? o0 : k0; k1 = o1 < k1 ? o1 : k1;
    }
    lowq_ge = __reduce_add_sync(0xffffffffu, lowq_ge); nn = __reduce_add_sync(0xffffffffu, nn);
    totalq = __reduce_add_sync(0xffffffffu, totalq); diff = __reduce_add_sync(0xffffffffu, diff);
    nbytes = __reduce_add_sync(0xffffffffu, nbytes);
    if (lane == 0) {
        sh64[0][wid] = k0; sh64[1][wid] = k1;
        sh32[0][wid] = nbytes - lowq_ge;                  // #(q < qualified)
        sh32[1][wid] = nn;
        sh32[2][wid] = totalq - 33 * nbytes;              // sum(q - 33)
        sh32[3][wid] = diff;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long m0 = sh64[0][0], m1 = sh64[1][0];
        int c0 = sh32[0][0], c1 = sh32[1][0], c2 = sh32[2][0], c3 = sh32[3][0];
        for (int i = 1; i < SF_WARPS; i++) {
            m0 = sh64[0][i] < m0 ? sh64[0][i] : m0; m1 = sh64[1][i] < m1 ? sh64[1][i] : m1;
            c0 += sh32[0][i]; c1 += sh32[1][i]; c2 += sh32[2][i]; c3 += sh32[3][i];
        }
        ReadState* o = &st[r];
        o->best[0] = m0; o->best[1] = m1;
        o->lowq = c0; o->nn = c1; o->totalq = c2; o->diff = c3;
    }
}

void launch_scan_fast(const DevParams& P, const ScanPlan& plan, const DevBatch& b, ReadState* st, cudaStream_t stream, int& launched) {
    if (b.n_reads == 0) return;
    const unsigned grid = (unsigned)b.n_reads;
#define SF_LAUNCH(N, H) k_scan_fast<N, H><<<grid, SF_THREADS, 0, stream>>>(P, plan, b, st)
    const int key = plan.npl * 10 + plan.halo_words;
    switch (key) {
        case 51: SF_LAUNCH(5, 1); break;
        case 61: SF_LAUNCH(6, 1); break;
        case 62: SF_LAUNCH(6, 2); break;
        case 72: SF_LAUNCH(7, 2); break;
        case 73: SF_LAUNCH(7, 3); break;
        case 74: SF_LAUNCH(7, 4); break;
        default: SF_LAUNCH(8, 4); break;
    }
#undef SF_LAUNCH
    launched++;
}
