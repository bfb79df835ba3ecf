// Stats::statRead (src/stats.cpp:265-375) as kernels over a list of segments
// (pre-filter Stats: every input read; post-filter Stats: every passing segment):
//
//  k_cycle_stats  column-tiled over the LENGTH-SORTED segment list: a CTA owns a 512-byte tile of the segments'
//                 16-byte-aligned byte ranges x a group of up to 4000 segments; its warps take the group's segments
//                 round-robin, one aligned 16-byte vector of sequence and of quality per lane (cp.async ring, several
//                 segments in flight).  The per-(base-bin, cycle) counters live in shared memory, one 32-bit word =
//                 (count << 20 | sum of raw quality chars), laid out so that the 32 lanes of a reduction hit 32 banks
//                 whatever the segment's misalignment; the tile is flushed once to the global int64 arrays
//                 mCycleBaseContents / mCycleBaseQual.  The 5-mer variant also fills lane-private 1024-bin tables
//                 (mKmer) from 2-bit codes packed by multiplication, with an exact A/C/G/T/U test.  Its fused form runs
//                 over the pre-filter list and counts each read's slot-0 passing segment into the post-filter counters
//                 too; the plain variant then counts the passing segments it did not take.
//  k_read_qual    row-shaped: a warp owns a read, builds its quality histogram with shared-memory atomics
//                 (16-byte vector loads, four per lane in flight), adds it to mBaseQualHistogram and derives the
//                 per-read median quality (mMedianReadQualHistogram / mMedianReadQualBases / mReads / mLengthSum)
//                 for BOTH Stats objects: a passing segment's histogram is the read's minus the removed ends.
//  k_kmer_fix     post-filter 5-mer table = pre-filter table - the 5-mers outside the passing segments.
#include "fpl_device.cuh"
#include "fpl_stats.h"

#include <atomic>
#include <stdlib.h>
#include <cub/cub.cuh>

#define CS_NT_KMER 1024                          // threads per CTA with the 5-mer tables (one CTA per SM: the fused pass takes 214 KB of shared memory, within H100's 227 KB per block)
#define CS_NT_PLAIN 512
#define CS_TILE 512                              // bytes of every segment a CTA looks at: one 16-byte vector per lane
#define CS_ROWW 33                               // words per counter row: 32 lanes + the carry column
#define CS_BINW (16 * CS_ROWW + 16)              // words per base bin: a multiple of 32, so the bank is the lane's whatever the bin
#define CS_GROUP 4000                            // segments per CTA; packed counter: count <= 4095, sum of q < 2^20
#define CS_STAGE 1000                            // descriptors staged in shared memory at a time
#define CS_SLOT 1040                             // ring slot: 16 B in front of the tile (its last 4 are used), 512 B sequence, 512 B quality
#define CS_DEPTH_KMER 1                          // segments in flight per warp (the 5-mer variant is bound by the logic pipe)
#define CS_DEPTH_PLAIN 3
#define CS_SMEM_BASE (8 * CS_BINW * 4 + CS_STAGE * 16)            // counters + staged descriptors
#define CS_MBAR_BYTES(NT, DEPTH) (((NT) / 32) * ((DEPTH) + 1) * 8)          // one mbarrier per ring slot (TMA staging)
#define CS_SMEM_PLAIN (CS_SMEM_BASE + (CS_NT_PLAIN / 32) * (CS_DEPTH_PLAIN + 1) * CS_SLOT + CS_MBAR_BYTES(CS_NT_PLAIN, CS_DEPTH_PLAIN))
#define CS_KMER_WORDS (512 * 32)                 // lane-private 5-mer tables: [code >> 1][lane], two 16-bit counters per word
#define CS_SMEM_KMER (CS_SMEM_BASE + (CS_NT_KMER / 32) * (CS_DEPTH_KMER + 1) * CS_SLOT + CS_KMER_WORDS * 4 + CS_MBAR_BYTES(CS_NT_KMER, CS_DEPTH_KMER))
// The fused pass (pre-filter list, each read carrying its slot-0 post-filter segment [s, e)): the post-filter counters
// of the columns a tile can reach.  Column pc is the post-filter cycle t0 - 15 - CS_REACH + pc, pc in [0, 16 * CS_PROWW):
// the pre-filter cycles [t0 - 15, t0 + 512) of the tile, moved back by s < CS_REACH.  The bin stride is a multiple of 32
// words (the bank of a reduction is its lane's whatever the bin) and CS_PBINW * 4 / 16 fits a dp4a weight byte.
#define CS_PROWW 62                              // positions per post row
#define CS_PBINW (16 * CS_PROWW)                 // words per post base bin
#define CS_REACH (16 * CS_PROWW - CS_TILE - 16)  // 464: post segments starting at s < CS_REACH are counted by the fused pass
#define CS_SMEM_FUSED (CS_SMEM_KMER + 8 * CS_PBINW * 4 + CS_STAGE * 16)   // + post counters + staged post descriptors

static_assert(CS_PBINW % 32 == 0 && CS_PBINW * 4 / 16 <= 255 && CS_PBINW * 4 % 16 == 0, "post bin stride: banks and dp4a weight");
static_assert(16 * CS_PROWW >= CS_TILE + 15 + CS_REACH && CS_REACH > 0 && CS_REACH % 16 == 0, "post window covers the reach");
static_assert(CS_GROUP * 16 <= 0xFFFF, "16-bit 5-mer counter: a lane adds at most 16 5-mers per segment of its group");
static_assert(CS_GROUP <= 4095 && 127 * CS_GROUP < (1 << 20), "packed counter: a segment adds at most one byte to a column");
static_assert(CS_SMEM_FUSED <= 232448, "fused pass: one CTA per SM");

namespace {

// byte -> (valid << 2 | 2-bit code) for the 5-mer table: A=0, T/U=1, C=2, G=3 (Stats::base2val, src/stats.cpp:411-425)
__device__ __forceinline__ uint32_t kmer_code(uint32_t b) {
    uint32_t v = 8;  // invalid
    v = b == 'A' ? 0u : v;
    v = (b == 'T' || b == 'U') ? 1u : v;
    v = b == 'C' ? 2u : v;
    v = b == 'G' ? 3u : v;
    return v;
}

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {   // PTX semantics: selector bit 3 = sign fill
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}
__device__ __forceinline__ uint32_t mad_u32(uint32_t a, uint32_t b, uint32_t c) {  // keeps the work on the IMAD pipe
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}

// ---- 1-D TMA (cp.async.bulk) staging: one lane copies a whole 512-byte tile row, completion on an mbarrier ----
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

template <int IMM>
__device__ __forceinline__ void red_shared_add_imm(uint32_t saddr, uint32_t v) {
    asm volatile("red.shared.add.u32 [%0 + %2], %1;" ::"r"(saddr), "r"(v), "n"(IMM) : "memory");
}

// Counter word of (bin, column): the CTA's columns are the cycles 512*tile - 15 + col, col in [0, 527).  Column col lives
// in row col & 15 at position col >> 4 (33 positions per row), so that the 32 lanes of one instruction — which hold the
// columns 16*lane + m for one m — hit 32 different banks (the bin stride is a multiple of 32 words).
// A lane's vector starts S columns into its 16-column stripe (S = 15 - (segment address & 15), warp-uniform): byte J
// is column 16*lane + J + S = row (J+S)&15, position lane + ((J+S)>>4).
//   wm: base & 7 in every byte; qm: quality chars; cw: 0x10 in every byte that counts (0 elsewhere, with qm = 0 there)
// Per base: one PRMT for the bin, one for the value (quality | 1 << 20), one IMAD for the address, one reduction.
// ROWW / BINW: the table's geometry (CS_ROWW / CS_BINW, or CS_PROWW / CS_PBINW for the post window, where S also holds
// the post shift and runs up to 30).
template <int S, int J, int ROWW, int BINW>
__device__ __forceinline__ void count1(const uint32_t (&wm)[4], const uint32_t (&qm)[4], const uint32_t (&cw)[4], uint32_t pk_lane) {
    constexpr int jj = J & 3, m = J + S, z = 8 | jj;                      // selector z: sign fill of a 7-bit byte = 0
    const uint32_t bin = prmt(wm[J >> 2], 0u, jj | z << 4 | z << 8 | z << 12);
    const uint32_t val = prmt(qm[J >> 2], cw[J >> 2], jj | z << 4 | (4 + jj) << 8 | z << 12);
    red_shared_add_imm<4 * ((m & 15) * ROWW + (m >> 4))>(mad_u32(bin, BINW * 4u, pk_lane), val);
}
template <int S, int ROWW = CS_ROWW, int BINW = CS_BINW>
__device__ __forceinline__ void count16(const uint32_t (&wm)[4], const uint32_t (&qm)[4], const uint32_t (&cw)[4], uint32_t pk) {
    count1<S, 0, ROWW, BINW>(wm, qm, cw, pk); count1<S, 1, ROWW, BINW>(wm, qm, cw, pk); count1<S, 2, ROWW, BINW>(wm, qm, cw, pk);
    count1<S, 3, ROWW, BINW>(wm, qm, cw, pk); count1<S, 4, ROWW, BINW>(wm, qm, cw, pk); count1<S, 5, ROWW, BINW>(wm, qm, cw, pk);
    count1<S, 6, ROWW, BINW>(wm, qm, cw, pk); count1<S, 7, ROWW, BINW>(wm, qm, cw, pk); count1<S, 8, ROWW, BINW>(wm, qm, cw, pk);
    count1<S, 9, ROWW, BINW>(wm, qm, cw, pk); count1<S, 10, ROWW, BINW>(wm, qm, cw, pk); count1<S, 11, ROWW, BINW>(wm, qm, cw, pk);
    count1<S, 12, ROWW, BINW>(wm, qm, cw, pk); count1<S, 13, ROWW, BINW>(wm, qm, cw, pk); count1<S, 14, ROWW, BINW>(wm, qm, cw, pk);
    count1<S, 15, ROWW, BINW>(wm, qm, cw, pk);
}

// The same for a vector whose 16 bytes all count (warp-uniform fast path): both operands of the reduction come from
// the FMA pipe, which issues beside the logic pipe (tools/ubench_pipes.cu measures LOP3 and IDP.4A alone and
// interleaved).  wb: (base & 7) << 4 in every byte, so that
// one dp4a with the weight 136 on byte J is bin * CS_BINW * 4 (+ the lane's base address); qm: quality chars.
// wa[j] = 136 << 8j and wv[j] = 1 << 8j arrive as run-time values (uniform registers for the whole loop): as literals
// the compiler re-materialises the eight of them with UMOVs in front of every vector.
template <int S, int J>
__device__ __forceinline__ void count1f(const uint32_t (&wb)[4], const uint32_t (&qm)[4], uint32_t pk_lane,
                                        const uint32_t (&wa)[4], const uint32_t (&wv)[4]) {
    constexpr int jj = J & 3, m = J + S;
    static_assert(CS_BINW * 4 == 136 * 16, "dp4a weight of the bin stride");
    const uint32_t addr = __dp4a(wb[J >> 2], wa[jj], pk_lane);
    const uint32_t val = __dp4a(qm[J >> 2], wv[jj], 1u << 20);
    red_shared_add_imm<4 * ((m & 15) * CS_ROWW + (m >> 4))>(addr, val);
}
template <int S>
__device__ __forceinline__ void count16f(const uint32_t (&wb)[4], const uint32_t (&qm)[4], uint32_t pk, const uint32_t (&wa)[4],
                                         const uint32_t (&wv)[4]) {
    count1f<S, 0>(wb, qm, pk, wa, wv); count1f<S, 1>(wb, qm, pk, wa, wv); count1f<S, 2>(wb, qm, pk, wa, wv); count1f<S, 3>(wb, qm, pk, wa, wv);
    count1f<S, 4>(wb, qm, pk, wa, wv); count1f<S, 5>(wb, qm, pk, wa, wv); count1f<S, 6>(wb, qm, pk, wa, wv); count1f<S, 7>(wb, qm, pk, wa, wv);
    count1f<S, 8>(wb, qm, pk, wa, wv); count1f<S, 9>(wb, qm, pk, wa, wv); count1f<S, 10>(wb, qm, pk, wa, wv); count1f<S, 11>(wb, qm, pk, wa, wv);
    count1f<S, 12>(wb, qm, pk, wa, wv); count1f<S, 13>(wb, qm, pk, wa, wv); count1f<S, 14>(wb, qm, pk, wa, wv); count1f<S, 15>(wb, qm, pk, wa, wv);
}

// The fused pass: the same value goes to the pre-filter column (m = J + 15, aligned) and to the post-filter window column
// J + T (T = 15 + (CS_REACH - s) & 15) at the segment's post lane base ppk = window + 4 * (lane + (CS_REACH - s) >> 4);
// the post bin offset is one more dp4a (wp[j] = (CS_PBINW * 4 / 16) << 8j).  Per base: three dp4a, two reductions.
template <int T, int J>
__device__ __forceinline__ void count1ff(const uint32_t (&wb)[4], const uint32_t (&qm)[4], uint32_t pk_lane, uint32_t ppk,
                                         const uint32_t (&wa)[4], const uint32_t (&wv)[4], const uint32_t (&wp)[4]) {
    constexpr int jj = J & 3, m = J + 15, mp = J + T;
    const uint32_t val = __dp4a(qm[J >> 2], wv[jj], 1u << 20);
    red_shared_add_imm<4 * ((m & 15) * CS_ROWW + (m >> 4))>(__dp4a(wb[J >> 2], wa[jj], pk_lane), val);
    red_shared_add_imm<4 * ((mp & 15) * CS_PROWW + (mp >> 4))>(__dp4a(wb[J >> 2], wp[jj], ppk), val);
}
template <int T>
__device__ __forceinline__ void count16ff(const uint32_t (&wb)[4], const uint32_t (&qm)[4], uint32_t pk, uint32_t ppk,
                                          const uint32_t (&wa)[4], const uint32_t (&wv)[4], const uint32_t (&wp)[4]) {
    count1ff<T, 0>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 1>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 2>(wb, qm, pk, ppk, wa, wv, wp);
    count1ff<T, 3>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 4>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 5>(wb, qm, pk, ppk, wa, wv, wp);
    count1ff<T, 6>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 7>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 8>(wb, qm, pk, ppk, wa, wv, wp);
    count1ff<T, 9>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 10>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 11>(wb, qm, pk, ppk, wa, wv, wp);
    count1ff<T, 12>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 13>(wb, qm, pk, ppk, wa, wv, wp); count1ff<T, 14>(wb, qm, pk, ppk, wa, wv, wp);
    count1ff<T, 15>(wb, qm, pk, ppk, wa, wv, wp);
}

// 0xFF in byte k of the result iff bit k of the nibble n
__device__ __forceinline__ uint32_t nibble_to_bytes(uint32_t n) { return ((n * 0x00204081u) & 0x01010101u) * 0xFFu; }

// Post-filter window, masked: the 16 bytes of the lane that lie in [plo, plim) of the tile (vmask as for the pre-filter
// columns), shift T = S + (CS_REACH - s) & 15 in [0, 30].
__device__ __forceinline__ void count_post_masked(const uint32_t (&wm)[4], const uint32_t (&q0)[4], int plo, int plim, int T,
                                                  int lane, uint32_t ppk) {
    const int lo = max(0, plo - 16 * lane), hi = min(16, max(0, plim - 16 * lane));
    const uint32_t pm = hi > lo ? ((0xFFFFu >> (16 - hi)) & (0xFFFFu << lo)) : 0u;
    uint32_t qm[4], cw[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t bm = nibble_to_bytes((pm >> (4 * i)) & 15u);
        qm[i] = q0[i] & bm; cw[i] = 0x10101010u & bm;
    }
#define CS_PM(t) case t: count16<t, CS_PROWW, CS_PBINW>(wm, qm, cw, ppk); break;
    switch (T) {
        CS_PM(0) CS_PM(1) CS_PM(2) CS_PM(3) CS_PM(4) CS_PM(5) CS_PM(6) CS_PM(7) CS_PM(8) CS_PM(9) CS_PM(10) CS_PM(11) CS_PM(12)
        CS_PM(13) CS_PM(14) CS_PM(15) CS_PM(16) CS_PM(17) CS_PM(18) CS_PM(19) CS_PM(20) CS_PM(21) CS_PM(22) CS_PM(23) CS_PM(24)
        CS_PM(25) CS_PM(26) CS_PM(27) CS_PM(28) CS_PM(29) default: count16<30, CS_PROWW, CS_PBINW>(wm, qm, cw, ppk); break;
    }
#undef CS_PM
}

// 5-mer ending at byte T of the lane's vector.  P: 2-bit codes, oldest first, the 5-mer's in bits [22-SHL .. 32-SHL); the
// table word is [code >> 1][lane] (no bank conflicts) and holds two 16-bit counters: the low one counts both codes 2w and
// 2w + 1, the high one code 2w + 1 (the flush takes the difference).  The low bit of the code is bit 1 of byte T
// (c' = (b >> 1) & 3 of the newest base); hb holds it in every byte, and one PRMT makes the value 1 | bit << 16.
// An invalid 5-mer adds 0 (no branch around the reduction — a reduction predicated on the validity bit is compiled into
// BSSY / BRA / BSYNC around it: four instructions instead of two).
// Left shifts as multiplies: they run on the IMAD pipe.  (Right shifts stay shifts: as mul.hi they would use the slower
// IMAD.HI; mask + shift-and-add compiles to the same four instructions.)
template <int T>
__device__ __forceinline__ uint32_t kmer_inc(const uint32_t (&hb)[4]) {
    return prmt(hb[T >> 2], 1u, 4 | 5 << 4 | (T & 3) << 8 | 5 << 12);      // byte 0 = 1, byte 2 = the code's low bit
}
template <int SHL, int T>
__device__ __forceinline__ void kmer1(uint32_t P, uint32_t ok, uint32_t km_lane, const uint32_t (&hb)[4]) {
    const uint32_t w = (SHL ? mad_u32(P, 1u << SHL, 0u) : P) >> 23;
    red_shared_add(mad_u32(w, 128u, km_lane), mad_u32((ok >> T) & 1u, kmer_inc<T>(hb), 0u));
}

// the same when the 5-mer is known to count
template <int SHL, int T>
__device__ __forceinline__ void kmer1f(uint32_t P, uint32_t km_lane, const uint32_t (&hb)[4]) {
    const uint32_t w = (SHL ? mad_u32(P, 1u << SHL, 0u) : P) >> 23;
    red_shared_add(mad_u32(w, 128u, km_lane), kmer_inc<T>(hb));
}

// Per 4 bytes of sequence: in7 = (nibble of "byte is not one of A, C, G, T, U") << 7, exact for any byte value, and
// pc = four 2-bit codes c' = (b >> 1) & 3, oldest first.  g = b2 & ~b1 (set for T/U); with bit 7 and bits 2..1 masked
// off, a valid byte is 0x41 (A, C, G) or, with g, 0x51 (T, U): d == 0.  d < 0x80, so d + 0x7f sets bit 7 iff d != 0 and
// cannot carry into the next byte; the byte's own bit 7 is or-ed in by the same LOP3.  The two gathers are dp4a.
__device__ __forceinline__ void encode4(uint32_t w, uint32_t one, uint32_t& nz, uint32_t& pc) {
    const uint32_t x1 = w >> 1;
    const uint32_t g = (x1 >> 1) & ~x1 & 0x01010101u;
    const uint32_t d = ((w & 0x79797979u) | g) ^ 0x41414141u ^ mad_u32(g, 16u, 0u);
    nz = (mad_u32(d, one, 0x7f7f7f7fu) | w) & 0x80808080u;
    pc = __dp4a(x1 & 0x03030303u, 0x01041040u, 0u);
}

}  // namespace

// Sorted segment descriptor (by length, longest first).  The fused pass: the read's slot-0 post-filter segment
// [ps, ps + pl) relative to the read (pl = 0: none, or one the residual pass counts).
struct SegD {
    int64_t off;
    int32_t len;
    int32_t ps, pl;
    int32_t pad;
};
// The same as a CTA stages it for its tile: a = 16-byte aligned byte offset of the tile's first vector, lim = how many
// of the tile's bytes lie in front of the segment's end (> 0), sh = segment address & 15.
struct __align__(16) TileSeg {
    int64_t a;
    int32_t lim;
    int32_t sh;
};
// The post-filter part (fused pass): the tile bytes [plo, plim) are post-filter cycles; d = CS_REACH - s.  plim <= plo:
// none in this tile.
struct __align__(16) TilePost {
    int32_t plo, plim, d, pad;
};

// "The fused pass counts this post-filter segment": a passing slot-0 segment starting fewer than CS_REACH bytes into its
// read.  read_off: the offset of the read's pre-filter segment (the whole read).  The residual pass counts the others.
__device__ __forceinline__ bool cs_fused_takes(const StatSeg& p, int64_t read_off) {
    return p.len > 0 && p.slot == 0 && p.off - read_off < CS_REACH;
}

// DO_KMER: also count the 5-mers; their table is flushed to `stats` and, if given, to `kmer_also` (the post-filter
// block: post 5-mers = pre 5-mers - the ones k_kmer_fix finds outside the passing segments).
//
// Grid: x = 512-byte tile of the segments' 16-byte-aligned byte ranges, y = group of CS_GROUP segments of the list
// sorted by length (so a group's segments end in the same few tiles and the CTAs beyond the longest one leave at once).
// Every load is an aligned 16-byte vector: the misalignment of a segment (its address & 15, different for every
// post-filter segment) moves the COLUMNS its bytes count into instead of the bytes (count16<S>).
// TMA = true: the tile rows are staged by 1-D bulk copies (cp.async.bulk + mbarrier) issued by one lane per warp instead
// of 32 lanes' cp.async — the variant FPL_CS_TMA=1 selects; both are measured in profiles/README.md.
// FUSE (5-mer variant over the pre-filter list): every byte of a read's post-filter segment is also counted into the
// post-filter window at cycle p - s, flushed to `stats_post` — one read of the payload feeds both Stats blocks.
template <bool DO_KMER, int NT, int DEPTH, bool TMA, bool FUSE>
__global__ void __launch_bounds__(NT, DO_KMER ? 1 : 2048 / NT / 2)
k_cycle_stats(const uint8_t* __restrict__ seqbuf, const uint8_t* __restrict__ qualbuf, const SegD* __restrict__ segs,
              int64_t nseg, unsigned long long* __restrict__ stats, int64_t C, unsigned long long* __restrict__ kmer_also,
              unsigned long long* __restrict__ stats_post, uint32_t one, int aligned) {
    static_assert(!FUSE || DO_KMER, "the fused pass is the 5-mer variant");
    extern __shared__ __align__(16) uint8_t cs_smem[];
    uint32_t* packed = reinterpret_cast<uint32_t*>(cs_smem);                       // [8][16][33]: count << 20 | sum of q
    TileSeg* stage = reinterpret_cast<TileSeg*>(cs_smem + 8 * CS_BINW * 4);
    uint8_t* ring = reinterpret_cast<uint8_t*>(stage + CS_STAGE);                  // [warps][DEPTH+1] slots of CS_SLOT bytes
    uint32_t* kmer = reinterpret_cast<uint32_t*>(ring + (NT / 32) * (DEPTH + 1) * CS_SLOT);   // [512][32]: one column per lane
    uint8_t* mbars = reinterpret_cast<uint8_t*>(kmer) + (DO_KMER ? CS_KMER_WORDS * 4 : 0);    // [warps][DEPTH+1] mbarriers (TMA)
    uint32_t* ptab = reinterpret_cast<uint32_t*>(mbars + CS_MBAR_BYTES(NT, DEPTH));          // FUSE: [8][16][CS_PROWW]
    TilePost* pstage = reinterpret_cast<TilePost*>(ptab + (FUSE ? 8 * CS_PBINW : 0));        // FUSE: [CS_STAGE]
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const int64_t t0 = (int64_t)blockIdx.x * CS_TILE;      // first byte of this tile, relative to the aligned segment start
    const int64_t g0 = (int64_t)blockIdx.y * CS_GROUP;
    const int64_t g1 = min(nseg, g0 + CS_GROUP);
    {
        const int maxlen = segs[g0].len;                   // sorted: the group's longest segment
        if (maxlen <= 0 || t0 >= (int64_t)maxlen + 15) return;
    }
    for (int i = threadIdx.x; i < 8 * CS_BINW; i += NT) packed[i] = 0;
    if (DO_KMER) {
        uint4* kz = reinterpret_cast<uint4*>(kmer);
        for (int i = threadIdx.x; i < CS_KMER_WORDS / 4; i += NT) kz[i] = make_uint4(0, 0, 0, 0);
    }
    if (FUSE)
        for (int i = threadIdx.x; i < 8 * CS_PBINW; i += NT) ptab[i] = 0;
    const uint32_t pk_lane = shared_addr(packed) + (uint32_t)lane * 4u;
    const uint32_t km_lane = shared_addr(kmer) + (uint32_t)lane * 4u;
    const uint32_t pt_lane = shared_addr(ptab) + (uint32_t)lane * 4u;
    const uint8_t* seq_lane = seqbuf + 16 * lane;
    const uint8_t* qual_lane = qualbuf + 16 * lane;
    // a slot: [16 bytes in front of the tile][512 bytes of sequence][512 bytes of quality]; the word in front of a lane's
    // vector — the previous lane's last word, for lane 0 the front bytes — is at the same offset for every lane
    const uint32_t ring_warp = shared_addr(ring) + (uint32_t)wid * ((DEPTH + 1) * CS_SLOT);
    const uint32_t ring_lane = ring_warp + 16u + (uint32_t)lane * 16u;
    const uint32_t bar_warp = shared_addr(mbars) + (uint32_t)wid * ((DEPTH + 1) * 8);
    const uint32_t wa[4] = {136u * one, (136u << 8) * one, (136u << 16) * one, (136u << 24) * one};   // one == 1
    const uint32_t wv[4] = {one, one << 8, one << 16, one << 24};
    constexpr uint32_t PW = CS_PBINW * 4 / 16;
    const uint32_t wp[4] = {PW * one, (PW << 8) * one, (PW << 16) * one, (PW << 24) * one};
    uint32_t phase = 0;                                  // TMA: the parity each slot's mbarrier completes next (bit per slot)
    if (TMA) {
        if (lane == 0)
            for (int d = 0; d <= DEPTH; d++) mbar_init(bar_warp + 8u * d, 1u);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    for (int64_t s0 = g0; s0 < g1; s0 += CS_STAGE) {
        __syncthreads();
        // stage the descriptors; the ones that can reach this tile are a prefix (sorted by length)
        int n = 0;
        for (int i0 = 0; i0 < CS_STAGE; i0 += NT) {
            const int i = i0 + threadIdx.x;
            bool reach = false;
            if (i < CS_STAGE && s0 + i < g1) {
                const SegD sg = segs[s0 + i];
                TileSeg ts;
                ts.sh = (int32_t)(sg.off & 15);
                ts.a = sg.off - ts.sh + t0;
                const int64_t lim = (int64_t)ts.sh + sg.len - t0;
                ts.lim = lim > 0 ? (int32_t)lim : 0;
                stage[i] = ts;
                if (FUSE) {
                    // tile byte of pre-filter cycle c: c + sh - t0
                    TilePost tp;
                    const int64_t lo = (int64_t)ts.sh + sg.ps - t0, hi = lo + sg.pl;
                    tp.plo = lo <= 0 ? 0 : lo >= CS_TILE ? CS_TILE : (int32_t)lo;
                    tp.plim = sg.pl <= 0 || hi <= 0 ? 0 : hi >= CS_TILE ? CS_TILE : (int32_t)hi;
                    tp.d = CS_REACH - sg.ps;
                    tp.pad = 0;
                    pstage[i] = tp;
                }
                reach = sg.len > 0 && (int64_t)sg.len + 15 > t0;
            }
            n += __syncthreads_count(reach);
        }
        if (n == 0) break;
        // software pipeline: the vectors of the next DEPTH segments of this warp are in flight (cp.async into the warp's
        // ring of DEPTH+1 slots: no registers held, every lane copies and later reads its own 16 bytes) while one is
        // processed; a lane beyond the segment's end copies 0 bytes, which zero-fills its slot bytes
        auto issue = [&](int k, int slot) {
            const TileSeg ts = stage[k];
            if (TMA) {
                // one lane: up to 512 bytes of sequence, the same of quality and (5-mers) the 16 bytes in front of the
                // tile; a tile the segment does not fill is copied up to its last vector, the rest of the slot keeps
                // stale bytes that the edge path masks
                __syncwarp();                              // every lane is done reading the slot that is refilled
                if (lane == 0) {
                    const uint32_t dst = ring_warp + (uint32_t)slot * CS_SLOT, bar = bar_warp + 8u * slot;
                    const uint32_t bytes = ts.lim > 0 ? (uint32_t)min(CS_TILE, (ts.lim + 15) & ~15) : 0u;
                    const uint32_t pb = (DO_KMER && t0 != 0 && bytes) ? 16u : 0u;
                    mbar_expect_tx(bar, 2u * bytes + pb);
                    if (bytes) { bulk_g2s(dst + 16u, seqbuf + ts.a, bytes, bar); bulk_g2s(dst + 528u, qualbuf + ts.a, bytes, bar); }
                    if (pb) bulk_g2s(dst, seqbuf + ts.a - 16, 16u, bar);
                }
                return;
            }
            const bool act = 16 * lane < ts.lim;
            const uint32_t dst = ring_lane + (uint32_t)slot * CS_SLOT;
            const int64_t la = ts.a + (act ? 16 * lane : 0);     // an inactive lane copies 0 bytes (zero fill); the address stays valid
            cp_async16(dst, seqbuf + la, act ? 16 : 0);
            cp_async16(dst + 512, qualbuf + la, act ? 16 : 0);
            // the four bases in front of the tile (lane 0's 5-mers): not needed in the first tile, where no 5-mer ends in
            // front of cycle 4; behind it a >= 512 - 15
            if (DO_KMER && lane == 0 && t0 != 0) cp_async4(dst - 4, seqbuf + ts.a - 4, 4);
        };
        int kk = wid;
#pragma unroll
        for (int d = 0; d < DEPTH; d++) {
            if (kk < n) issue(kk, d);
            if (!TMA) cp_async_commit();
            kk += NT / 32;
        }
        int slot = 0, fill = DEPTH;
        for (int k = wid; k < n; k += (NT / 32)) {
            if (TMA) { mbar_wait(bar_warp + 8u * slot, (phase >> slot) & 1u); phase ^= 1u << slot; }
            else {
                cp_async_wait<DEPTH - 1>();
                // the word in front of a lane's vector was copied by the lane below: a lane's wait covers its own copies
                // only, and the slot refilled further down was read by the neighbours in the previous round
                if (DO_KMER) __syncwarp();
            }
            const uint32_t src = ring_lane + (uint32_t)slot * CS_SLOT;
            const uint4 ns = lds128(src), nq = lds128(src + 512);
            const uint32_t pw = DO_KMER ? lds32(src - 4) : 0u;     // the four bases in front of this lane's vector
            const uint32_t sw[4] = {ns.x, ns.y, ns.z, ns.w};
            uint32_t qm[4] = {nq.x, nq.y, nq.z, nq.w};
            const int sh = stage[k].sh, lim = stage[k].lim;
            TilePost tp = {0, 0, 0, 0};
            if (FUSE) tp = pstage[k];
            if (kk < n) issue(kk, fill);
            if (!TMA) cp_async_commit();
            kk += NT / 32;
            static_assert(((DEPTH + 1) & DEPTH) == 0, "ring slots: a power of two");
            slot = (slot + 1) & DEPTH;
            fill = (fill + 1) & DEPTH;
            if (lim <= 0) continue;                        // warp-uniform: the segment ends in front of this tile
            const bool full = lim >= CS_TILE && t0 != 0;   // warp-uniform: every byte of every lane is a cycle >= 4
            // FUSE, warp-uniform: the tile holds bytes of the post-filter segment (post), all of its bytes are (pfull);
            // ppk: the segment's post lane base, T - S: its post shift
            const bool post = FUSE && tp.plim > tp.plo;
            const bool pfull = post && tp.plo == 0 && tp.plim >= CS_TILE;
            const uint32_t ppk = pt_lane + 4u * (uint32_t)(tp.d >> 4);
            const uint32_t q0[4] = {nq.x, nq.y, nq.z, nq.w};
            bool post_done = false;
            uint32_t kmask = 0xFFFFu;
            if (full) {
                // ---- per-(bin, cycle) counters, all 16 bytes of every lane: address and value by dp4a ----
                const uint32_t wb[4] = {mad_u32(sw[0], 16u, 0u) & 0x70707070u, mad_u32(sw[1], 16u, 0u) & 0x70707070u,
                                        mad_u32(sw[2], 16u, 0u) & 0x70707070u, mad_u32(sw[3], 16u, 0u) & 0x70707070u};
                // aligned: every segment starts on a 16-byte boundary (the pre-filter pass: whole reads in their slots)
                if (FUSE && pfull && (aligned || sh == 0)) {
                    // both Stats blocks from one value per base
                    post_done = true;
#define CS_FF(r) case r: count16ff<15 + r>(wb, qm, pk_lane, ppk, wa, wv, wp); break;
                    switch (tp.d & 15) {
                        CS_FF(0) CS_FF(1) CS_FF(2) CS_FF(3) CS_FF(4) CS_FF(5) CS_FF(6) CS_FF(7) CS_FF(8) CS_FF(9) CS_FF(10) CS_FF(11)
                        CS_FF(12) CS_FF(13) CS_FF(14) default: count16ff<30>(wb, qm, pk_lane, ppk, wa, wv, wp); break;
                    }
#undef CS_FF
                } else if (aligned) count16f<15>(wb, qm, pk_lane, wa, wv);
                else switch (sh) {
                    case 0: count16f<15>(wb, qm, pk_lane, wa, wv); break;
                    case 1: count16f<14>(wb, qm, pk_lane, wa, wv); break;
                    case 2: count16f<13>(wb, qm, pk_lane, wa, wv); break;
                    case 3: count16f<12>(wb, qm, pk_lane, wa, wv); break;
                    case 4: count16f<11>(wb, qm, pk_lane, wa, wv); break;
                    case 5: count16f<10>(wb, qm, pk_lane, wa, wv); break;
                    case 6: count16f<9>(wb, qm, pk_lane, wa, wv); break;
                    case 7: count16f<8>(wb, qm, pk_lane, wa, wv); break;
                    case 8: count16f<7>(wb, qm, pk_lane, wa, wv); break;
                    case 9: count16f<6>(wb, qm, pk_lane, wa, wv); break;
                    case 10: count16f<5>(wb, qm, pk_lane, wa, wv); break;
                    case 11: count16f<4>(wb, qm, pk_lane, wa, wv); break;
                    case 12: count16f<3>(wb, qm, pk_lane, wa, wv); break;
                    case 13: count16f<2>(wb, qm, pk_lane, wa, wv); break;
                    case 14: count16f<1>(wb, qm, pk_lane, wa, wv); break;
                    default: count16f<0>(wb, qm, pk_lane, wa, wv); break;
                }
            } else {
                // the segment starts or ends in this tile: which of the lane's 16 bytes are cycles of the segment (vmask)
                // and can end a 5-mer (kmask: cycle >= 4)
                uint32_t cw[4] = {0x10101010u, 0x10101010u, 0x10101010u, 0x10101010u};
                const int cyc0 = (int)t0 + 16 * lane - sh;                          // cycle of byte 0, negative in front
                const int lo = max(0, -cyc0), hi = min(16, max(0, lim - 16 * lane));
                const uint32_t vmask = hi > lo ? ((0xFFFFu >> (16 - hi)) & (0xFFFFu << lo)) : 0u;
                const int klo = min(16, max(0, 4 - cyc0));
                kmask = vmask & (0xFFFFu << klo);
                if (vmask != 0xFFFFu) {
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const uint32_t bm = nibble_to_bytes((vmask >> (4 * i)) & 15u);
                        qm[i] &= bm; cw[i] &= bm;
                    }
                }
                const uint32_t wm[4] = {sw[0] & 0x07070707u, sw[1] & 0x07070707u, sw[2] & 0x07070707u, sw[3] & 0x07070707u};
                switch (sh) {
                    case 0: count16<15>(wm, qm, cw, pk_lane); break;
                    case 1: count16<14>(wm, qm, cw, pk_lane); break;
                    case 2: count16<13>(wm, qm, cw, pk_lane); break;
                    case 3: count16<12>(wm, qm, cw, pk_lane); break;
                    case 4: count16<11>(wm, qm, cw, pk_lane); break;
                    case 5: count16<10>(wm, qm, cw, pk_lane); break;
                    case 6: count16<9>(wm, qm, cw, pk_lane); break;
                    case 7: count16<8>(wm, qm, cw, pk_lane); break;
                    case 8: count16<7>(wm, qm, cw, pk_lane); break;
                    case 9: count16<6>(wm, qm, cw, pk_lane); break;
                    case 10: count16<5>(wm, qm, cw, pk_lane); break;
                    case 11: count16<4>(wm, qm, cw, pk_lane); break;
                    case 12: count16<3>(wm, qm, cw, pk_lane); break;
                    case 13: count16<2>(wm, qm, cw, pk_lane); break;
                    case 14: count16<1>(wm, qm, cw, pk_lane); break;
                    default: count16<0>(wm, qm, cw, pk_lane); break;
                }
            }
            if (FUSE && post && !post_done) {
                // the tile holds s or e (or the segment is not 16-byte aligned): the post bytes by their own mask
                const uint32_t wm[4] = {sw[0] & 0x07070707u, sw[1] & 0x07070707u, sw[2] & 0x07070707u, sw[3] & 0x07070707u};
                count_post_masked(wm, q0, tp.plo, tp.plim, 15 - sh + (tp.d & 15), lane, ppk);
            }
            if (!DO_KMER) continue;
            // ---- 5-mers ending in this lane's 16 bytes (SURVEY A.1): all five bases in ACGTU, end cycle in [4, len) ----
            // per word: the "not ACGTU" flags and four 2-bit codes c' = (b >> 1) & 3 (A=0, C=1, T/U=2, G=3; the flush maps
            // them to base2val's); the word in front of the lane's vector (pw) supplies the four bases before it — every
            // lane encodes its own copy: cheaper than two shuffles plus a lane-0 branch around a fifth encode
            uint32_t nz[4], pc[4], pnz, ppc;
#pragma unroll
            for (int i = 0; i < 4; i++) encode4(sw[i], one, nz[i], pc[i]);
            encode4(pw, one, pnz, ppc);
            // flags << 7: bit 7+t = byte t-4 of the 20 bytes (previous four, then the lane's sixteen)
            const uint32_t pin7 = __dp4a(pnz, 0x08040201u, 0u);
            const uint32_t in01 = __dp4a(nz[0], 0x08040201u, __dp4a(nz[1], 0x80402010u, 0u));
            const uint32_t in23 = __dp4a(nz[2], 0x08040201u, __dp4a(nz[3], 0x80402010u, 0u));
            const uint32_t I27 = mad_u32(in23, 4096u, mad_u32(in01, 16u, pin7));     // 20 flags at bits 7..26
            // 20 codes, oldest first, 2 bits each: Phi = codes of bytes -4..11 (32 bits), Plo = bytes 4..15, then 8 zero bits
            const uint32_t Phi = mad_u32(ppc, 1u << 24, mad_u32(pc[0], 1u << 16, mad_u32(pc[1], 256u, pc[2])));
            const uint32_t Plo = mad_u32(pc[1], 1u << 24, mad_u32(pc[2], 1u << 16, pc[3] * 256u));
            // bit 1 of every byte (the low bit of its code) in bit 0 of the byte: which half of a table word a 5-mer adds to
            const uint32_t hb[4] = {(sw[0] >> 1) & 0x01010101u, (sw[1] >> 1) & 0x01010101u, (sw[2] >> 1) & 0x01010101u,
                                    (sw[3] >> 1) & 0x01010101u};
            if (full && !__any_sync(0xffffffffu, (I27 & 0x07FFFF80u) != 0u)) {
                // plain bases everywhere in the warp's 512 bytes: every 5-mer counts
                kmer1f<0, 0>(Phi, km_lane, hb); kmer1f<2, 1>(Phi, km_lane, hb); kmer1f<4, 2>(Phi, km_lane, hb); kmer1f<6, 3>(Phi, km_lane, hb);
                kmer1f<8, 4>(Phi, km_lane, hb); kmer1f<10, 5>(Phi, km_lane, hb); kmer1f<12, 6>(Phi, km_lane, hb); kmer1f<14, 7>(Phi, km_lane, hb);
                kmer1f<16, 8>(Phi, km_lane, hb); kmer1f<18, 9>(Phi, km_lane, hb); kmer1f<20, 10>(Phi, km_lane, hb); kmer1f<22, 11>(Phi, km_lane, hb);
                kmer1f<8, 12>(Plo, km_lane, hb); kmer1f<10, 13>(Plo, km_lane, hb); kmer1f<12, 14>(Plo, km_lane, hb); kmer1f<14, 15>(Plo, km_lane, hb);
            } else {
                // some lane holds an N (or another byte outside ACGTU), or the segment starts or ends in this tile: the
                // reductions add the value times the validity bit (a predicated reduction is compiled into a branch around
                // it: four instructions per 5-mer instead of two)
                const uint32_t I20 = I27 >> 7;
                const uint32_t bad = I20 | (I20 >> 1) | (I20 >> 2) | (I20 >> 3) | (I20 >> 4);   // bit t: a byte of t-4..t is invalid
                const uint32_t ok = ~bad & kmask;                                              // kmask = 0xFFFF when full
                kmer1<0, 0>(Phi, ok, km_lane, hb); kmer1<2, 1>(Phi, ok, km_lane, hb); kmer1<4, 2>(Phi, ok, km_lane, hb); kmer1<6, 3>(Phi, ok, km_lane, hb);
                kmer1<8, 4>(Phi, ok, km_lane, hb); kmer1<10, 5>(Phi, ok, km_lane, hb); kmer1<12, 6>(Phi, ok, km_lane, hb); kmer1<14, 7>(Phi, ok, km_lane, hb);
                kmer1<16, 8>(Phi, ok, km_lane, hb); kmer1<18, 9>(Phi, ok, km_lane, hb); kmer1<20, 10>(Phi, ok, km_lane, hb); kmer1<22, 11>(Phi, ok, km_lane, hb);
                kmer1<8, 12>(Plo, ok, km_lane, hb); kmer1<10, 13>(Plo, ok, km_lane, hb); kmer1<12, 14>(Plo, ok, km_lane, hb); kmer1<14, 15>(Plo, ok, km_lane, hb);
            }
        }
        if (n < CS_STAGE) break;     // the rest of the group is shorter still
    }
    __syncthreads();
    // flush: content[b][c] += count ; qual[b][c] += sumq - 33*count
    unsigned long long* content = stats;
    unsigned long long* qualsum = stats + 8 * C;
    for (int i = threadIdx.x; i < 8 * CS_BINW; i += NT) {
        const uint32_t v = packed[i];
        if (v) {
            const int bin = i / CS_BINW, p = i % CS_BINW;
            const int64_t c = t0 - 15 + 16 * (p % CS_ROWW) + p / CS_ROWW;
            const long long cnt = v >> 20, sq = v & 0xFFFFFu;
            atomicAdd(&content[(int64_t)bin * C + c], (unsigned long long)cnt);
            atomicAdd(&qualsum[(int64_t)bin * C + c], (unsigned long long)(sq - 33 * cnt));
        }
    }
    if (DO_KMER) {
        unsigned long long* tail = stats + 16 * C;
        for (int i = threadIdx.x; i < 1024; i += NT) {
            // word [i >> 1][lane]: low half = codes 2w and 2w + 1, high half = code 2w + 1
            uint32_t sum = 0;
            const int hi = i & 1;
#pragma unroll 8
            for (int l = 0; l < 32; l++) {
                const uint32_t v = kmer[(i >> 1) * 32 + ((l + threadIdx.x) & 31)];
                sum += hi ? v >> 16 : (v & 0xFFFFu) - (v >> 16);
            }
            if (sum) {
                // table index: five c' pairs (b2, b1); base2val's code is (b1, b2): swap the bits of every pair
                const int code = ((i & 0x155) << 1) | ((i >> 1) & 0x155);
                atomicAdd(&tail[FPL_STATS_KMER + code], (unsigned long long)sum);
                if (kmer_also) atomicAdd(&kmer_also[code], (unsigned long long)sum);
            }
        }
    }
    if (FUSE) {
        // post window: column 16 * pos + row is the post-filter cycle t0 - 15 - CS_REACH + column
        unsigned long long* pcontent = stats_post;
        unsigned long long* pqualsum = stats_post + 8 * C;
        for (int i = threadIdx.x; i < 8 * CS_PBINW; i += NT) {
            const uint32_t v = ptab[i];
            if (v) {
                const int bin = i / CS_PBINW, p = i % CS_PBINW;
                const int64_t c = t0 - 15 - CS_REACH + 16 * (p % CS_PROWW) + p / CS_PROWW;
                const long long cnt = v >> 20, sq = v & 0xFFFFFu;
                atomicAdd(&pcontent[(int64_t)bin * C + c], (unsigned long long)cnt);
                atomicAdd(&pqualsum[(int64_t)bin * C + c], (unsigned long long)(sq - 33 * cnt));
            }
        }
    }
}

namespace {
// taken_by (residual pass, or nullptr): the pre-filter list of the fused pass; a segment it counted gets the key 0
__global__ void k_cs_keys(const StatSeg* __restrict__ segs, int64_t n, uint32_t* __restrict__ keys, int32_t* __restrict__ vals,
                          const StatSeg* __restrict__ taken_by) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const StatSeg s = segs[i];
    keys[i] = s.len <= 0 || (taken_by && cs_fused_takes(s, taken_by[s.read].off)) ? 0u : (uint32_t)s.len;
    vals[i] = (int32_t)i;
}
// post (fused pass, or nullptr): the post-filter list; a read's slot-0 segment [2 * read] rides on its descriptor
__global__ void k_cs_gather(const StatSeg* __restrict__ segs, const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals,
                            int64_t n, SegD* __restrict__ out, const StatSeg* __restrict__ post) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const StatSeg sg = segs[vals[i]];
    SegD d;
    d.off = sg.off; d.len = (int32_t)keys[i]; d.ps = 0; d.pl = 0; d.pad = 0;
    if (post && d.len > 0) {
        const StatSeg p = post[2 * (int64_t)sg.read];
        if (cs_fused_takes(p, sg.off)) { d.ps = (int32_t)(p.off - sg.off); d.pl = p.len; }
    }
    out[i] = d;
}
}  // namespace

// kmer_also: where the 5-mer counts of this launch go besides `stats` (nullptr = nowhere else); do_kmer = false skips
// them.  fused_post (with do_kmer, segs = the pre-filter list, one per read): the post-filter list; the segments
// cs_fused_takes accepts are counted into stats_post by the same pass.  residual_of (segs = that post-filter list): the
// pre-filter list of the fused pass, whose segments this pass skips.  Returns 0, or -1 when the workspace cannot be
// allocated (before any launch).
int launch_cycle_stats(CycleWs* ws, const uint8_t* seq, const uint8_t* qual, const StatSeg* segs, int64_t nseg, int64_t max_len,
                       unsigned long long* stats, int64_t C, bool do_kmer, unsigned long long* kmer_also, bool aligned,
                       const StatSeg* fused_post, unsigned long long* stats_post, const StatSeg* residual_of,
                       cudaStream_t stream, int& launched) {
    if (nseg == 0 || max_len <= 0) return 0;
    // the opt-in to more than 48 KB of dynamic shared memory is a per-device function attribute
    static std::atomic<unsigned long long> attr_set{0};
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    if (!(attr_set.load() & bit)) {
        if (cudaFuncSetAttribute(k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM_KMER) != cudaSuccess ||
            cudaFuncSetAttribute(k_cycle_stats<false, CS_NT_PLAIN, CS_DEPTH_PLAIN, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM_PLAIN) != cudaSuccess ||
            cudaFuncSetAttribute(k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM_KMER) != cudaSuccess ||
            cudaFuncSetAttribute(k_cycle_stats<false, CS_NT_PLAIN, CS_DEPTH_PLAIN, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM_PLAIN) != cudaSuccess ||
            cudaFuncSetAttribute(k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM_FUSED) != cudaSuccess ||
            cudaFuncSetAttribute(k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM_FUSED) != cudaSuccess)
            return -1;
        attr_set.fetch_or(bit);
    }
    int end_bit = 1;
    while (end_bit < 31 && (max_len >> end_bit)) end_bit++;
    size_t need = 0;
    cub::DeviceRadixSort::SortPairsDescending(nullptr, need, ws->k_in.get(), ws->k_out.get(), ws->v_in.get(), ws->v_out.get(), (int)nseg, 0,
                                              end_bit, stream);
    if (nseg > ws->cap || (int64_t)need > ws->tmp.bytes()) {
        cudaStreamSynchronize(stream);
        if (nseg > ws->cap) {
            ws->cap = 0;
            if (ws->k_in.grow_exact(nseg) || ws->k_out.grow_exact(nseg) || ws->v_in.grow_exact(nseg) || ws->v_out.grow_exact(nseg) ||
                ws->sorted.grow_exact(nseg))
                return -1;
            ws->cap = nseg;
            // the temporary storage grows with the item count
            cub::DeviceRadixSort::SortPairsDescending(nullptr, need, ws->k_in.get(), ws->k_out.get(), ws->v_in.get(), ws->v_out.get(),
                                                      (int)nseg, 0, 31, stream);
        }
        if (ws->tmp.grow_exact((int64_t)need)) return -1;
    }
    const unsigned blocks = (unsigned)((nseg + 255) / 256);
    k_cs_keys<<<blocks, 256, 0, stream>>>(segs, nseg, ws->k_in, ws->v_in, residual_of);
    size_t bytes = (size_t)ws->tmp.bytes();
    cub::DeviceRadixSort::SortPairsDescending(ws->tmp.get(), bytes, ws->k_in.get(), ws->k_out.get(), ws->v_in.get(), ws->v_out.get(), (int)nseg,
                                              0, end_bit, stream);
    const bool fuse = do_kmer && fused_post != nullptr;
    k_cs_gather<<<blocks, 256, 0, stream>>>(segs, ws->k_out, ws->v_out, nseg, ws->sorted, fuse ? fused_post : nullptr);
    dim3 grid((unsigned)((max_len + 15 + CS_TILE - 1) / CS_TILE), (unsigned)((nseg + CS_GROUP - 1) / CS_GROUP));
    const SegD* sorted = ws->sorted;
    const int al = aligned ? 1 : 0;
    static const bool tma = getenv("FPL_CS_TMA") != nullptr && atoi(getenv("FPL_CS_TMA")) != 0;
    if (tma) {
        if (fuse) k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, true, true><<<grid, CS_NT_KMER, CS_SMEM_FUSED, stream>>>(seq, qual, sorted, nseg, stats, C, kmer_also, stats_post, 1u, al);
        else if (do_kmer) k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, true, false><<<grid, CS_NT_KMER, CS_SMEM_KMER, stream>>>(seq, qual, sorted, nseg, stats, C, kmer_also, nullptr, 1u, al);
        else k_cycle_stats<false, CS_NT_PLAIN, CS_DEPTH_PLAIN, true, false><<<grid, CS_NT_PLAIN, CS_SMEM_PLAIN, stream>>>(seq, qual, sorted, nseg, stats, C, nullptr, nullptr, 1u, al);
    } else {
        if (fuse) k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, false, true><<<grid, CS_NT_KMER, CS_SMEM_FUSED, stream>>>(seq, qual, sorted, nseg, stats, C, kmer_also, stats_post, 1u, al);
        else if (do_kmer) k_cycle_stats<true, CS_NT_KMER, CS_DEPTH_KMER, false, false><<<grid, CS_NT_KMER, CS_SMEM_KMER, stream>>>(seq, qual, sorted, nseg, stats, C, kmer_also, nullptr, 1u, al);
        else k_cycle_stats<false, CS_NT_PLAIN, CS_DEPTH_PLAIN, false, false><<<grid, CS_NT_PLAIN, CS_SMEM_PLAIN, stream>>>(seq, qual, sorted, nseg, stats, C, nullptr, nullptr, 1u, al);
    }
    launched += 3;                       // k_cs_keys, k_cs_gather (around the library's radix sort), k_cycle_stats
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// k_kmer_fix: the post-filter 5-mer table is the pre-filter one minus the 5-mers that do not lie inside a passing
// segment (trimmed ends, split gaps, failed or dropped reads).  A 5-mer ending at read position e (e >= 4) survives
// iff a passing segment [a, b) has a + 4 <= e < b (Stats::statRead skips the first four cycles of every read it is
// given, src/stats.cpp:309-311).  The removed ranges are short for almost every read.
// ------------------------------------------------------------------------------------------------------------------
#define KF_WARPS 8
#define KF_LONG 2048          // a removed range longer than this is shared by the block's warps
#define KF_LIST 16

namespace {
// the 5-mers ending at e in [from, to) of one read, strided over `nlanes` lanes (lane id `me`): rem[code]++
__device__ __forceinline__ void kmer_remove_one(const uint8_t* seq, int e, uint32_t rem_base) {
    const uint32_t c4 = kmer_code(seq[e - 4]), c3 = kmer_code(seq[e - 3]), c2 = kmer_code(seq[e - 2]),
                   c1 = kmer_code(seq[e - 1]), c0 = kmer_code(seq[e]);
    if (((c4 | c3 | c2 | c1 | c0) & 8u) == 0u)
        red_shared_add(rem_base + (((c4 << 8) | (c3 << 6) | (c2 << 4) | (c1 << 2) | c0) << 2), 1u);
}
__device__ __forceinline__ void kmer_remove_range(const uint8_t* seq, int from, int to, int me, int nlanes, uint32_t rem_base) {
    if (to - from <= 4 * nlanes) {            // the usual case: a trimmed end or a short gap
        for (int e = from + me; e < to; e += nlanes) kmer_remove_one(seq, e, rem_base);
        return;
    }
    // a long range: four positions per lane in flight (the loads of one round are independent; a lone warp walking a
    // long range is bound by their latency otherwise)
    int e0 = from + me;
    for (; e0 + 3 * nlanes < to; e0 += 4 * nlanes) {
        uint32_t c[4][5];
#pragma unroll
        for (int u = 0; u < 4; u++)
#pragma unroll
            for (int i = 0; i < 5; i++) c[u][i] = (uint32_t)seq[e0 + u * nlanes - 4 + i];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const uint32_t c4 = kmer_code(c[u][0]), c3 = kmer_code(c[u][1]), c2 = kmer_code(c[u][2]), c1 = kmer_code(c[u][3]),
                           c0 = kmer_code(c[u][4]);
            if (((c4 | c3 | c2 | c1 | c0) & 8u) == 0u)
                red_shared_add(rem_base + (((c4 << 8) | (c3 << 6) | (c2 << 4) | (c1 << 2) | c0) << 2), 1u);
        }
    }
    for (; e0 < to; e0 += nlanes) kmer_remove_one(seq, e0, rem_base);
}
}  // namespace

__global__ void __launch_bounds__(KF_WARPS * 32)
k_kmer_fix(DevBatch b, const fpl_read_result* __restrict__ res, unsigned long long* __restrict__ post_kmer) {
    __shared__ uint32_t rem[1024];
    __shared__ int n_long;
    __shared__ long long long_off[KF_LIST];
    __shared__ int long_from[KF_LIST], long_to[KF_LIST];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) rem[i] = 0;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const uint32_t rem_base = shared_addr(&rem[0]);
    const int64_t nwarps = (int64_t)gridDim.x * KF_WARPS;
    for (int64_t r = (int64_t)blockIdx.x * KF_WARPS + wid; r < b.n_reads; r += nwarps) {
        const int L = b.lens[r];
        if (L < 5) continue;
        const uint8_t* seq = b.seq + b.offsets[r];
        const fpl_read_result* o = &res[r];
        // kept intervals of ending positions, in read order
        int ks[2], ke[2], nk = 0;
        const int nseg = o->n_segments;
        for (int k = 0; k < nseg; k++)
            if (o->seg_result[k] == FPL_PASS_FILTER) { ks[nk] = o->seg_lo[k] + 4; ke[nk] = o->seg_lo[k] + o->seg_len[k]; nk++; }
        // removed ranges: [4, ks0) [ke0, ks1) [ke1, L)
        int from = 4;
        for (int k = 0; k <= nk; k++) {
            const int to = k < nk ? min(ks[k], L) : L;
            if (to - from > KF_LONG) {
                // a failed long read, or the gap between two far-apart adapter hits of an ultra-long read: the block's
                // warps share it after the loop (a lone warp would walk it at the latency of its loads)
                int slot = -1;
                if (lane == 0) slot = atomicAdd(&n_long, 1);
                slot = __shfl_sync(0xffffffffu, slot, 0);
                if (slot < KF_LIST) {
                    if (lane == 0) { long_off[slot] = b.offsets[r]; long_from[slot] = from; long_to[slot] = to; }
                } else {
                    kmer_remove_range(seq, from, to, lane, 32, rem_base);
                }
            } else {
                kmer_remove_range(seq, from, to, lane, 32, rem_base);
            }
            // the next removed range starts behind this one and behind the segment; a passing segment shorter than
            // four bases (only possible with --length_required < 5) ends in front of `to` and must not pull it back
            if (k < nk) from = max(from, max(to, ke[k]));
        }
    }
    __syncthreads();
    const int nl = min(n_long, KF_LIST);
    for (int i = 0; i < nl; i++)
        kmer_remove_range(b.seq + long_off[i], long_from[i], long_to[i], threadIdx.x, KF_WARPS * 32, rem_base);
    __syncthreads();
    for (int i = threadIdx.x; i < 1024; i += blockDim.x)
        if (rem[i]) atomicAdd(&post_kmer[i], 0ull - (unsigned long long)rem[i]);
}

void launch_kmer_fix(const DevBatch& b, const fpl_read_result* res, unsigned long long* post_kmer, cudaStream_t stream, int& launched) {
    if (b.n_reads == 0) return;
    const int64_t want = (b.n_reads + KF_WARPS - 1) / KF_WARPS;
    const unsigned grid = (unsigned)(want < FPL_NUM_SMS * 16 ? want : FPL_NUM_SMS * 16);
    k_kmer_fix<<<grid, KF_WARPS * 32, 0, stream>>>(b, res, post_kmer);
    launched++;
}

// ------------------------------------------------------------------------------------------------------------------
#define RQ_WARPS 8

namespace {
// median: smallest char m with sum_{c<=m} hist[c] > len>>1 (src/stats.cpp:351-361); lane l owns bins 4l..4l+3
__device__ __forceinline__ uint8_t hist_median(const uint32_t* h, int len, int lane, uint32_t (&own)[4]) {
    own[0] = h[4 * lane]; own[1] = h[4 * lane + 1]; own[2] = h[4 * lane + 2]; own[3] = h[4 * lane + 3];
    if (len <= 0) return 0;
    const int half = len >> 1;
    const int tot = (int)(own[0] + own[1] + own[2] + own[3]);
    int run = warp_incl_scan(tot) - tot;
    int m = 1 << 30;
    run += own[0]; if (run > half) m = min(m, 4 * lane);
    run += own[1]; if (run > half) m = min(m, 4 * lane + 1);
    run += own[2]; if (run > half) m = min(m, 4 * lane + 2);
    run += own[3]; if (run > half) m = min(m, 4 * lane + 3);
    return (uint8_t)__reduce_min_sync(0xffffffffu, m);
}

// h[q] += delta for the bytes qp[0..n): 16-byte vector body, byte head/tail (delta = 1 or 0xFFFFFFFF)
__device__ __forceinline__ void hist_vec(uint32_t hbase, const uint4& v, uint32_t delta) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        // bin address = hbase + 4 * (byte & 127): one dp4a per byte (weight 4 on that byte) on the FMA pipe, after one
        // LOP3 per word that keeps the bytes inside the 128-bin table
        const uint32_t m = w[k] & 0x7f7f7f7fu;
#pragma unroll
        for (int j = 0; j < 4; j++) red_shared_add(__dp4a(m, 4u << (8 * j), hbase), delta);
    }
}
// h[q] += delta for the bytes qp[0..n) (delta = 1 or 0xFFFFFFFF): 16-byte vector body, byte head/tail; the work is
// strided over `nth` threads, this one being `me` (a warp: lane / 32; a whole block: threadIdx.x / blockDim.x)
__device__ __forceinline__ void hist_bytes(uint32_t hbase, const uint8_t* qp, int n, uint32_t delta, int me, int nth) {
    const int head = min(n, (int)((16 - (reinterpret_cast<uintptr_t>(qp) & 15)) & 15));
    if (me < head) red_shared_add(hbase + ((uint32_t)(qp[me] & 127) << 2), delta);
    const int nvec = (n - head) >> 4;
    const uint4* vp = reinterpret_cast<const uint4*>(qp + head);
    // four vectors per thread in flight: a warp alone keeps 2 KB of loads outstanding (the kernel is latency-bound otherwise)
    int i = me;
    for (; i + 3 * nth < nvec; i += 4 * nth) {
        const uint4 v0 = __ldg(vp + i), v1 = __ldg(vp + i + nth), v2 = __ldg(vp + i + 2 * nth), v3 = __ldg(vp + i + 3 * nth);
        hist_vec(hbase, v0, delta); hist_vec(hbase, v1, delta); hist_vec(hbase, v2, delta); hist_vec(hbase, v3, delta);
    }
    for (; i < nvec; i += nth) hist_vec(hbase, __ldg(vp + i), delta);
    const int done = head + (nvec << 4);
    if (me < 16 && done + me < n) red_shared_add(hbase + ((uint32_t)(qp[done + me] & 127) << 2), delta);   // < 16 tail bytes
}

// One read: the histogram of the whole read gives the pre-filter median and mBaseQualHistogram; the histogram of each
// passing segment is derived from it by subtracting the (short) removed ends — or counted directly when the segment is
// the smaller part — and gives the post-filter median and histogram.  One pass over the quality bytes serves both Stats
// objects.  COOP = false: one warp owns the read.  COOP = true: the whole block does (an ultra-long read streamed by
// one warp is bound by the latency of that warp's loads); every thread of the block calls it for the same read, the
// histograms are warp 0's, warp 0 does the medians.
// EXC (k_read_qual_exc, a read k_final listed): k_scan_jit has already counted an alive read's whole histogram into the
// pre-filter sums and its window's into the post-filter ones, and set its pre-filter median.  Such a read histograms its
// window instead of the whole read, takes it out of the post-filter sums (block_sub) and counts its passing segments
// as above, relative to the window; a read that is not alive gets the pre-filter part in full.  The per-read sums
// (reads, lengths, median histograms) are k_count's in this mode.
template <bool COOP, bool EXC = false>
__device__ __forceinline__ void read_qual_one(const DevBatch& b, int64_t r, uint32_t* hfull, uint32_t* hseg, uint32_t (*block_hist)[128],
                                              unsigned long long (*block_misc)[2], unsigned long long* const* tail,
                                              fpl_read_result* __restrict__ res, bool pre_only,
                                              const ReadState* __restrict__ st = nullptr, uint32_t* block_sub = nullptr) {
    const int lane = lane_id(), wid = threadIdx.x >> 5;
    const int me = COOP ? (int)threadIdx.x : lane, nth = COOP ? (int)blockDim.x : 32;
    auto sync = [] { if (COOP) __syncthreads(); else __syncwarp(); };
    const bool lead = !COOP || wid == 0;                 // the warp that owns the medians and the flushes
    const uint32_t hfull_s = shared_addr(hfull), hseg_s = shared_addr(hseg);
    const int Lread = b.lens[r];
    fpl_read_result* o = &res[r];
    bool win = false;                                    // EXC: hfull is the window [w0, w0 + L) of an alive read
    int w0 = 0, L = Lread;
    if (EXC) {
        const ReadState s = st[r];
        if (s.alive) { win = true; w0 = s.lo; L = s.len; }
    }
    const uint8_t* qp = b.qual + b.offsets[r] + w0;
    sync();
    for (int i = me; i < 128; i += nth) hfull[i] = 0;
    sync();
    hist_bytes(hfull_s, qp, L, 1u, me, nth);
    sync();
    uint32_t own[4];
    if (lead) {
        if (win) {
            own[0] = hfull[4 * lane]; own[1] = hfull[4 * lane + 1]; own[2] = hfull[4 * lane + 2]; own[3] = hfull[4 * lane + 3];
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (own[k]) atomicAdd(&block_sub[4 * lane + k], own[k]);
        } else {
            const uint8_t med = hist_median(hfull, L, lane, own);
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (own[k]) atomicAdd(&block_hist[0][4 * lane + k], own[k]);
            if (lane == 0) {
                if (!EXC) {
                    atomicAdd(&block_misc[0][0], 1ull);
                    atomicAdd(&block_misc[0][1], (unsigned long long)L);
                    if (L > 0) {
                        atomicAdd(&tail[0][FPL_STATS_MEDHIST + med], 1ull);
                        atomicAdd(&tail[0][FPL_STATS_MEDBASES + med], (unsigned long long)L);
                    }
                }
                o->pre_median_qual = med;
            }
        }
    }
    const int nseg = pre_only ? 0 : o->n_segments;   // --mask/--break: the post-filter part is k_ext_seg_qual's
    for (int k = 0; k < nseg; k++) {
        if (o->seg_result[k] != FPL_PASS_FILTER) continue;      // uniform
        const int a = o->seg_lo[k] - w0, n = o->seg_len[k];
        sync();
        if (L - n <= n) {            // copy the read's histogram and take the removed ends out
            for (int i = me; i < 128; i += nth) hseg[i] = hfull[i];
            sync();
            hist_bytes(hseg_s, qp, a, 0xFFFFFFFFu, me, nth);
            hist_bytes(hseg_s, qp + a + n, L - a - n, 0xFFFFFFFFu, me, nth);
        } else {
            for (int i = me; i < 128; i += nth) hseg[i] = 0;
            sync();
            hist_bytes(hseg_s, qp + a, n, 1u, me, nth);
        }
        sync();
        if (lead) {
            const uint8_t smed = hist_median(hseg, n, lane, own);
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (own[j]) atomicAdd(&block_hist[1][4 * lane + j], own[j]);
            if (lane == 0) {
                if (!EXC) {
                    atomicAdd(&block_misc[1][0], 1ull);
                    atomicAdd(&block_misc[1][1], (unsigned long long)n);
                    if (n > 0) {
                        atomicAdd(&tail[1][FPL_STATS_MEDHIST + smed], 1ull);
                        atomicAdd(&tail[1][FPL_STATS_MEDBASES + smed], (unsigned long long)n);
                    }
                }
                o->seg_median_qual[k] = smed;
            }
        }
    }
    sync();
}
}  // namespace

#define RQ_LONG (96 * 1024)      // reads longer than this are streamed by the whole block
#define RQ_LIST 24

// Shared-memory atomics are the fast way to histogram on this part (tools/ubench_hist.cu: a 128-bin table updated
// with atomicAdd by 8 warps streams quality bytes at HBM speed, 4x faster than lane-private read-modify-write).
__global__ void __launch_bounds__(RQ_WARPS * 32)
k_read_qual(DevBatch b, unsigned long long* __restrict__ stats_pre, unsigned long long* __restrict__ stats_post, int64_t C,
            fpl_read_result* __restrict__ res, bool pre_only) {
    __shared__ uint32_t hist[RQ_WARPS][2][128];        // per warp: [0] whole read, [1] current segment
    __shared__ uint32_t block_hist[2][128];            // this block's reads -> one flush per Stats block
    __shared__ unsigned long long block_misc[2][2];    // reads, length sum
    __shared__ int n_long;
    __shared__ long long long_read[RQ_LIST];
    const int wid = threadIdx.x >> 5, lane = lane_id();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) (&block_hist[0][0])[i] = 0;
    if (threadIdx.x < 4) (&block_misc[0][0])[threadIdx.x] = 0;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    unsigned long long* tail[2] = {stats_pre + 16 * C, stats_post + 16 * C};
    const int64_t nwarps = (int64_t)gridDim.x * RQ_WARPS;
    for (int64_t r = (int64_t)blockIdx.x * RQ_WARPS + wid; r < b.n_reads; r += nwarps) {
        if (b.lens[r] > RQ_LONG) {
            int slot = -1;
            if (lane == 0) slot = atomicAdd(&n_long, 1);
            slot = __shfl_sync(0xffffffffu, slot, 0);
            if (slot < RQ_LIST) { if (lane == 0) long_read[slot] = r; continue; }
        }
        read_qual_one<false>(b, r, hist[wid][0], hist[wid][1], block_hist, block_misc, tail, res, pre_only);
    }
    __syncthreads();
    const int nl = min(n_long, RQ_LIST);
    for (int i = 0; i < nl; i++)
        read_qual_one<true>(b, long_read[i], hist[0][0], hist[0][1], block_hist, block_misc, tail, res, pre_only);
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        const int which = i >> 7, bin = i & 127;
        if (block_hist[which][bin]) atomicAdd(&tail[which][FPL_STATS_QUALHIST + bin], (unsigned long long)block_hist[which][bin]);
    }
    if (threadIdx.x < 2 && block_misc[threadIdx.x][0]) {
        atomicAdd(&tail[threadIdx.x][FPL_STATS_READS], block_misc[threadIdx.x][0]);
        atomicAdd(&tail[threadIdx.x][FPL_STATS_LENSUM], block_misc[threadIdx.x][1]);
    }
}

void launch_read_qual(const DevBatch& b, unsigned long long* stats_pre, unsigned long long* stats_post, int64_t C,
                      fpl_read_result* res, bool pre_only, cudaStream_t stream, int& launched) {
    if (b.n_reads == 0) return;
    // persistent-ish grid: enough blocks to fill the GPU several times over, each warp strides over the reads
    const int64_t want = (b.n_reads + RQ_WARPS - 1) / RQ_WARPS;
    const unsigned grid = (unsigned)(want < FPL_NUM_SMS * 64 ? want : FPL_NUM_SMS * 64);
    k_read_qual<<<grid, RQ_WARPS * 32, 0, stream>>>(b, stats_pre, stats_post, C, res, pre_only);
    launched++;
}

// k_read_qual's work for the reads k_final listed (exc[0, *n_exc)) when k_scan_jit counted the quality histograms: the
// exceptions to "the read's one passing segment is its window" (see read_qual_one<_, true>).  The grid is capped and the
// count is read on the device.  block_sub: the windows' histograms, taken out of the post-filter sums.
__global__ void __launch_bounds__(RQ_WARPS * 32)
k_read_qual_exc(DevBatch b, const ReadState* __restrict__ st, const int32_t* __restrict__ exc, const int* __restrict__ n_exc,
                unsigned long long* __restrict__ stats_pre, unsigned long long* __restrict__ stats_post, int64_t C,
                fpl_read_result* __restrict__ res) {
    __shared__ uint32_t hist[RQ_WARPS][2][128];
    __shared__ uint32_t block_hist[2][128];
    __shared__ uint32_t block_sub[128];
    __shared__ int n_long;
    __shared__ long long long_read[RQ_LIST];
    const int wid = threadIdx.x >> 5, lane = lane_id();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) (&block_hist[0][0])[i] = 0;
    for (int i = threadIdx.x; i < 128; i += blockDim.x) block_sub[i] = 0;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    unsigned long long* tail[2] = {stats_pre + 16 * C, stats_post + 16 * C};
    const int64_t n = *n_exc;
    const int64_t nwarps = (int64_t)gridDim.x * RQ_WARPS;
    for (int64_t i = (int64_t)blockIdx.x * RQ_WARPS + wid; i < n; i += nwarps) {
        const int64_t r = exc[i];
        if (b.lens[r] > RQ_LONG) {
            int slot = -1;
            if (lane == 0) slot = atomicAdd(&n_long, 1);
            slot = __shfl_sync(0xffffffffu, slot, 0);
            if (slot < RQ_LIST) { if (lane == 0) long_read[slot] = r; continue; }
        }
        read_qual_one<false, true>(b, r, hist[wid][0], hist[wid][1], block_hist, nullptr, tail, res, false, st, block_sub);
    }
    __syncthreads();
    const int nl = min(n_long, RQ_LIST);
    for (int i = 0; i < nl; i++)
        read_qual_one<true, true>(b, long_read[i], hist[0][0], hist[0][1], block_hist, nullptr, tail, res, false, st, block_sub);
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        const int which = i >> 7, bin = i & 127;
        if (block_hist[which][bin]) atomicAdd(&tail[which][FPL_STATS_QUALHIST + bin], (unsigned long long)block_hist[which][bin]);
    }
    for (int i = threadIdx.x; i < 128; i += blockDim.x)
        if (block_sub[i]) atomicAdd(&tail[1][FPL_STATS_QUALHIST + i], 0ull - (unsigned long long)block_sub[i]);
}

void launch_read_qual_exc(const DevBatch& b, const ReadState* st, const int32_t* exc, const int* n_exc, unsigned long long* stats_pre,
                          unsigned long long* stats_post, int64_t C, fpl_read_result* res, cudaStream_t stream, int& launched) {
    if (b.n_reads == 0) return;
    // the list is a few percent of the reads: a grid of a few blocks per SM, capped by what the whole batch would need
    const int64_t want = (b.n_reads + RQ_WARPS - 1) / RQ_WARPS;
    const unsigned grid = (unsigned)(want < FPL_NUM_SMS * 8 ? want : FPL_NUM_SMS * 8);
    k_read_qual_exc<<<grid, RQ_WARPS * 32, 0, stream>>>(b, st, exc, n_exc, stats_pre, stats_post, C, res);
    launched++;
}

// the striped sums of k_scan_jit's histograms ([QH_STRIPES][2][128]: whole reads, windows) -> mBaseQualHistogram of the
// pre-filter and of the post-filter block; one thread per (block, bin)
__global__ void k_qhist_fold(const unsigned long long* __restrict__ stripes, int n_stripes, unsigned long long* __restrict__ stats_pre,
                             unsigned long long* __restrict__ stats_post, int64_t C) {
    const int i = threadIdx.x;           // 256 threads
    unsigned long long sum = 0;
    for (int k = 0; k < n_stripes; k++) sum += stripes[(int64_t)k * 256 + i];
    if (sum) atomicAdd(&((i >> 7) ? stats_post : stats_pre)[16 * C + FPL_STATS_QUALHIST + (i & 127)], sum);
}

void launch_qhist_fold(const unsigned long long* stripes, int n_stripes, unsigned long long* stats_pre, unsigned long long* stats_post,
                       int64_t C, cudaStream_t stream, int& launched) {
    k_qhist_fold<<<1, 256, 0, stream>>>(stripes, n_stripes, stats_pre, stats_post, C);
    launched++;
}

// pre-stats segment list: every input read, full length
__global__ void k_make_preseg(DevBatch b, StatSeg* __restrict__ segs) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= b.n_reads) return;
    StatSeg s;
    s.off = b.offsets[r]; s.len = b.lens[r]; s.read = (int)r; s.slot = 2; s.pad = 0;
    segs[r] = s;
}

void launch_make_preseg(const DevBatch& b, StatSeg* segs, cudaStream_t stream, int& launched) {
    if (b.n_reads == 0) return;
    k_make_preseg<<<(unsigned)((b.n_reads + 255) / 256), 256, 0, stream>>>(b, segs);
    launched++;
}

// ------------------------------------------------------------------------------------------------------------------
// The per-cycle curves of the JSON report (fpl_report_json; Stats::summarize src/stats.cpp:150-256 computes them,
// Stats::reportJson :473-548 prints them with ostream <<, i.e. "%.6g").  A cycle's eleven values depend on that cycle's
// sixteen counters only, so the text is a per-cycle map and a stream compaction:
//   k_report_cycles  per Stats block: total_cycles (the first cycle whose count over the 8 bins is 0), total bases, G+C
//   k_report_sizes   thread per cycle: the bytes of its 11 values (with the ',' behind all but a curve's last)
//   cub scan         -> where each value starts
//   k_report_text    thread per cycle: the 11 values at their places; k_report_frame drops the host-built JSON frame
//                    around the 22 curves
// ------------------------------------------------------------------------------------------------------------------

// The curve values exactly as the reference's doubles are computed: tot / totq over the 8 bins, IEEE division,
// round-to-nearest int64 -> double.  curve 0..4: quality A, T (U with is_rna), C, G, mean; 5..10: content A, T (U), C, G,
// N, GC.  blk is one FPL_STATS_WORDS(C) block.
__device__ __forceinline__ double report_value(const unsigned long long* blk, int64_t C, int64_t c, int curve, int is_rna) {
    long long tot = 0, totq = 0;
    for (int b = 0; b < 8; b++) {
        tot += (long long)blk[b * C + c];
        totq += (long long)blk[(8 + b) * C + c];
    }
    const double mean = (double)totq / (double)tot;
    if (curve == 4) return mean;
    const int tbin = is_rna ? ('U' & 7) : ('T' & 7);
    if (curve < 4) {
        const int b = curve == 0 ? ('A' & 7) : curve == 1 ? tbin : curve == 2 ? ('C' & 7) : ('G' & 7);
        const long long n = (long long)blk[b * C + c];
        return n == 0 ? mean : (double)(long long)blk[(8 + b) * C + c] / (double)n;
    }
    if (curve == 10) return (double)((long long)blk[('G' & 7) * C + c] + (long long)blk[('C' & 7) * C + c]) / (double)tot;
    const int k = curve - 5;
    const int b = k == 0 ? ('A' & 7) : k == 1 ? tbin : k == 2 ? ('C' & 7) : k == 3 ? ('G' & 7) : ('N' & 7);
    return (double)(long long)blk[b * C + c] / (double)tot;
}

// v as printf("%.6g") / libstdc++'s default ostream << double prints it, into out (at most 12 bytes); returns the length.
// Integer-only and exact on the domain of the curves: 0 and 2^-64 <= |v| < 10^6.  |v| = m * 2^e2 with a 53-bit m (exact
// scaling by powers of two), six significant digits = |v| * 10^k = m * 5^k * 2^(e2 + k) in 128 bits, rounded half to even;
// the decimal exponent estimated from the binary one is corrected by exact comparison with 10^5 and 10^6.
__device__ __forceinline__ int fmt_g6(double v, char* out) {
    if (v == 0) { out[0] = '0'; return 1; }
    int n = 0;
    double a = v;
    if (a < 0) { out[n++] = '-'; a = -a; }
    int e2 = 0;
    while (a < 2097152.0) { a *= 4294967296.0; e2 -= 32; }              // a in [2^21, 2^53)
    const int p = 63 - __clzll((long long)(unsigned long long)a);        // its leading bit
    a *= (double)(1ull << (52 - p));
    e2 -= 52 - p;
    const unsigned long long m = (unsigned long long)a;                  // 2^52 <= m < 2^53, |v| = m * 2^e2
    int E = ((e2 + 52) * 78913) >> 18;                                   // floor(log10(2^(e2+52))), may be 1 short
    E = E < -21 ? -21 : E > 5 ? 5 : E;
    unsigned long long q = 0;
    unsigned __int128 P = 0;
    int s = 0;
    for (int it = 0; it < 4; it++) {
        const int k = 5 - E;                                             // 0 <= k <= 26: 5^k < 2^61
        unsigned long long p5 = 1;
        for (int i = 0; i < k; i++) p5 *= 5;
        P = (unsigned __int128)m * p5;                                   // |v| * 10^k = P * 2^-s
        s = -(e2 + k);
        q = s >= 128 ? 0 : (unsigned long long)(P >> s);
        if (q >= 1000000ull && E < 5) { E++; continue; }
        if (q < 100000ull && E > -21) { E--; continue; }
        break;
    }
    if (s > 0 && s < 128) {                                              // round half to even
        const unsigned __int128 rem = P - ((unsigned __int128)q << s), half = (unsigned __int128)1 << (s - 1);
        if (rem > half || (rem == half && (q & 1))) q++;
    }
    if (q >= 1000000ull) { q /= 10; E++; }                               // 999999.5 -> 100000, one decade up
    char d[6];
    for (int i = 5; i >= 0; i--) { d[i] = (char)('0' + q % 10); q /= 10; }
    int nd = 6;
    while (nd > 1 && d[nd - 1] == '0') nd--;                             // %g drops trailing zeros
    if (E < -4 || E >= 6) {
        out[n++] = d[0];
        if (nd > 1) { out[n++] = '.'; for (int i = 1; i < nd; i++) out[n++] = d[i]; }
        out[n++] = 'e';
        out[n++] = E < 0 ? '-' : '+';
        const int ae = E < 0 ? -E : E;
        out[n++] = (char)('0' + ae / 10);
        out[n++] = (char)('0' + ae % 10);
    } else if (E >= 0) {
        for (int i = 0; i <= E; i++) out[n++] = d[i];
        if (nd > E + 1) { out[n++] = '.'; for (int i = E + 1; i < nd; i++) out[n++] = d[i]; }
    } else {
        out[n++] = '0'; out[n++] = '.';
        for (int i = 0; i < -E - 1; i++) out[n++] = '0';
        for (int i = 0; i < nd; i++) out[n++] = d[i];
    }
    return n;
}

namespace {

// sum[3w + 0] = total_cycles of block w (initialised to C by the host), [3w + 1] = its bases, [3w + 2] = its G + C.  Cycle
// counts never increase with the cycle, so every count of the block lies before total_cycles.
__global__ void k_report_cycles(const unsigned long long* __restrict__ pre, const unsigned long long* __restrict__ post, int64_t C,
                                unsigned long long* __restrict__ sum) {
    const unsigned long long* blk = blockIdx.y ? post : pre;
    unsigned long long bases = 0, gc = 0, first = (unsigned long long)C;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long t = 0;
        for (int b = 0; b < 8; b++) t += blk[b * C + c];
        bases += t;
        gc += blk[('G' & 7) * C + c] + blk[('C' & 7) * C + c];
        if (t == 0 && (unsigned long long)c < first) first = (unsigned long long)c;
    }
    for (int o = 16; o > 0; o >>= 1) {
        bases += __shfl_down_sync(0xffffffffu, bases, o);
        gc += __shfl_down_sync(0xffffffffu, gc, o);
        const unsigned long long f = __shfl_down_sync(0xffffffffu, first, o);
        first = f < first ? f : first;
    }
    if (lane_id() == 0) {
        unsigned long long* s = sum + 3 * blockIdx.y;
        if (first < (unsigned long long)C) atomicMin(&s[0], first);
        if (bases) atomicAdd(&s[1], bases);
        if (gc) atomicAdd(&s[2], gc);
    }
}

// the values of block w live at [base_w + curve * T_w + c) of the size / offset vectors
__device__ __forceinline__ bool report_cycle(const ReportCurves& R, int64_t i, int& w, int64_t& c) {
    if (i < R.T[0]) { w = 0; c = i; return true; }
    if (i < R.T[0] + R.T[1]) { w = 1; c = i - R.T[0]; return true; }
    return false;
}

__global__ void k_report_sizes(const ReportCurves R, int64_t* __restrict__ size) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int w; int64_t c;
    if (!report_cycle(R, i, w, c)) return;
    const int64_t T = R.T[w], base = w ? 11 * R.T[0] : 0;
    char buf[16];
    for (int k = 0; k < 11; k++)
        size[base + k * T + c] = fmt_g6(report_value(R.blk[w], R.C, c, k, R.is_rna), buf) + (c + 1 < T ? 1 : 0);
}

// off: exclusive sum of the sizes; curve j (block j / 11, curve j % 11) lands behind frame pieces 0..j: shift[j] bytes of frame
__global__ void k_report_text(const ReportCurves R, const int64_t* __restrict__ off, uint8_t* __restrict__ text) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int w; int64_t c;
    if (!report_cycle(R, i, w, c)) return;
    const int64_t T = R.T[w], base = w ? 11 * R.T[0] : 0;
    char buf[16];
    for (int k = 0; k < 11; k++) {
        const int64_t j = base + k * T + c;
        uint8_t* dst = text + off[j] + R.shift[11 * w + k];
        const int n = fmt_g6(report_value(R.blk[w], R.C, c, k, R.is_rna), buf);
        for (int b = 0; b < n; b++) dst[b] = (uint8_t)buf[b];
        if (c + 1 < T) dst[n] = ',';
    }
}

// frame piece j = frame[src[j], src[j + 1]) goes to text + dst[j]; block j copies piece j
__global__ void k_report_frame(const uint8_t* __restrict__ frame, const int64_t* __restrict__ src, const int64_t* __restrict__ dst,
                               uint8_t* __restrict__ text) {
    const int j = blockIdx.x;
    for (int64_t b = threadIdx.x; b < src[j + 1] - src[j]; b += blockDim.x) text[dst[j] + b] = frame[src[j] + b];
}

}  // namespace

void launch_report_cycles(const unsigned long long* pre, const unsigned long long* post, int64_t C, unsigned long long* sum,
                          cudaStream_t stream, int& launched) {
    const int64_t want = (C + 255) / 256;
    k_report_cycles<<<dim3((unsigned)(want < FPL_NUM_SMS * 8 ? want : FPL_NUM_SMS * 8), 2), 256, 0, stream>>>(pre, post, C, sum);
    launched++;
}

void launch_report_sizes(const ReportCurves& R, int64_t* size, cudaStream_t stream, int& launched) {
    const int64_t n = R.T[0] + R.T[1];
    if (n) k_report_sizes<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(R, size);
    launched += n != 0;
}

void launch_report_text(const ReportCurves& R, const int64_t* off, const uint8_t* frame, const int64_t* src, const int64_t* dst,
                        int n_pieces, uint8_t* text, cudaStream_t stream, int& launched) {
    k_report_frame<<<n_pieces, 256, 0, stream>>>(frame, src, dst, text);
    const int64_t n = R.T[0] + R.T[1];
    if (n) k_report_text<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(R, off, text);
    launched += n ? 2 : 1;
}

// ------------------------------------------------------------------------------------------------------------------
// fpl_report_html (HtmlReporter::report, src/htmlreporter.cpp:75-253).  What grows with the input is printed here:
//   k_html_capture   on the processing path (fpl_keep_read_lists): appends each call's (length, median) entries of both
//                    Stats blocks — input order, then output-read order within a read — to the context's lists
//   k_html_hist      grouping by median, stable: per-warp 130-bin histograms of contiguous chunks (medians 0..127, empty
//   cub scan         reads, post-filter slots without an output read), the exclusive sum of the bin-major matrix,
//   k_html_scatter   and a scatter that ranks equal bins inside a warp by ballots, 32 entries at a time in chunk order:
//                    mQualLength's iteration order (a map<char, vector<int>>: ascending median, then statRead order)
//   k_html_len*      Stats::calcLengthHistogram (src/stats.cpp:377-409): a length histogram, scans of the counts and of
//                    the int * int products (wrapped to 32 bits, as the reference's imul is), and the first keys that pass
//   k_html_bins      mBaseContents of each bin over the block's total_cycles (the content curves' names)
//   k_html_values    the 11 per-cycle curves (report_value), then k_html_sums: one thread per (curve, range) of
//                    Stats::list2string's down-sampling (:550-573), the range summed in order in double
//   k_html_sizes / cub scan / k_html_text: every value's text at its place; k_report_frame drops the host-built frame
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int html_bin(const HtmlEntry& e) { return e.len < 0 ? 129 : e.len == 0 ? 128 : (e.med & 127); }

__device__ __forceinline__ int html_itoa(long long v, char* out) {
    char d[24];
    int n = 0, k = 0;
    unsigned long long a = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
    do { d[k++] = (char)('0' + a % 10); a /= 10; } while (a);
    if (v < 0) out[n++] = '-';
    while (k) out[n++] = d[--k];
    return n;
}

namespace {

__global__ void k_html_capture(const fpl_read_result* __restrict__ res, const int32_t* __restrict__ lens, int64_t n,
                               const fpl_segment* __restrict__ segs, int64_t n_segs, HtmlEntry* __restrict__ pre,
                               HtmlEntry* __restrict__ post) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const fpl_read_result& r = res[i];
        pre[i] = HtmlEntry{lens[i], r.pre_median_qual};
        if (!segs)
            for (int k = 0; k < 2; k++) {
                const bool out = k < r.n_segments && r.seg_result[k] == FPL_PASS_FILTER;
                post[2 * i + k] = out ? HtmlEntry{r.seg_len[k], r.seg_median_qual[k]} : HtmlEntry{-1, 0};
            }
    }
    if (segs)
        for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_segs; j += stride) {
            const fpl_segment& s = segs[j];
            post[j] = s.result == FPL_PASS_FILTER ? HtmlEntry{s.len, s.median_qual} : HtmlEntry{-1, 0};
        }
}

// warp w of block b owns chunk 4b + w: mat[bin * nchunks + chunk] = its entries of that bin
__global__ void k_html_hist(const HtmlEntry* __restrict__ e, int64_t n, int64_t nchunks, long long* __restrict__ mat) {
    __shared__ int h[4][HTML_BINS];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t chunk = (int64_t)blockIdx.x * 4 + wid;
    if (chunk >= nchunks) return;
    for (int b = lane; b < HTML_BINS; b += 32) h[wid][b] = 0;
    __syncwarp();
    const int64_t lo = chunk * HTML_CHUNK, hi = lo + HTML_CHUNK < n ? lo + HTML_CHUNK : n;
    for (int64_t i = lo + lane; i < hi; i += 32) atomicAdd(&h[wid][html_bin(e[i])], 1);
    __syncwarp();
    for (int b = lane; b < HTML_BINS; b += 32) mat[(int64_t)b * nchunks + chunk] = h[wid][b];
}

// off: the exclusive sum of mat.  32 entries at a time, in order: an entry's rank among the equal bins of lower lanes comes
// from 8 ballots (one per bit of the bin), the lowest lane of each bin then moves that bin's cursor
__global__ void k_html_scatter(const HtmlEntry* __restrict__ e, int64_t n, int64_t nchunks, const long long* __restrict__ off,
                               HtmlEntry* __restrict__ out) {
    __shared__ long long cur[4][HTML_BINS];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t chunk = (int64_t)blockIdx.x * 4 + wid;
    if (chunk >= nchunks) return;
    for (int b = lane; b < HTML_BINS; b += 32) cur[wid][b] = off[(int64_t)b * nchunks + chunk];
    __syncwarp();
    const int64_t lo = chunk * HTML_CHUNK, hi = lo + HTML_CHUNK < n ? lo + HTML_CHUNK : n;
    for (int64_t i0 = lo; i0 < hi; i0 += 32) {
        const int64_t i = i0 + lane;
        const bool ok = i < hi;
        const HtmlEntry v = ok ? e[i] : HtmlEntry{0, 0};
        const int key = ok ? html_bin(v) : 255;
        unsigned peers = 0xffffffffu;
        for (int bit = 0; bit < 8; bit++) {
            const unsigned m = __ballot_sync(0xffffffffu, (key >> bit) & 1);
            peers &= ((key >> bit) & 1) ? m : ~m;
        }
        const unsigned lower = peers & ((1u << lane) - 1u);
        if (ok) out[cur[wid][key] + __popc(lower)] = v;
        __syncwarp();
        if (ok && lower == 0) cur[wid][key] += __popc(peers);
        __syncwarp();
    }
}

__global__ void k_html_lenhist(const HtmlEntry* __restrict__ e, int64_t n, unsigned long long* __restrict__ hist) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int len = e[i].len;
        if (len >= 0) atomicAdd(&hist[len], 1ull);
    }
}

// totalBase += iter->first * iter->second: an int * int product, wrapped to 32 bits before it is added
__global__ void k_html_lenprod(const unsigned long long* __restrict__ cnt, int64_t H, long long* __restrict__ prod) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < H) prod[b] = (long long)(int32_t)((uint32_t)b * (uint32_t)cnt[b]);
}

// out: min, max, median, N50 length.  A key of 0 that passes sets its value to 0, which the next key overwrites: the
// answer is the smallest POSITIVE key whose running sum passes.
__global__ void k_html_lensearch(const unsigned long long* __restrict__ cnt, const long long* __restrict__ ccum,
                                 const long long* __restrict__ prod, const long long* __restrict__ pcum, int64_t H,
                                 long long half_sum, unsigned long long half_n, int* __restrict__ out) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= H || cnt[b] == 0) return;
    atomicMin(&out[0], (int)b);
    atomicMax(&out[1], (int)b);
    if (b == 0) return;
    if ((unsigned long long)(ccum[b] + (long long)cnt[b]) > half_n) atomicMin(&out[2], (int)b);
    if (pcum[b] + prod[b] > half_sum) atomicMin(&out[3], (int)b);
}

// out[b] += the block's count of base bin b over cycles [0, T)
__global__ void k_html_bins(const unsigned long long* __restrict__ blk, int64_t C, int64_t T, unsigned long long* __restrict__ out) {
    unsigned long long s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < T; c += (int64_t)gridDim.x * blockDim.x)
        for (int b = 0; b < 8; b++) s[b] += blk[b * C + c];
    for (int b = 0; b < 8; b++) {
        unsigned long long v = s[b];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane_id() == 0 && v) atomicAdd(&out[b], v);
    }
}

__global__ void k_html_values(const unsigned long long* __restrict__ blk, int64_t C, int64_t T, int is_rna, double* __restrict__ vals) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < 11 * T; t += (int64_t)gridDim.x * blockDim.x)
        vals[t] = report_value(blk, C, t % T, (int)(t / T), is_rna);
}

// sums[k * R + i] = the mean of curve k over [x[i - 1], x[i]) (x[-1] = 0), the adds in the reference's order; the division is
// the only non-add and is off the chain.  An empty range (k_html_text prints "0.0" for it) is left 0.
__global__ void k_html_sums(const double* __restrict__ vals, int64_t T, const long long* __restrict__ x, int64_t R,
                            double* __restrict__ sums) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 11 * R) return;
    const int64_t k = t / R, i = t % R;
    const long long start = i ? x[i - 1] : 0, end = x[i];
    const double* v = vals + k * T;
    double total = 0.0;
#pragma unroll 8
    for (long long j = start; j < end; j++) total += v[j];
    sums[t] = end == start ? 0.0 : total / (double)(end - start);
}

__device__ __forceinline__ int html_seg(const HtmlText& H, int64_t i) {
    int s = 0;
    while (s + 1 < HTML_SEGS && H.start[s + 1] <= i) s++;
    return s;
}

__device__ __forceinline__ int html_value(const HtmlText& H, int s, int64_t i, char* buf) {
    const int w = H.blk[s];
    if (H.kind[s] == 2) {
        const long long* x = H.x[w];
        if (x[i] == (i ? x[i - 1] : 0)) { buf[0] = '0'; buf[1] = '.'; buf[2] = '0'; return 3; }     // list2string: end == start
        return fmt_g6(H.sums[w][H.base[s] + i], buf);
    }
    long long v = 0;                                  // the reference's unset tail of the density arrays: 0 here
    if (i < H.nonempty[w]) {
        const HtmlEntry e = H.grp[w][i];
        v = H.kind[s] == 0 ? (long long)(short)(e.med - 33) : (long long)e.len;
    }
    return html_itoa(v, buf);
}

__global__ void k_html_sizes(const HtmlText H, int64_t* __restrict__ size) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= H.start[HTML_SEGS]) return;
    const int s = html_seg(H, g);
    char buf[24];
    size[g] = html_value(H, s, g - H.start[s], buf) + (g + 1 < H.start[s + 1] ? 1 : 0);
}

__global__ void k_html_text(const HtmlText H, const int64_t* __restrict__ off, uint8_t* __restrict__ text) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= H.start[HTML_SEGS]) return;
    const int s = html_seg(H, g);
    char buf[24];
    const int n = html_value(H, s, g - H.start[s], buf);
    uint8_t* dst = text + off[g] + H.shift[s];
    for (int b = 0; b < n; b++) dst[b] = (uint8_t)buf[b];
    if (g + 1 < H.start[s + 1]) dst[n] = ',';
}

unsigned grid_for(int64_t n, int64_t cap) {
    const int64_t want = (n + 255) / 256;
    return (unsigned)(want < 1 ? 1 : want < cap ? want : cap);
}

}  // namespace

void launch_html_capture(const fpl_read_result* res, const int32_t* lens, int64_t n, const fpl_segment* segs, int64_t n_segs,
                         HtmlEntry* pre, HtmlEntry* post, cudaStream_t stream, int& launched) {
    const int64_t m = n > n_segs ? n : n_segs;
    if (m) k_html_capture<<<grid_for(m, FPL_NUM_SMS * 8), 256, 0, stream>>>(res, lens, n, segs, n_segs, pre, post);
    launched += m != 0;
}

void launch_html_hist(const HtmlEntry* e, int64_t n, int64_t nchunks, long long* mat, cudaStream_t stream, int& launched) {
    if (nchunks) k_html_hist<<<(unsigned)((nchunks + 3) / 4), 128, 0, stream>>>(e, n, nchunks, mat);
    launched += nchunks != 0;
}

void launch_html_scatter(const HtmlEntry* e, int64_t n, int64_t nchunks, const long long* off, HtmlEntry* out, cudaStream_t stream, int& launched) {
    if (nchunks) k_html_scatter<<<(unsigned)((nchunks + 3) / 4), 128, 0, stream>>>(e, n, nchunks, off, out);
    launched += nchunks != 0;
}

void launch_html_lenhist(const HtmlEntry* e, int64_t n, unsigned long long* hist, cudaStream_t stream, int& launched) {
    if (n) k_html_lenhist<<<grid_for(n, FPL_NUM_SMS * 8), 256, 0, stream>>>(e, n, hist);
    launched += n != 0;
}

void launch_html_lenprod(const unsigned long long* cnt, int64_t H, long long* prod, cudaStream_t stream, int& launched) {
    k_html_lenprod<<<(unsigned)((H + 255) / 256), 256, 0, stream>>>(cnt, H, prod);
    launched++;
}

void launch_html_lensearch(const unsigned long long* cnt, const long long* ccum, const long long* prod, const long long* pcum,
                           int64_t H, long long half_sum, unsigned long long half_n, int* out, cudaStream_t stream, int& launched) {
    k_html_lensearch<<<(unsigned)((H + 255) / 256), 256, 0, stream>>>(cnt, ccum, prod, pcum, H, half_sum, half_n, out);
    launched++;
}

void launch_html_bins(const unsigned long long* blk, int64_t C, int64_t T, unsigned long long* out, cudaStream_t stream, int& launched) {
    if (T) k_html_bins<<<grid_for(T, FPL_NUM_SMS * 8), 256, 0, stream>>>(blk, C, T, out);
    launched += T != 0;
}

void launch_html_values(const unsigned long long* blk, int64_t C, int64_t T, int is_rna, double* vals, cudaStream_t stream, int& launched) {
    if (T) k_html_values<<<grid_for(11 * T, FPL_NUM_SMS * 16), 256, 0, stream>>>(blk, C, T, is_rna, vals);
    launched += T != 0;
}

void launch_html_sums(const double* vals, int64_t T, const long long* x, int64_t R, double* sums, cudaStream_t stream, int& launched) {
    if (R) k_html_sums<<<(unsigned)((11 * R + 127) / 128), 128, 0, stream>>>(vals, T, x, R, sums);
    launched += R != 0;
}

void launch_html_sizes(const HtmlText& H, int64_t* size, cudaStream_t stream, int& launched) {
    const int64_t n = H.start[HTML_SEGS];
    if (n) k_html_sizes<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(H, size);
    launched += n != 0;
}

void launch_html_text(const HtmlText& H, const int64_t* off, const uint8_t* frame, const int64_t* src, const int64_t* dst, int n_pieces,
                      uint8_t* text, cudaStream_t stream, int& launched) {
    k_report_frame<<<n_pieces, 256, 0, stream>>>(frame, src, dst, text);
    const int64_t n = H.start[HTML_SEGS];
    if (n) k_html_text<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(H, off, text);
    launched += n ? 2 : 1;
}

// ------------------------------------------------------------------------------------------------------------------
// fpl_merge_stats (Stats::merge, src/stats.cpp:1013-1082; FilterResult::merge, src/filterresult.cpp:28-61): one thread owns
// each destination word — rows [0, rows) of the 16 per-cycle arrays and the tail of both Stats blocks, then the counter
// block — and adds the sources to it in list order.  No atomics; the sums do not depend on the grid.
// ------------------------------------------------------------------------------------------------------------------
namespace {

__global__ void k_merge_stats(unsigned long long* __restrict__ pre, unsigned long long* __restrict__ post,
                              unsigned long long* __restrict__ cnt, int64_t C, int64_t rows, int64_t cnt_words,
                              const MergeSrc* __restrict__ src, int n_src) {
    const int64_t per = 16 * rows + FPL_STATS_TAIL, total = 2 * per + cnt_words;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        if (i >= 2 * per) {                      // counter block
            const int64_t k = i - 2 * per;
            unsigned long long v = cnt[k];
            for (int s = 0; s < n_src; s++) v += src[s].cnt[k];
            cnt[k] = v;
            continue;
        }
        const int w = i >= per;
        const int64_t j = i - (w ? per : 0);
        unsigned long long* d = w ? post : pre;
        if (j >= 16 * rows) {                    // tail
            const int64_t t = j - 16 * rows;
            unsigned long long v = d[16 * C + t];
            for (int s = 0; s < n_src; s++) v += src[s].blk[w][16 * src[s].C + t];
            d[16 * C + t] = v;
        } else {                                 // row b, cycle c: only sources whose rows reach c hold counts there
            const int64_t b = j / rows, c = j - b * rows;
            unsigned long long v = d[b * C + c];
            for (int s = 0; s < n_src; s++)
                if (c < src[s].rows) v += src[s].blk[w][b * src[s].C + c];
            d[b * C + c] = v;
        }
    }
}

}  // namespace

void launch_merge_stats(unsigned long long* pre, unsigned long long* post, unsigned long long* cnt, int64_t C, int64_t rows,
                        int64_t cnt_words, const MergeSrc* src, int n_src, cudaStream_t stream, int& launched) {
    const int64_t total = 2 * (16 * rows + FPL_STATS_TAIL) + cnt_words;
    k_merge_stats<<<grid_for(total, FPL_NUM_SMS * 8), 256, 0, stream>>>(pre, post, cnt, C, rows, cnt_words, src, n_src);
    launched++;
}
