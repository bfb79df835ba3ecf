// k_scan: the per-base pass over each trimmed read window — the "adapter + quality" kernel:
//   * AdapterTrimmer::findMiddleAdapters' two whole-read searchAdapter scans in generic mode
//     (src/adaptertrimmer.cpp:13-40, 135-154): first arg-min over p in [0, len-alen) of the Hamming distance
//     between read[p..p+alen) and the adapter, for -s and for -e;
//   * Filter::passFilter's counts (src/filter.cpp:23-38): #(qual < qualifiedQual), #(base == 'N'), sum(qual-33);
//   * Filter::passLowComplexityFilter's count (src/filter.cpp:67-81): #(seq[i] != seq[i+1]).
// One CTA per read walks the window in tiles staged in shared memory; sequence bytes are compared four
// positions at a time (SWAR on 32-bit words).  k_final then verifies the arg-mins with one edit distance each,
// derives the segments (Read::breakByGap, src/read.cpp:192-215) and evaluates the filter thresholds.
#include "fpl_device.cuh"

#define SCAN_THREADS 256
#define SCAN_TILE 4096                      // positions per tile (multiple of 4*SCAN_THREADS... see loop)
#define SCAN_HALO (FPL_MAX_ADAPTER_LEN + 8)

namespace {

__device__ __forceinline__ uint32_t nz_bytes(uint32_t d) {
    // 0x01 in every byte lane of d that is non-zero
    uint32_t t = ((d & 0x7f7f7f7fu) + 0x7f7f7f7fu) | d;
    return (t >> 7) & 0x01010101u;
}

__device__ __forceinline__ unsigned long long block_min_u64(unsigned long long v, unsigned long long* sh) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        unsigned long long o = __shfl_xor_sync(0xffffffffu, v, d);
        v = o < v ? o : v;
    }
    const int wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane_id() == 0) sh[wid] = v;
    __syncthreads();
    v = sh[0];
    for (int i = 1; i < SCAN_THREADS / 32; i++) v = sh[i] < v ? sh[i] : v;
    return v;
}

__device__ __forceinline__ int block_sum(int v, int* sh) {
    v = __reduce_add_sync(0xffffffffu, v);
    const int wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane_id() == 0) sh[wid] = v;
    __syncthreads();
    int s = 0;
    for (int i = 0; i < SCAN_THREADS / 32; i++) s += sh[i];
    return s;
}

}  // namespace

__global__ void __launch_bounds__(SCAN_THREADS)
k_scan(const __grid_constant__ DevParams P, DevBatch b, ReadState* __restrict__ st) {
    // tile bytes live at sseq[0 .. SCAN_TILE + SCAN_HALO), 4-byte aligned so that index 0 == window position tile0
    __shared__ __align__(16) uint8_t sseq[SCAN_TILE + SCAN_HALO + 8];
    __shared__ unsigned long long sh64[SCAN_THREADS / 32];
    __shared__ int sh32[SCAN_THREADS / 32];
    const int64_t r = blockIdx.x;
    ReadState s = st[r];
    if (!s.alive) return;
    const int len = s.len;
    const uint8_t* seq = b.seq + b.offsets[r] + s.lo;
    const uint8_t* qual = b.qual + b.offsets[r] + s.lo;
    const bool doAdapters = P.opt.adapter_enabled != 0;
    const bool doCounts = (P.opt.qual_filter_enabled || P.opt.length_filter_enabled);
    const bool doCplx = P.opt.complexity_enabled != 0;
    const int qq = (int)(signed char)P.opt.qualified_qual;
    const int alen0 = P.alen[0], alen1 = P.alen[1];
    const int maxa = max(alen0, alen1);
    // number of scan positions per adapter: p in [0, len - alen)  (and none at all if alen > len)
    const int np0 = (doAdapters && alen0 <= len) ? len - alen0 : 0;
    const int np1 = (doAdapters && alen1 <= len) ? len - alen1 : 0;
    unsigned long long best0 = ~0ull, best1 = ~0ull;
    int lowq = 0, nn = 0, totalq = 0, diff = 0;
    const uint8_t* a0 = P.adapters;
    const uint8_t* a1 = P.adapters + FPL_MAX_ADAPTER_LEN;

    for (int t0 = 0; t0 < len; t0 += SCAN_TILE) {
        const int tn = min(SCAN_TILE, len - t0);                 // positions in this tile
        const int need = min(tn + maxa + 4, len - t0);           // bytes to stage (tile + halo)
        __syncthreads();
        for (int i = threadIdx.x; i < need; i += SCAN_THREADS) sseq[i] = seq[t0 + i];
        // zero pad so that word loads past the staged bytes are defined (they never contribute to a result)
        for (int i = need + threadIdx.x; i < need + 8; i += SCAN_THREADS) sseq[i] = 0;
        __syncthreads();
        // ---- passFilter / complexity counts: one byte per thread per step ----
        if (doCounts || doCplx) {
            for (int i = threadIdx.x; i < tn; i += SCAN_THREADS) {
                const uint8_t base = sseq[i];
                if (doCounts) {
                    const int q = (int)(signed char)qual[t0 + i];
                    totalq += q - 33;
                    lowq += q < qq;
                    nn += base == 'N';
                }
                if (doCplx && t0 + i < len - 1) diff += base != sseq[i + 1];
            }
        }
        // ---- Hamming scans: each thread owns 4 consecutive positions (one SWAR word) per step ----
        if (doAdapters) {
            const uint32_t* w32 = reinterpret_cast<const uint32_t*>(sseq);
            for (int g = threadIdx.x; g * 4 < tn; g += SCAN_THREADS) {
                const int pbase = t0 + g * 4;
#pragma unroll
                for (int which = 0; which < 2; which++) {
                    const int alen = which ? alen1 : alen0;
                    const int np = which ? np1 : np0;
                    if (pbase >= np) continue;
                    const uint8_t* ad = which ? a1 : a0;
                    uint32_t acc = 0;  // four byte-wide mismatch counters, emptied into cnt[] before they can overflow
                    uint32_t cnt[4] = {0, 0, 0, 0};
                    uint32_t wlo = w32[g], whi = w32[g + 1];
                    int wi = g + 1;
                    for (int i = 0; i < alen; i++) {
                        const int sh = i & 3;
                        uint32_t x = sh == 0 ? wlo : __funnelshift_r(wlo, whi, sh * 8);
                        uint32_t a4 = (uint32_t)__ldg(&ad[i]) * 0x01010101u;
                        acc += nz_bytes(x ^ a4);
                        if (sh == 3) { wlo = whi; whi = w32[++wi]; }
                        if ((i & 127) == 127) {
#pragma unroll
                            for (int k = 0; k < 4; k++) cnt[k] += (acc >> (8 * k)) & 0xFFu;
                            acc = 0;
                        }
                    }
#pragma unroll
                    for (int k = 0; k < 4; k++) cnt[k] += (acc >> (8 * k)) & 0xFFu;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const int p = pbase + k;
                        if (p < np) {
                            unsigned long long key = ((unsigned long long)cnt[k] << 32) | (unsigned)p;
                            if (which) best1 = key < best1 ? key : best1;
                            else best0 = key < best0 ? key : best0;
                        }
                    }
                }
            }
        }
    }
    best0 = block_min_u64(best0, sh64);
    best1 = block_min_u64(best1, sh64);
    lowq = block_sum(lowq, sh32);
    nn = block_sum(nn, sh32);
    totalq = block_sum(totalq, sh32);
    diff = block_sum(diff, sh32);
    if (threadIdx.x == 0) {
        ReadState* o = &st[r];
        o->best[0] = best0; o->best[1] = best1;
        o->lowq = lowq; o->nn = nn; o->totalq = totalq; o->diff = diff;
    }
}

void launch_scan(const DevParams& P, const DevBatch& b, ReadState* st, cudaStream_t stream) {
    if (b.n_reads == 0) return;
    k_scan<<<(unsigned)b.n_reads, SCAN_THREADS, 0, stream>>>(P, b, st);
}

// ------------------------------------------------------------------------------------------------------------------
// k_final: one warp per read.  ED-verifies the two arg-mins (searchAdapter :156-165), merges them into the gap
// (findMiddleAdapters :19-37), derives the segments (breakByGap), recounts the filter sums for split reads and
// evaluates Filter::passFilter's thresholds (src/filter.cpp:40-63) in their integer forms (SURVEY A.9).
// ------------------------------------------------------------------------------------------------------------------
namespace {

__device__ int myers128_f(const uint8_t* text, int n, const uint4* peq, int m) {
    // same recurrence as in fpl_trim.cu (pattern = whole adapter, m = alen <= 128)
    if (m == 0) return n;
    if (n == 0) return m;
    unsigned long long VPl, VPh, VNl = 0, VNh = 0;
    if (m < 64) { VPl = (1ull << m) - 1; VPh = 0; }
    else if (m == 64) { VPl = ~0ull; VPh = 0; }
    else if (m < 128) { VPl = ~0ull; VPh = (1ull << (m - 64)) - 1; }
    else { VPl = ~0ull; VPh = ~0ull; }
    const bool topHi = m > 64;
    const unsigned long long top = 1ull << ((m - 1) & 63);
    int score = m;
    for (int i = 0; i < n; i++) {
        uint4 v = __ldg(&peq[text[i]]);
        unsigned long long El = ((unsigned long long)v.y << 32) | v.x, Eh = ((unsigned long long)v.w << 32) | v.z;
        unsigned long long Xvl = El | VNl, Xvh = Eh | VNh;
        unsigned long long al = El & VPl, ah = Eh & VPh;
        unsigned long long sl = al + VPl;
        unsigned long long carry = sl < al ? 1ull : 0ull;
        unsigned long long sh = ah + VPh + carry;
        unsigned long long Xhl = (sl ^ VPl) | El, Xhh = (sh ^ VPh) | Eh;
        unsigned long long HPl = VNl | ~(Xhl | VPl), HPh = VNh | ~(Xhh | VPh);
        unsigned long long HNl = VPl & Xhl, HNh = VPh & Xhh;
        unsigned long long hpTop = topHi ? HPh : HPl, hnTop = topHi ? HNh : HNl;
        if (hpTop & top) score++;
        else if (hnTop & top) score--;
        HPh = (HPh << 1) | (HPl >> 63); HPl = (HPl << 1) | 1ull;
        HNh = (HNh << 1) | (HNl >> 63); HNl = HNl << 1;
        VPl = HNl | ~(Xvl | HPl); VPh = HNh | ~(Xvh | HPh);
        VNl = HPl & Xvl; VNh = HPh & Xvh;
    }
    return score;
}

struct Counts { int lowq, nn, totalq, diff; };

// Filter::passFilter on integer counts.  lowQ > limit*len/100.0  <=>  lowQ*100 > limit*len, etc. (SURVEY A.9)
__device__ int pass_filter(const fpl_options& o, int rlen, const Counts& c) {
    if (rlen == 0) return FPL_FAIL_LENGTH;
    if (o.qual_filter_enabled) {
        if ((long long)c.lowq * 100 > (long long)o.unqualified_percent_limit * rlen) return FPL_FAIL_QUALITY;
        else if (o.avg_qual_req > 0 && (c.totalq / rlen) < o.avg_qual_req) return FPL_FAIL_QUALITY;
        else if ((long long)c.nn * 100 > (long long)rlen * o.n_base_percent_limit) return FPL_FAIL_N_BASE;
        else if (o.n_base_limit != 1000000 && c.nn > o.n_base_limit) return FPL_FAIL_N_BASE;
    }
    if (o.length_filter_enabled) {
        if (rlen < o.length_required) return FPL_FAIL_LENGTH;
        if (o.length_max > 0 && rlen > o.length_max) return FPL_FAIL_TOO_LONG;
    }
    if (o.complexity_enabled) {
        if (rlen <= 1) return FPL_FAIL_COMPLEXITY;
        // (double)diff/(double)(len-1) >= pct/100.0  <=>  diff*100 >= pct*(len-1)
        if (!((long long)c.diff * 100 >= (long long)o.complexity_threshold_pct * (rlen - 1))) return FPL_FAIL_COMPLEXITY;
    }
    return FPL_PASS_FILTER;
}

// Filter::passFilter's counts for a byte range of a split read (warp-wide): #(q < qualified), #N, sum(q - 33) over
// [0, len) and #(seq[i] != seq[i+1]) over i in [0, len - 1).  16-byte vector loads: the range starts anywhere, so the
// vectors are aligned down (sequence and quality buffers are equally aligned, one misalignment serves both).  A vector
// whose 16 bytes and 16 adjacent pairs all lie inside the range takes the word-wise path — the quality counts as in
// k_scan_jit (x = q + (128 - qualified) by IMAD; the unsigned and the signed dp4a sums of x differ by 256 per q >=
// qualified), N and the unequal neighbours by zero-byte tests — the two ragged ends go byte by byte.
__device__ __forceinline__ uint32_t zero_bytes80(uint32_t d) {     // 0x80 in every byte of d that is zero
    return ~(((d & 0x7f7f7f7fu) + 0x7f7f7f7fu) | d) & 0x80808080u;
}

__device__ Counts count_range(const fpl_options& o, uint32_t one, const uint8_t* seq, const uint8_t* qual, int len) {
    Counts c = {0, 0, 0, 0};
    const int lane = lane_id();
    const bool doCounts = (o.qual_filter_enabled || o.length_filter_enabled);
    const bool doCplx = o.complexity_enabled != 0;
    if (!doCounts && !doCplx) return c;                    // no filter reads these counts: touch nothing
    const int qq = (int)(signed char)o.qualified_qual;
    const uint32_t KQ = (uint32_t)(128 - (o.qualified_qual & 0x7f));
    const int pre = (int)(reinterpret_cast<uintptr_t>(seq) & 15);
    const uint4* sv = reinterpret_cast<const uint4*>(seq - pre);
    const uint4* qv = reinterpret_cast<const uint4*>(qual - pre);
    const int total = pre + len;
    uint32_t accU = 0; int accS = 0, nfast = 0;
    for (int v = lane; v * 16 < total; v += 32) {
        const uint4 s4 = __ldg(sv + v), q4 = __ldg(qv + v);
        const uint32_t sw[4] = {s4.x, s4.y, s4.z, s4.w}, qw[4] = {q4.x, q4.y, q4.z, q4.w};
        const int first = v * 16 - pre, after = first + 16;
        // the byte after this vector, for the last adjacent pair
        const uint32_t nextb = (doCplx && after < len) ? (uint32_t)seq[after] : 0u;
        if (first >= 0 && after <= len - 1) {
            if (doCounts) {
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    uint32_t x;
                    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(x) : "r"(qw[k]), "r"(one), "r"(KQ * 0x01010101u));
                    accU = __dp4a(x, 0x01010101u, accU);
                    accS = __dp4a((int)x, 0x01010101, accS);
                    c.nn += __popc(zero_bytes80(sw[k] ^ 0x4E4E4E4Eu));
                }
                nfast += 16;
            }
            if (doCplx) {
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const uint32_t w2 = k < 3 ? sw[k + 1] : nextb;
                    c.diff += 4 - __popc(zero_bytes80(sw[k] ^ __funnelshift_r(sw[k], w2, 8)));
                }
            }
            continue;
        }
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int pos = first + j;
            if (pos < 0 || pos >= len) continue;
            const uint32_t sb = (sw[j >> 2] >> (8 * (j & 3))) & 0xFFu;
            if (doCounts) {
                const int q = (int)(signed char)((qw[j >> 2] >> (8 * (j & 3))) & 0xFFu);
                c.totalq += q - 33; c.lowq += q < qq; c.nn += sb == 'N';
            }
            if (doCplx && pos < len - 1) {
                const uint32_t nb = j < 15 ? (sw[(j + 1) >> 2] >> (8 * ((j + 1) & 3))) & 0xFFu : nextb;
                c.diff += sb != nb;
            }
        }
    }
    // fast vectors: #(q >= qualified) = (accU - accS) / 256, sum(q) = accU - KQ * n
    c.lowq += nfast - (int)((accU - (uint32_t)accS) >> 8);
    c.totalq += (int)accU - (int)(KQ + 33u) * nfast;
    c.lowq = __reduce_add_sync(0xffffffffu, c.lowq); c.nn = __reduce_add_sync(0xffffffffu, c.nn);
    c.totalq = __reduce_add_sync(0xffffffffu, c.totalq); c.diff = __reduce_add_sync(0xffffffffu, c.diff);
    return c;
}

}  // namespace

#define FINAL_WARPS 4

// CLS: size class of -s / -e (DevParams::small_adapters): 0 = both <= 32 bp — the kernel is then compiled without the
// 128-bit and multi-word Myers forms and their local arrays, which would otherwise set its register budget and occupancy
// (it is bound by the latency of its dependent loads).  QH: k_scan_jit counted the quality histograms, k_final hands the
// window's median on and lists the other reads in exc (a separate instance: the other paths run the kernel as it was)
template <int CLS, bool QH>
__global__ void __launch_bounds__(FINAL_WARPS * 32)
k_final(const __grid_constant__ DevParams P, DevBatch b, const ReadState* __restrict__ st,
        fpl_read_result* __restrict__ res, StatSeg* __restrict__ postseg, int32_t* __restrict__ exc, int* __restrict__ n_exc) {
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const int64_t r = (int64_t)blockIdx.x * FINAL_WARPS + wid;
    if (r >= b.n_reads) return;
    // the kernel is a chain of dependent loads per warp: the read's offset is loaded beside its ReadState (not after the
    // alive test), so that the bytes at the arg-mins are one load away from both
    const int64_t off = b.offsets[r];
    const ReadState s = st[r];
    fpl_read_result* out = &res[r];
    StatSeg ps0 = {0, 0, -1, 0, 0}, ps1 = ps0;
    bool one_window = false;                             // the read's one passing segment is its window
    if (s.alive) {
        const uint8_t* seq = b.seq + off + s.lo;
        const uint8_t* qual = b.qual + off + s.lo;
        const int L = s.len;
        int nseg = 0, segLo[2] = {0, 0}, segLen[2] = {0, 0};
        bool split = false, seg0right = false;
        int gapLo = 0, gapLen = 0;                       // the gap Read::breakByGap cuts out: [gapLo, gapLo + gapLen)
        if (P.opt.adapter_enabled) {
            const int ext = P.opt.trimming_extension;
            int pos[2] = {-1, -1};
            if (CLS == 0 && P.alen[0] > 0 && P.alen[1] > 0) {
                // both verifications side by side: half-warp k checks the arg-min of adapter k
                const int k = lane >> 4;
                const bool on = s.best[k] != ~0ull;
                const int alen = P.alen[k];
                const int p = (int)(s.best[k] & 0xFFFFFFFFu);
                const int ed = myers32_halves(seq + (on ? p : 0), alen, P.peq + (size_t)k * 256, alen, on);
                const bool hit = on && ed <= P.thr[alen];
                const unsigned hm = __ballot_sync(0xffffffffu, hit);
                if (hm & 1u) pos[0] = (int)(s.best[0] & 0xFFFFFFFFu);
                if (hm & 0x10000u) pos[1] = (int)(s.best[1] & 0xFFFFFFFFu);
            } else {
#pragma unroll
                for (int k = 0; k < 2; k++) {
                    if (s.best[k] != ~0ull) {
                        const int alen = P.alen[k];
                        const int p = (int)(s.best[k] & 0xFFFFFFFFu);
                        int ed;
                        if (CLS == 0 || alen <= 32) ed = myers32_warp(seq + p, alen, P.peq + (size_t)k * 256, 0, alen);
                        else if (alen <= 128) ed = myers128_f(seq + p, alen, P.peq + (size_t)k * 256, alen);
                        else ed = myers_long(seq + p, alen, P.peq_long + (size_t)k * 256 * P.peq_words, P.peq_words, 0, alen);
                        if (ed <= P.thr[alen]) pos[k] = p;
                    }
                }
            }
            int start = -1, glen = 0;
            const int sp = pos[0], ep = pos[1], slen = P.alen[0], elen = P.alen[1];
            if (sp >= 0 && ep >= 0) {
                int stt = min(sp, ep), en = max(sp + slen, ep + elen);
                stt = max(0, stt - ext); en = min(L, en + ext);
                start = stt; glen = en - stt; split = true;
            } else if (sp >= 0) {
                int en = min(L, sp + slen + ext);
                start = max(0, sp - ext); glen = en - start; split = true;
            } else if (ep >= 0) {
                int en = min(L, ep + elen + ext);
                start = max(0, ep - ext); glen = en - start; split = true;
            }
            if (split) {
                gapLo = start; gapLen = glen;
                const int len1 = start, len2 = L - start - glen;
                if (len1 > 0) { segLo[nseg] = 0; segLen[nseg] = len1; nseg++; }
                if (len2 > 0) { segLo[nseg] = start + glen; segLen[nseg] = len2; nseg++; }
                seg0right = (nseg == 1 && len1 <= 0);
            } else { segLo[0] = 0; segLen[0] = L; nseg = 1; }
        } else { segLo[0] = 0; segLen[0] = L; nseg = 1; }

        int code[2] = {0, 0};
        if (split && nseg > 0) {
            // Read::breakByGap left [0, start) and [start + glen, L); the filter counts of the two sides come from the
            // scan's counts of the whole window minus what is counted here.
            const int lenA = max(gapLo, 0);                                       // left side [0, lenA)
            const int loB = gapLo + gapLen;                                        // right side [loB, L)
            const int lenB = max(L - loB, 0);
            const Counts tot = {s.lowq, s.nn, s.totalq, s.diff};
            // the window is [A | gap | B] and the scan counted all of it: count the two SMALLEST parts here and take the
            // largest by subtraction (two far-apart adapter hits of an ultra-long read make the gap the big part)
            // adjacent pairs that straddle a boundary belong to no part
            const int x1 = (lenA > 0 && gapLen > 0) ? (seq[gapLo - 1] != seq[gapLo]) : 0;
            const int x2 = (lenB > 0 && gapLen > 0) ? (seq[loB - 1] != seq[loB]) : 0;
            const int biggest = (lenA >= lenB && lenA >= gapLen) ? 0 : (lenB >= gapLen ? 2 : 1);      // 0 A, 1 gap, 2 B
            const int partLo[3] = {0, gapLo, loB}, partLen[3] = {lenA, gapLen, lenB};
            Counts part[3] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
            Counts rest = tot;
            rest.diff = P.opt.complexity_enabled ? tot.diff - x1 - x2 : 0;
#pragma unroll 1
            for (int k = 0; k < 3; k++) {
                if (k == biggest) continue;
                const Counts c = count_range(P.opt, P.one, seq + partLo[k], qual + partLo[k], partLen[k]);
                part[k] = c;
                rest.lowq -= c.lowq; rest.nn -= c.nn; rest.totalq -= c.totalq;
                if (P.opt.complexity_enabled) rest.diff -= c.diff;
            }
            Counts cA = part[0], cB = part[2];
            if (biggest == 0) cA = rest; else if (biggest == 2) cB = rest;
            if (nseg == 2) { code[0] = pass_filter(P.opt, segLen[0], cA); code[1] = pass_filter(P.opt, segLen[1], cB); }
            else code[0] = pass_filter(P.opt, segLen[0], seg0right ? cB : cA);
        } else {
            for (int k = 0; k < nseg; k++) {
                Counts c;
                c.lowq = s.lowq; c.nn = s.nn; c.totalq = s.totalq; c.diff = s.diff;
                code[k] = pass_filter(P.opt, segLen[k], c);
            }
        }
        if (lane == 0) {
            // k_trim wrote the record's other flags: these are or-ed in without reading it back (a reduction, nothing
            // for the warp to wait for), and only by the split reads
            const uint32_t flags = (split ? FPL_FLAG_MIDDLE_ADAPTER : 0u) | (seg0right ? FPL_FLAG_SEG0_IS_RIGHT : 0u);
            if (flags) atomicOr(&out->flags, flags);
            out->n_segments = nseg;
            for (int k = 0; k < nseg; k++) {
                out->seg_lo[k] = s.lo + segLo[k];
                out->seg_len[k] = segLen[k];
                out->seg_result[k] = (uint8_t)code[k];
            }
        }
        // k_scan_jit counted the quality histograms (QH): the window's median is the median of a read whose
        // one passing segment is the window
        one_window = !split && nseg == 1 && code[0] == FPL_PASS_FILTER;
        if (QH && lane == 0) out->pre_median_qual = (uint8_t)s.pad;          // the scan's median of the whole read
        if (QH && lane == 0 && one_window) out->seg_median_qual[0] = (uint8_t)s.reserved[0];
        if (nseg > 0 && code[0] == FPL_PASS_FILTER) { ps0.off = off + s.lo + segLo[0]; ps0.len = segLen[0]; ps0.read = (int)r; ps0.slot = 0; }
        if (nseg > 1 && code[1] == FPL_PASS_FILTER) { ps1.off = off + s.lo + segLo[1]; ps1.len = segLen[1]; ps1.read = (int)r; ps1.slot = 1; }
        // a passing zero-length segment cannot exist (passFilter fails rlen == 0), so len == 0 <=> "no segment"
    }
    if (lane == 0) { postseg[2 * r] = ps0; postseg[2 * r + 1] = ps1; }
    // every other read (not alive, split, or a failing segment) goes to k_read_qual_exc's list: one atomic per read
    if (QH && lane == 0 && !one_window) exc[atomicAdd(n_exc, 1)] = (int32_t)r;
}

// exc / n_exc (nullptr: k_scan_jit did not count the quality histograms): the list of the reads k_read_qual_exc treats
void launch_final(const DevParams& P, const DevBatch& b, const ReadState* st, fpl_read_result* res, StatSeg* postseg,
                  int32_t* exc, int* n_exc, cudaStream_t stream) {
    if (b.n_reads == 0) return;
    unsigned grid = (unsigned)((b.n_reads + FINAL_WARPS - 1) / FINAL_WARPS);
    if (exc) {
        if (P.small_adapters == 0) k_final<0, true><<<grid, FINAL_WARPS * 32, 0, stream>>>(P, b, st, res, postseg, exc, n_exc);
        else k_final<2, true><<<grid, FINAL_WARPS * 32, 0, stream>>>(P, b, st, res, postseg, exc, n_exc);
    } else {
        if (P.small_adapters == 0) k_final<0, false><<<grid, FINAL_WARPS * 32, 0, stream>>>(P, b, st, res, postseg, exc, n_exc);
        else k_final<2, false><<<grid, FINAL_WARPS * 32, 0, stream>>>(P, b, st, res, postseg, exc, n_exc);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// k_count: FilterResult counters (src/filterresult.cpp:22-81) from the finished records; block-level
// aggregation in shared memory, one global atomic per non-zero counter per block.
// stats_pre != nullptr (k_scan_jit counted the quality histograms): also the per-read sums of both Stats blocks
// (mReads, mLengthSum, mMedianReadQualHistogram, mMedianReadQualBases, src/stats.cpp:362-374) — every read for the
// pre-filter block, every passing segment for the post-filter one — which k_read_qual adds on the other paths.
// ------------------------------------------------------------------------------------------------------------------
#define CNT_SUMS (2 + 2 * 128)       // per Stats block: reads, length sum, median histogram, median bases

__global__ void __launch_bounds__(256)
k_count(const fpl_read_result* __restrict__ res, int64_t n, unsigned long long* __restrict__ counters, bool count_segments,
        const int32_t* __restrict__ lens, unsigned long long* __restrict__ stats_pre, unsigned long long* __restrict__ stats_post,
        int64_t C) {
    __shared__ unsigned long long sh[FPL_CNT_FIXED];
    __shared__ unsigned long long sums[2][CNT_SUMS];
    for (int i = threadIdx.x; i < FPL_CNT_FIXED; i += blockDim.x) sh[i] = 0;
    if (stats_pre)
        for (int i = threadIdx.x; i < 2 * CNT_SUMS; i += blockDim.x) (&sums[0][0])[i] = 0;
    __syncthreads();
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) {
        const fpl_read_result* o = &res[r];
        const uint32_t flags = o->flags;
        const int nseg = o->n_segments;
        if (count_segments)
            for (int k = 0; k < nseg; k++) atomicAdd(&sh[FPL_CNT_FILTER + o->seg_result[k]], 1ull);
        const int tb = o->adapter_trimmed_bases;
        if (tb > 0) {
            atomicAdd(&sh[FPL_CNT_ADAPTER_READS], 1ull);
            atomicAdd(&sh[FPL_CNT_ADAPTER_BASES], (unsigned long long)tb);
        }
        if (flags & FPL_FLAG_DROPPED_BY_CUT) atomicAdd(&sh[FPL_CNT_DROPPED], 1ull);
        if (flags & FPL_FLAG_MIDDLE_ADAPTER) atomicAdd(&sh[FPL_CNT_SPLIT], 1ull);
        if (stats_pre) {
            // the same order of effects as Stats::statRead: a read counts, its median only when it has bases
            const int L = lens[r];
            atomicAdd(&sums[0][0], 1ull);
            atomicAdd(&sums[0][1], (unsigned long long)L);
            if (L > 0) {
                atomicAdd(&sums[0][2 + o->pre_median_qual], 1ull);
                atomicAdd(&sums[0][2 + 128 + o->pre_median_qual], (unsigned long long)L);
            }
            for (int k = 0; k < nseg; k++) {
                if (o->seg_result[k] != FPL_PASS_FILTER) continue;
                const int sl = o->seg_len[k];
                atomicAdd(&sums[1][0], 1ull);
                atomicAdd(&sums[1][1], (unsigned long long)sl);
                if (sl > 0) {
                    atomicAdd(&sums[1][2 + o->seg_median_qual[k]], 1ull);
                    atomicAdd(&sums[1][2 + 128 + o->seg_median_qual[k]], (unsigned long long)sl);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < FPL_CNT_FIXED; i += blockDim.x)
        if (sh[i]) atomicAdd(&counters[i], sh[i]);
    if (stats_pre)
        for (int i = threadIdx.x; i < 2 * CNT_SUMS; i += blockDim.x) {
            const int w = i / CNT_SUMS, j = i % CNT_SUMS;
            const unsigned long long v = sums[w][j];
            if (!v) continue;
            unsigned long long* tail = (w ? stats_post : stats_pre) + 16 * C;
            const int at = j == 0 ? FPL_STATS_READS : j == 1 ? FPL_STATS_LENSUM : j < 2 + 128 ? FPL_STATS_MEDHIST + (j - 2)
                                                                                                : FPL_STATS_MEDBASES + (j - 2 - 128);
            atomicAdd(&tail[at], v);
        }
}

// count_segments = false: --mask/--break, where the output reads are counted by k_ext_filter instead.  stats_pre /
// stats_post / C (stats_pre == nullptr: not here): see k_count.
void launch_count(const fpl_read_result* res, int64_t n, unsigned long long* counters, bool count_segments, const int32_t* lens,
                  unsigned long long* stats_pre, unsigned long long* stats_post, int64_t C, cudaStream_t stream) {
    if (n == 0) return;
    k_count<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(res, n, counters, count_segments, lens, stats_pre, stats_post, C);
}
