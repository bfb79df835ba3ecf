// --mask / --break (SURVEY §8f row 3): the part of processSingleEnd between the adapter stage and passFilter
// (src/seprocessor.cpp:235-262) on the device, for a variable number of output reads per input read.
//   Filter::detectLowQualityRegions (src/filter.cpp:83-128)  detect_regions(): transcribed literally, including the
//                                                             absolute pre-sum bound that makes the running sum
//                                                             restart from 0 after the first region (SURVEY A.8)
//   Read::breakByRegions (src/read.cpp:227-262)               walk_break(): pieces between the regions, "r<k>-" indices
//   Read::maskRegionWithN (src/read.cpp:217-225)              k_ext_mask_emit: 'N' into a private copy of the sequence
//   Filter::passFilter on every output read                   k_ext_filter (counts on the masked copy)
// The region walk is sequential by construction (each region's start depends on the previous one's end), so one
// thread walks one read; these flags are not on the benchmarked configuration, the kernels are written for exactness.
#include <cub/device/device_scan.cuh>
#include "fpl_device.cuh"
#include "fpl_ext.h"

namespace {

__device__ __forceinline__ int sq(const uint8_t* q, int i) { return (int)(signed char)q[i]; }

template <class Emit>
__device__ int detect_regions(const uint8_t* qualstr, int l, int windowSize, int quality, Emit emit) {
    int n = 0;
    if (l == 0 || windowSize <= 0) return 0;
    int start = 0;
    const int need = (33 + quality) * windowSize;
    while (start + windowSize <= l) {
        int totalQual = 0;
        for (int i = start; i < windowSize - 1 && i < l; i++) totalQual += sq(qualstr, i);
        int windowStart = -1;
        for (int s = start; s + windowSize < l; s++) {
            if (totalQual < need) { windowStart = s; break; }
            totalQual += sq(qualstr, s + windowSize);
            totalQual -= sq(qualstr, s);
        }
        if (windowStart == -1) break;
        int e;
        for (e = windowStart; e + windowSize < l; e++) {
            totalQual += sq(qualstr, e + windowSize);
            totalQual -= sq(qualstr, e);
            if (totalQual >= need) break;
        }
        emit(windowStart, e + windowSize - 1);
        n++;
        start = e + windowSize;
    }
    return n;
}

// pieces of a read of `len` bases; piece(lo_rel, len, break_index).  Returns -1 if no region was found (the read stays
// as it is), else the number of pieces (possibly 0: the read vanishes).
template <class Piece>
__device__ int walk_break(const uint8_t* qual, int len, int w, int Q, Piece piece) {
    int lastEnd = -1, npieces = 0, nreg = 0;
    detect_regions(qual, len, w, Q, [&](int first, int last) {
        const int i = nreg++;
        const int start = first < 0 ? 0 : first, end = last >= len ? len - 1 : last;
        if (start > end || start >= len) return;
        if (start > lastEnd + 1) { piece(lastEnd + 1, start - lastEnd - 1, i + 1); npieces++; }
        lastEnd = end;
    });
    if (nreg == 0) return -1;
    if (lastEnd < len - 1) { piece(lastEnd + 1, len - lastEnd - 1, nreg + 1); npieces++; }
    return npieces;
}

// initial segment k of read r (after the adapter stage), from the record k_final wrote
__device__ __forceinline__ bool initial_segment(const fpl_read_result* o, int k, int& lo, int& len, int& side) {
    if (k >= o->n_segments) return false;
    lo = o->seg_lo[k]; len = o->seg_len[k];
    const bool split = (o->flags & FPL_FLAG_MIDDLE_ADAPTER) != 0;
    side = split ? ((k == 1 || (o->flags & FPL_FLAG_SEG0_IS_RIGHT)) ? 2 : 1) : 0;
    return true;
}

}  // namespace

// pass 1: pieces per initial segment (index 2r + k); the records still hold k_final's initial segments
__global__ void k_ext_count(const __grid_constant__ DevParams P, DevBatch b, const fpl_read_result* __restrict__ res,
                            int32_t* __restrict__ cnt) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * b.n_reads) return;
    const int64_t r = t >> 1;
    const int k = (int)(t & 1);
    int lo, len, side, n = 0;
    if (initial_segment(&res[r], k, lo, len, side)) {
        n = 1;
        if (P.opt.break_enabled) {
            const int np = walk_break(b.qual + b.offsets[r] + lo, len, P.opt.break_window, P.opt.break_quality,
                                      [](int, int, int) {});
            if (np >= 0) n = np;
        }
    }
    cnt[t] = n;
}

// pass 2: write the pieces
__global__ void k_ext_emit(const __grid_constant__ DevParams P, DevBatch b, const fpl_read_result* __restrict__ res,
                           const int32_t* __restrict__ off, fpl_segment* __restrict__ segs) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * b.n_reads) return;
    const int64_t r = t >> 1;
    const int k = (int)(t & 1);
    int lo, len, side;
    if (!initial_segment(&res[r], k, lo, len, side)) return;
    fpl_segment* out = segs + off[t];
    fpl_segment sg;
    sg.read = (int32_t)r; sg.result = 0; sg.median_qual = 0; sg.split_side = (uint8_t)side; sg.is_r1 = 0;
    int np = -1;
    if (P.opt.break_enabled)
        np = walk_break(b.qual + b.offsets[r] + lo, len, P.opt.break_window, P.opt.break_quality,
                        [&](int plo, int plen, int bidx) {
                            sg.lo = lo + plo; sg.len = plen; sg.break_index = bidx;
                            *out++ = sg;
                        });
    if (np < 0) {   // unbroken: the output read is the initial segment itself (r1 when the read was not split)
        sg.lo = lo; sg.len = len; sg.break_index = 0; sg.is_r1 = side == 0 ? 1 : 0;
        *out = sg;
    }
}

// mask regions per piece: count, then emit + paint 'N' into the private sequence copy
__global__ void k_ext_mask_count(const __grid_constant__ DevParams P, DevBatch b, const fpl_segment* __restrict__ segs,
                                 int64_t nseg, int32_t* __restrict__ cnt) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nseg) return;
    const fpl_segment sg = segs[t];
    int n = 0;
    const int length = sg.len;
    detect_regions(b.qual + b.offsets[sg.read] + sg.lo, length, P.opt.mask_window, P.opt.mask_quality, [&](int first, int last) {
        const int start = first, len = last - first + 1;
        if (start < 0 || len <= 0 || start >= length) return;   // what Read::maskRegionWithN itself skips
        n++;
    });
    cnt[t] = n;
}

__global__ void k_ext_mask_emit(const __grid_constant__ DevParams P, DevBatch b, const fpl_segment* __restrict__ segs,
                                int64_t nseg, const int32_t* __restrict__ off, fpl_region* __restrict__ regs,
                                uint8_t* __restrict__ mseq) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nseg) return;
    const fpl_segment sg = segs[t];
    fpl_region* out = regs + off[t];
    const int length = sg.len;
    uint8_t* base = mseq + b.offsets[sg.read] + sg.lo;
    detect_regions(b.qual + b.offsets[sg.read] + sg.lo, length, P.opt.mask_window, P.opt.mask_quality, [&](int first, int last) {
        int start = first, len = last - first + 1;
        if (start < 0 || len <= 0 || start >= length) return;
        if (start + len > length) len = length - start;
        for (int i = 0; i < len; i++) base[start + i] = 'N';
        fpl_region rg; rg.read = sg.read; rg.lo = sg.lo + start; rg.len = len;
        *out++ = rg;
    });
}

// Filter::passFilter per output read (one warp each) on the (masked) sequence; builds the post-filter Stats segments
namespace {
struct Counts { int lowq, nn, totalq, diff; };
__device__ int pass_filter_ext(const fpl_options& o, int rlen, const Counts& c) {
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
        if (!((long long)c.diff * 100 >= (long long)o.complexity_threshold_pct * (rlen - 1))) return FPL_FAIL_COMPLEXITY;
    }
    return FPL_PASS_FILTER;
}
}  // namespace

#define EF_WARPS 8
__global__ void __launch_bounds__(EF_WARPS * 32)
k_ext_filter(const __grid_constant__ DevParams P, DevBatch b, const uint8_t* __restrict__ fseq, fpl_segment* __restrict__ segs,
             int64_t nseg, StatSeg* __restrict__ stat, unsigned long long* __restrict__ counters) {
    const int lane = lane_id();
    const int64_t t = (int64_t)blockIdx.x * EF_WARPS + (threadIdx.x >> 5);
    if (t >= nseg) return;
    const fpl_segment sg = segs[t];
    const int64_t off = b.offsets[sg.read] + sg.lo;
    const uint8_t* seq = fseq + off;
    const uint8_t* qual = b.qual + off;
    const fpl_options& o = P.opt;
    Counts c = {0, 0, 0, 0};
    const bool doCounts = (o.qual_filter_enabled || o.length_filter_enabled);
    const int qq = (int)(signed char)o.qualified_qual;
    for (int i = lane; i < sg.len; i += 32) {
        if (doCounts) {
            const int q = (int)(signed char)qual[i];
            c.totalq += q - 33; c.lowq += q < qq; c.nn += seq[i] == 'N';
        }
        if (o.complexity_enabled && i < sg.len - 1) c.diff += seq[i] != seq[i + 1];
    }
    c.lowq = __reduce_add_sync(0xffffffffu, c.lowq); c.nn = __reduce_add_sync(0xffffffffu, c.nn);
    c.totalq = __reduce_add_sync(0xffffffffu, c.totalq); c.diff = __reduce_add_sync(0xffffffffu, c.diff);
    const int code = pass_filter_ext(o, sg.len, c);
    if (lane == 0) {
        segs[t].result = (uint8_t)code;
        atomicAdd(&counters[FPL_CNT_FILTER + code], 1ull);
        StatSeg ps = {0, 0, -1, 0, 0};
        if (code == FPL_PASS_FILTER) { ps.off = off; ps.len = sg.len; ps.read = (int)t; ps.slot = 0; }
        stat[t] = ps;
    }
}

// post-filter quality histogram + median per passing output read (one warp each)
#define EQ_WARPS 8
__global__ void __launch_bounds__(EQ_WARPS * 32)
k_ext_seg_qual(const uint8_t* __restrict__ qualbuf, const StatSeg* __restrict__ stat, int64_t nseg,
               unsigned long long* __restrict__ stats_post, int64_t C, fpl_segment* __restrict__ segs) {
    __shared__ uint32_t hist[EQ_WARPS][128];
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const int64_t t = (int64_t)blockIdx.x * EQ_WARPS + wid;
    if (t >= nseg) return;
    const StatSeg sg = stat[t];
    if (sg.read < 0) return;
    uint32_t* h = hist[wid];
    for (int i = lane; i < 128; i += 32) h[i] = 0;
    __syncwarp();
    const uint8_t* qp = qualbuf + sg.off;
    for (int i = lane; i < sg.len; i += 32) atomicAdd(&h[qp[i] & 127], 1u);
    __syncwarp();
    unsigned long long* tail = stats_post + 16 * C;
    const uint32_t h0 = h[4 * lane], h1 = h[4 * lane + 1], h2 = h[4 * lane + 2], h3 = h[4 * lane + 3];
    uint8_t median = 0;
    if (sg.len > 0) {
        const int half = sg.len >> 1;
        const int tot = (int)(h0 + h1 + h2 + h3);
        int run = warp_incl_scan(tot) - tot;
        int m = 1 << 30;
        run += h0; if (run > half) m = min(m, 4 * lane);
        run += h1; if (run > half) m = min(m, 4 * lane + 1);
        run += h2; if (run > half) m = min(m, 4 * lane + 2);
        run += h3; if (run > half) m = min(m, 4 * lane + 3);
        median = (uint8_t)__reduce_min_sync(0xffffffffu, m);
    }
    if (h0) atomicAdd(&tail[FPL_STATS_QUALHIST + 4 * lane], (unsigned long long)h0);
    if (h1) atomicAdd(&tail[FPL_STATS_QUALHIST + 4 * lane + 1], (unsigned long long)h1);
    if (h2) atomicAdd(&tail[FPL_STATS_QUALHIST + 4 * lane + 2], (unsigned long long)h2);
    if (h3) atomicAdd(&tail[FPL_STATS_QUALHIST + 4 * lane + 3], (unsigned long long)h3);
    if (lane == 0) {
        atomicAdd(&tail[FPL_STATS_READS], 1ull);
        atomicAdd(&tail[FPL_STATS_LENSUM], (unsigned long long)sg.len);
        if (sg.len > 0) {
            atomicAdd(&tail[FPL_STATS_MEDHIST + median], 1ull);
            atomicAdd(&tail[FPL_STATS_MEDBASES + median], (unsigned long long)sg.len);
        }
        segs[t].median_qual = median;
    }
}

// records: total number of output reads + the first two inline
__global__ void k_ext_fill_records(int64_t n_reads, const int32_t* __restrict__ off, const fpl_segment* __restrict__ segs,
                                   fpl_read_result* __restrict__ res) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    const int s0 = off[2 * r], s1 = off[2 * r + 2];
    fpl_read_result* o = &res[r];
    o->n_segments = s1 - s0;
    for (int k = 0; k < 2; k++) {
        if (s0 + k < s1) {
            const fpl_segment sg = segs[s0 + k];
            o->seg_lo[k] = sg.lo; o->seg_len[k] = sg.len; o->seg_result[k] = sg.result; o->seg_median_qual[k] = sg.median_qual;
        } else {
            o->seg_lo[k] = 0; o->seg_len[k] = 0; o->seg_result[k] = 0; o->seg_median_qual[k] = 0;
        }
    }
}

// Runs after k_final (which left the initial segments in the records).  Returns the sequence buffer the post-filter
// Stats must read (the masked copy when --mask is on) through *fseq_out, and the StatSeg list in x->d_stat.
int fpl_ext_run(FplExt* x, const DevParams& P, const DevBatch& b, int64_t n_bytes, fpl_read_result* res,
                unsigned long long* counters, unsigned long long* stats_post, int64_t C, const uint8_t** fseq_out,
                cudaStream_t s, char* err, size_t errlen) {
    const int64_t n = b.n_reads;
    x->n_segs = 0; x->n_regs = 0;
    *fseq_out = b.seq;
    if (n == 0) return 0;
    if (2 * n + 1 >= (1ll << 31)) { snprintf(err, errlen, "too many reads for --mask/--break in one call"); return -1; }
    FPL_CK_ERR(x->d_cnt.grow(2 * n + 1));
    FPL_CK_ERR(x->d_off.grow(2 * n + 1));
    const unsigned g2 = (unsigned)((2 * n + 255) / 256);
    k_ext_count<<<g2, 256, 0, s>>>(P, b, res, x->d_cnt);
    FPL_CK_ERR(cudaMemsetAsync(x->d_cnt + 2 * n, 0, sizeof(int32_t), s));
    FPL_CK_ERR(cub_call(x->d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, x->d_cnt.get(), x->d_off.get(), 2 * n + 1, s); }));
    int32_t total = 0;
    FPL_CK_ERR(cudaMemcpyAsync(&total, x->d_off + 2 * n, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    FPL_CK_ERR(cudaStreamSynchronize(s));
    x->n_segs = total;
    FPL_CK_ERR(x->d_segs.grow((int64_t)total + 1));
    FPL_CK_ERR(x->d_stat.grow((int64_t)total + 1));
    k_ext_emit<<<g2, 256, 0, s>>>(P, b, res, x->d_off, x->d_segs);
    if (P.opt.mask_enabled && total > 0) {
        // the masked copy is a batch of its own: its tail pad is defined, not whatever the buffer held before
        FPL_CK_ERR(x->d_mseq.grow(FPL_BATCH_BYTES(n_bytes)));
        FPL_CK_ERR(cudaMemcpyAsync(x->d_mseq, b.seq, (size_t)n_bytes, cudaMemcpyDeviceToDevice, s));
        FPL_CK_ERR(cudaMemsetAsync(x->d_mseq + n_bytes, 0, (size_t)(FPL_BATCH_BYTES(n_bytes) - n_bytes), s));
        FPL_CK_ERR(x->d_rcnt.grow((int64_t)total + 1));
        FPL_CK_ERR(x->d_roff.grow((int64_t)total + 1));
        const unsigned gs = (unsigned)((total + 255) / 256);
        k_ext_mask_count<<<gs, 256, 0, s>>>(P, b, x->d_segs, total, x->d_rcnt);
        FPL_CK_ERR(cudaMemsetAsync(x->d_rcnt + total, 0, sizeof(int32_t), s));
        FPL_CK_ERR(cub_call(x->d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, x->d_rcnt.get(), x->d_roff.get(), (int64_t)total + 1, s); }));
        int32_t nreg = 0;
        FPL_CK_ERR(cudaMemcpyAsync(&nreg, x->d_roff + total, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        FPL_CK_ERR(cudaStreamSynchronize(s));
        x->n_regs = nreg;
        FPL_CK_ERR(x->d_regs.grow((int64_t)nreg + 1));
        k_ext_mask_emit<<<gs, 256, 0, s>>>(P, b, x->d_segs, total, x->d_roff, x->d_regs, x->d_mseq);
        *fseq_out = x->d_mseq;
    }
    if (total > 0) {
        k_ext_filter<<<(unsigned)((total + EF_WARPS - 1) / EF_WARPS), EF_WARPS * 32, 0, s>>>(P, b, *fseq_out, x->d_segs, total,
                                                                                      x->d_stat, counters);
        k_ext_seg_qual<<<(unsigned)((total + EQ_WARPS - 1) / EQ_WARPS), EQ_WARPS * 32, 0, s>>>(b.qual, x->d_stat, total,
                                                                                      stats_post, C, x->d_segs);
    }
    k_ext_fill_records<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(n, x->d_off, x->d_segs, res);
    FPL_CK_ERR(cudaGetLastError());
    return 0;
}
