// Output assembly on the device (SURVEY §8f row 2, device half): the output reads of the last fpl_process_* call, in the
// order processSingleEnd hands them to the two writers (src/seprocessor.cpp:264-288).  The records, the batch and — with
// --mask / --break — the list of output reads and the masked bases are already in HBM, so both sinks are stream compactions.
// FASTQ text (fpl_emit_fastq_host): Read::appendToString / appendToStringWithTag (src/read.cpp:119-173) for a chunk that
// fpl_process_fastq_host has just processed:
//   k_emit_sizes        thread per read: bytes this read contributes to --out and to --failed_out
//   cub scan            one exclusive sum over both size vectors -> where each read's text starts
//   k_emit_copy         warp per read: name (+ "r<k>-" / "split-by-adapter-…-" after the '@', or " <reason>" behind it), the
//                       window of the bases, the '+' line as it was, the window of the qualities; 16-byte stores, source
//                       words re-aligned by funnel shifts
// Packed batches (fpl_emit_batch_device), after any fpl_process_* call:
//   k_emit_batch_sizes  thread per read: output reads and slot bytes this read contributes to `out` and to `failed`
//   cub scan            one exclusive sum over the four count vectors -> each read's first output read and first slot byte
//   k_emit_batch_copy   warp per read: the windows of the bases and qualities into 16-byte slots (zero behind the read),
//                       offsets, lengths and the fpl_segment of every output read
// Every kernel walks a read with the same code (walk_read) and differs in the sink only, so sizes cannot drift from bytes
// and the two outputs cannot disagree on which reads go where.
#include <cub/device/device_scan.cuh>
#include "fpl_device.cuh"
#include "fpl_emit.h"

namespace {

// Read::breakByGap's name tags (src/read.cpp:204,209) and the --failed_out reasons by filter result code
// (src/common.h:55-64)
__constant__ char c_left[24] = "split-by-adapter-left-";
__constant__ char c_right[24] = "split-by-adapter-right-";
__constant__ char c_failed[32][24] = {
    "passed", "", "", "", "failed_polyx_filter", "", "", "", "failed_bad_overlap", "", "", "",
    "failed_too_many_n_bases", "", "", "", "failed_too_short", "failed_too_long", "", "",
    "failed_quality_filter", "", "", "", "failed_low_complexity", "", "", "", "", "", "", ""};
__constant__ int c_failed_len[32] = {6, 0, 0, 0, 19, 0, 0, 0, 18, 0, 0, 0, 23, 0, 0, 0, 16, 15, 0, 0, 21, 0, 0, 0, 21, 0, 0, 0, 0, 0, 0, 0};

__device__ __forceinline__ int dec_digits(int v) {
    int nd = 1;
    for (unsigned t = (unsigned)v; t >= 10; t /= 10) nd++;
    return nd;
}

// counts bytes (one thread walks a read)
struct SizeSink {
    int64_t n = 0;
    __device__ __forceinline__ void bytes(const uint8_t*, int64_t k) { n += k; }
    __device__ __forceinline__ void lit(const char*, int k) { n += k; }
    __device__ __forceinline__ void ch(char) { n++; }
    __device__ __forceinline__ void dec(int v) { n += dec_digits(v); }
};

// n bytes from src to dst, any alignment, by one warp.  Every load is an aligned 4-byte word that holds at least one byte of
// [src, src + n): the first word is src's own, and the extra word a re-aligned vector reads (w4, only when src is not
// word-aligned) starts at src + 16 * nv - (src & 3), a byte this call copies.  So the loads stay inside the 16-byte
// vectors that hold the window: inside any fpl_batch, and nothing in front of its offset 0.
__device__ __forceinline__ void warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int64_t n, int lane) {
    if (n <= 0) return;
    int head = (int)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15);
    if (head > n) head = (int)n;
    if (lane < head) dst[lane] = src[lane];
    dst += head; src += head; n -= head;
    const int64_t nv = n >> 4;
    if (nv) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(src);
        const uint32_t* sw = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
        const unsigned sh = (unsigned)(a & 3) * 8;
        uint4* dv = reinterpret_cast<uint4*>(dst);
        for (int64_t k = lane; k < nv; k += 32) {
            const uint32_t* p = sw + 4 * k;
            const uint32_t w0 = __ldg(p), w1 = __ldg(p + 1), w2 = __ldg(p + 2), w3 = __ldg(p + 3);
            uint4 o = make_uint4(w0, w1, w2, w3);
            if (sh) {
                const uint32_t w4 = __ldg(p + 4);
                o = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                               __funnelshift_r(w3, w4, sh));
            }
            dv[k] = o;
        }
    }
    const int64_t done = nv << 4;
    if (lane < (int)(n - done)) dst[done + lane] = src[done + lane];
}

// writes bytes (one warp walks a read; p is warp-uniform)
struct CopySink {
    uint8_t* p;
    int lane;
    __device__ __forceinline__ void bytes(const uint8_t* s, int64_t k) { warp_copy(p, s, k, lane); p += k; }
    __device__ __forceinline__ void lit(const char* s, int k) { if (lane < k) p[lane] = (uint8_t)s[lane]; p += k; }   // k <= 32
    __device__ __forceinline__ void ch(char c) { if (lane == 0) *p = (uint8_t)c; p++; }
    __device__ __forceinline__ void dec(int v) {
        const int nd = dec_digits(v);
        if (lane < nd) {
            unsigned d = 1;
            for (int i = 0; i < nd - 1 - lane; i++) d *= 10;
            p[lane] = (uint8_t)('0' + ((unsigned)v / d) % 10);
        }
        p += nd;
    }
};

template <class Sink>
__device__ __forceinline__ void put_record(Sink& o, const uint8_t* name, int name_len, int bidx, int side, const char* reason,
                                           int reason_len, const uint8_t* bases, const uint8_t* plus, int plus_len,
                                           const uint8_t* qual, int lo, int len) {
    if ((bidx || side) && name_len > 0) {        // the tag goes between the '@' and the rest of the name line
        o.bytes(name, 1);
        if (bidx) { o.ch('r'); o.dec(bidx); o.ch('-'); }
        if (side) o.lit(side == 2 ? c_right : c_left, side == 2 ? 23 : 22);
        o.bytes(name + 1, name_len - 1);
    } else {
        o.bytes(name, name_len);
    }
    if (reason) { o.ch(' '); o.lit(reason, reason_len); }
    o.ch('\n');
    o.bytes(bases + lo, len);
    o.ch('\n');
    o.bytes(plus, plus_len);
    o.ch('\n');
    o.bytes(qual + lo, len);
    o.ch('\n');
}

// One output read as a writer receives it: the window on the original read, the filter code, the name tags, whether it is
// r1 itself, its post-filter median, and whether its bases are the masked copy's
struct OutRead {
    int lo, len, code, side, bidx, is_r1, median;
    bool masked;
};

// Everything read r sends to the two writers, in the reference's order (src/seprocessor.cpp:264-288), as
// visit(to_failed, OutRead): a passing output read goes to --out; a failing one goes to --failed_out only when it is the
// read's only output read, and then as r1 after the trims (the record's trim window, no name tag), masked only if that
// output read is r1 itself.
template <class Visit>
__device__ __forceinline__ void walk_read(const EmitSource& S, int64_t r, bool want_failed, Visit&& visit) {
    const fpl_read_result* rr = S.res + r;
    const int nseg = rr->n_segments;
    const uint32_t flags = rr->flags;
    const int s0 = S.segs ? S.seg_off[2 * r] : 0;
    for (int k = 0; k < nseg; k++) {
        OutRead o;
        if (S.segs) {
            const fpl_segment sg = S.segs[s0 + k];
            o.lo = sg.lo; o.len = sg.len; o.code = sg.result; o.side = sg.split_side; o.bidx = sg.break_index; o.is_r1 = sg.is_r1;
            o.median = sg.median_qual;
        } else {
            o.lo = rr->seg_lo[k]; o.len = rr->seg_len[k]; o.code = rr->seg_result[k]; o.median = rr->seg_median_qual[k];
            o.side = (flags & FPL_FLAG_MIDDLE_ADAPTER) ? ((k == 1 || (flags & FPL_FLAG_SEG0_IS_RIGHT)) ? 2 : 1) : 0;
            o.bidx = 0; o.is_r1 = o.side == 0;
        }
        if (o.code == FPL_PASS_FILTER) {
            o.masked = S.mseq != nullptr;
            visit(false, o);
        } else if (want_failed && nseg == 1) {
            o.lo = rr->trim_lo; o.len = rr->trim_len; o.side = 0; o.bidx = 0;
            o.masked = S.mseq != nullptr && o.is_r1;
            visit(true, o);
        }
    }
}

// the text sink: one output read as its FASTQ record
template <class Sink>
__device__ __forceinline__ void put_text(const EmitSource& S, int64_t r, const fpl_fastq_record& fq, const OutRead& o, bool to_failed,
                                         Sink& out, Sink& failed) {
    const uint8_t* name = S.text + fq.name_off;
    const uint8_t* plus = S.text + fq.plus_off;
    const uint8_t* qual = S.text + fq.qual_off;
    const uint8_t* bases = o.masked ? S.mseq + S.offsets[r] : S.text + fq.seq_off;
    if (!to_failed)
        put_record(out, name, fq.name_len, o.bidx, o.side, nullptr, 0, bases, plus, fq.plus_len, qual, o.lo, o.len);
    else
        put_record(failed, name, fq.name_len, 0, 0, c_failed[o.code & 31], c_failed_len[o.code & 31], bases, plus, fq.plus_len,
                   qual, o.lo, o.len);
}

// size[r] = --out bytes of read r, size[n + 1 + r] = --failed_out bytes (size[n] and size[2n + 1] stay 0: the totals
// appear there after the exclusive sum)
__global__ void k_emit_sizes(const EmitSource S, bool want_failed, int64_t* __restrict__ size) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= S.n_reads) return;
    const fpl_fastq_record fq = S.rec[r];
    SizeSink out, failed;
    walk_read(S, r, want_failed, [&](bool f, const OutRead& o) { put_text(S, r, fq, o, f, out, failed); });
    size[r] = out.n;
    size[S.n_reads + 1 + r] = failed.n;
}

__global__ void __launch_bounds__(256)
k_emit_copy(const EmitSource S, bool want_failed, const int64_t* __restrict__ off, uint8_t* __restrict__ d_out,
            uint8_t* __restrict__ d_failed) {
    const int lane = lane_id();
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t n = S.n_reads;
    const int64_t total_out = off[n];
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nwarps) {
        const fpl_fastq_record fq = S.rec[r];
        CopySink out{d_out + off[r], lane}, failed{d_failed + (off[n + 1 + r] - total_out), lane};
        walk_read(S, r, want_failed, [&](bool f, const OutRead& o) { put_text(S, r, fq, o, f, out, failed); });
    }
}

__device__ __forceinline__ int64_t slot_bytes(int len) { return ((int64_t)len + 15) & ~(int64_t)15; }

// cnt: four vectors of n + 1 entries — output reads to `out`, their slot bytes, output reads to `failed`, their slot bytes —
// whose entry n is 0 (after the exclusive sum over all 4n + 4 entries a vector's total is the difference of its ends)
__global__ void k_emit_batch_sizes(const EmitSource S, int64_t* __restrict__ cnt) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t q = S.n_reads + 1;
    if (r == 0)
        for (int i = 0; i < 4; i++) cnt[i * q + S.n_reads] = 0;
    if (r >= S.n_reads) return;
    int64_t reads_out = 0, bytes_out = 0, reads_failed = 0, bytes_failed = 0;
    walk_read(S, r, true, [&](bool f, const OutRead& o) {
        if (f) { reads_failed++; bytes_failed += slot_bytes(o.len); }
        else { reads_out++; bytes_out += slot_bytes(o.len); }
    });
    cnt[r] = reads_out; cnt[q + r] = bytes_out; cnt[2 * q + r] = reads_failed; cnt[3 * q + r] = bytes_failed;
}

// the window [src, src + n) into the 16-byte aligned slot at dst, the rest of the slot zero
__device__ __forceinline__ void slot_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int n, int lane) {
    warp_copy(dst, src, n, lane);
    const int tail = n & 15;
    if (tail && lane >= tail && lane < 16) dst[(n & ~15) + lane] = 0;
}

// the batch sink: output read j of one destination at slot byte `at`
__device__ __forceinline__ void put_slot(const EmitSource& S, int64_t r, const OutRead& o, const EmitBatchOut& d, int64_t j,
                                         int64_t at, int lane) {
    if (lane == 0) {
        d.offsets[j] = at;
        d.lens[j] = o.len;
        if (d.segs) {
            fpl_segment sg;
            sg.read = (int32_t)r; sg.lo = o.lo; sg.len = o.len; sg.result = (uint8_t)o.code; sg.median_qual = (uint8_t)o.median;
            sg.split_side = (uint8_t)o.side; sg.is_r1 = (uint8_t)o.is_r1; sg.break_index = o.bidx;
            d.segs[j] = sg;
        }
    }
    const int64_t src = S.offsets[r] + o.lo;
    slot_copy(d.seq + at, (o.masked ? S.mseq : S.seq) + src, o.len, lane);
    slot_copy(d.qual + at, S.qual + src, o.len, lane);
}

__global__ void __launch_bounds__(256)
k_emit_batch_copy(const EmitSource S, const int64_t* __restrict__ off, const EmitBatchOut out, const EmitBatchOut failed) {
    const int lane = lane_id();
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t n = S.n_reads, q = n + 1;
    const bool want_failed = failed.seq != nullptr;
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nwarps) {
        int64_t jo = off[r], bo = off[q + r] - off[q];
        int64_t jf = off[2 * q + r] - off[2 * q], bf = off[3 * q + r] - off[3 * q];
        walk_read(S, r, want_failed, [&](bool f, const OutRead& o) {
            if (f) { put_slot(S, r, o, failed, jf++, bf, lane); bf += slot_bytes(o.len); }
            else { put_slot(S, r, o, out, jo++, bo, lane); bo += slot_bytes(o.len); }
        });
    }
}

}  // namespace

#define CKM(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { snprintf(err, errlen, "%s failed: %s", #call, cudaGetErrorString(e_)); return -1; } } while (0)

static int growm(void** p, int64_t* cap, int64_t need, char* err, size_t errlen) {
    if (need <= *cap) return 0;
    int64_t c = *cap ? *cap : (1 << 16);
    while (c < need) c *= 2;
    cudaFree(*p); *p = nullptr; *cap = 0;
    CKM(cudaMalloc(p, (size_t)c));
    *cap = c;
    return 0;
}

int fpl_emit_build(FplEmit* e, const EmitSource& src, bool want_failed, cudaStream_t s, char* err, size_t errlen) {
    e->built = false; e->out_bytes = e->failed_bytes = 0; e->with_failed = want_failed;
    const int64_t n = src.n_reads;
    if (n == 0) { e->built = true; return 0; }
    const int64_t m = 2 * n + 2;
    if (growm((void**)&e->d_size, &e->cap_size, (int64_t)sizeof(int64_t) * m, err, errlen)) return -1;
    if (growm((void**)&e->d_off, &e->cap_off, (int64_t)sizeof(int64_t) * m, err, errlen)) return -1;
    CKM(cudaMemsetAsync(e->d_size + n, 0, sizeof(int64_t), s));
    CKM(cudaMemsetAsync(e->d_size + 2 * n + 1, 0, sizeof(int64_t), s));
    k_emit_sizes<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, want_failed, e->d_size);
    size_t tb = 0;
    CKM(cub::DeviceScan::ExclusiveSum(nullptr, tb, e->d_size, e->d_off, m, s));
    if (growm(&e->d_tmp, &e->cap_tmp, (int64_t)tb + 256, err, errlen)) return -1;
    CKM(cub::DeviceScan::ExclusiveSum(e->d_tmp, tb, e->d_size, e->d_off, m, s));
    int64_t total_out = 0, total_both = 0;
    CKM(cudaMemcpyAsync(&total_out, e->d_off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CKM(cudaMemcpyAsync(&total_both, e->d_off + 2 * n + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CKM(cudaStreamSynchronize(s));
    e->out_bytes = total_out;
    e->failed_bytes = total_both - total_out;
    // + 16: a warp's last 16-byte store never needs a bounds test against the next buffer
    if (growm((void**)&e->d_out, &e->cap_out, e->out_bytes + 16, err, errlen)) return -1;
    if (growm((void**)&e->d_failed, &e->cap_failed, e->failed_bytes + 16, err, errlen)) return -1;
    const int64_t want = (n + 7) / 8;
    k_emit_copy<<<(unsigned)(want < FPL_NUM_SMS * 16 ? want : FPL_NUM_SMS * 16), 256, 0, s>>>(src, want_failed, e->d_off, e->d_out, e->d_failed);
    CKM(cudaGetLastError());
    e->built = true;
    return 0;
}

void fpl_emit_free(FplEmit* e) {
    cudaFree(e->d_size); cudaFree(e->d_off); cudaFree(e->d_out); cudaFree(e->d_failed); cudaFree(e->d_tmp);
    *e = FplEmit();
}

int fpl_emit_batch_reserve(FplBatchEmit* e, int64_t n_reads, char* err, size_t errlen) {
    const int64_t m = 4 * (n_reads + 1);
    if (growm((void**)&e->d_cnt, &e->cap_cnt, (int64_t)sizeof(int64_t) * m, err, errlen)) return -1;
    if (growm((void**)&e->d_off, &e->cap_off, (int64_t)sizeof(int64_t) * m, err, errlen)) return -1;
    return 0;
}

void launch_emit_batch_sizes(const EmitSource& src, int64_t* cnt, cudaStream_t s) {
    k_emit_batch_sizes<<<(unsigned)((src.n_reads + 255) / 256), 256, 0, s>>>(src, cnt);
}

int fpl_emit_batch_scan(FplBatchEmit* e, int64_t n_reads, cudaStream_t s, char* err, size_t errlen) {
    const int64_t q = n_reads + 1, m = 4 * q;
    size_t tb = 0;
    CKM(cub::DeviceScan::ExclusiveSum(nullptr, tb, e->d_cnt, e->d_off, m, s));
    if (growm(&e->d_tmp, &e->cap_tmp, (int64_t)tb + 256, err, errlen)) return -1;
    CKM(cub::DeviceScan::ExclusiveSum(e->d_tmp, tb, e->d_cnt, e->d_off, m, s));
    int64_t end[4] = {0, 0, 0, 0};    // running sum at the end of each vector (its entry n is 0, so that is the next one's start)
    for (int i = 0; i < 4; i++) CKM(cudaMemcpyAsync(&end[i], e->d_off + (i + 1) * q - 1, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CKM(cudaStreamSynchronize(s));
    e->n_out = end[0]; e->out_bytes = end[1] - end[0]; e->n_failed = end[2] - end[1]; e->failed_bytes = end[3] - end[2];
    return 0;
}

void launch_emit_batch_copy(const EmitSource& src, const int64_t* off, const EmitBatchOut& out, const EmitBatchOut& failed,
                            cudaStream_t s) {
    const int64_t want = (src.n_reads + 7) / 8;
    k_emit_batch_copy<<<(unsigned)(want < FPL_NUM_SMS * 16 ? want : FPL_NUM_SMS * 16), 256, 0, s>>>(src, off, out, failed);
}

void fpl_emit_batch_free(FplBatchEmit* e) {
    cudaFree(e->d_cnt); cudaFree(e->d_off); cudaFree(e->d_tmp);
    *e = FplBatchEmit();
}
