// FASTQ ingest on the device (SURVEY §8f row 1): FastqReader::getLine / FastqReader::read
// (src/fastqreader.cpp:219-347) for a chunk of plain-text FASTQ, as three small HBM-bound kernels:
//   newline index   cub::DeviceSelect over the byte positions whose byte is '\n'  (+ a '\r' detector)
//   k_fastq_records one thread per record: the four line extents, the checks FastqReader::read makes
//                   ('@' first, '+' third line, |sequence| == |quality|), the slot size of the packed layout
//   k_fastq_pack    one warp per record: sequence and quality lines -> the packed batch layout (aligned slots)
// Only the strict layout (LF line ends, exactly four lines per record, no blank lines) is handled here; anything else
// is reported to the caller, which then parses that input with the reference's own reader.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include "fpl_device.cuh"
#include "fpl_ingest.h"

namespace {

struct IsNewline {
    const uint8_t* text;
    __device__ __forceinline__ bool operator()(const int64_t& i) const { return text[i] == '\n'; }
};

// misc[0] += number of '\n', misc[4] |= 1 if any '\r' (16 bytes per thread, one 16-byte load each: text is 16-byte aligned)
__global__ void k_count_lines(const uint8_t* __restrict__ text, int64_t n, unsigned long long* __restrict__ misc) {
    const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16;
    int cnt = 0;
    bool cr = false;
    if (i0 < n) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(text + i0));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t b = (w[k] >> (8 * j)) & 0xFFu;
                const bool in = i0 + 4 * k + j < n;
                cnt += in && b == '\n';
                cr |= in && b == '\r';
            }
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane_id() == 0 && cnt) atomicAdd(&misc[0], (unsigned long long)cnt);
    if (__any_sync(0xffffffffu, cr) && lane_id() == 0) atomicOr(reinterpret_cast<int*>(&misc[4]), 1);
}

// line l spans [start, end): start = (l ? nl[l-1] + 1 : 0), end = (l < n_nl ? nl[l] : n)  (virtual newline at EOF)
__global__ void k_fastq_records(const uint8_t* __restrict__ text, int64_t n, const int64_t* __restrict__ nl, int64_t n_nl,
                                int64_t n_records, fpl_fastq_record* __restrict__ rec, int32_t* __restrict__ lens,
                                int64_t* __restrict__ slots, unsigned long long* __restrict__ first_bad) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_records) return;
    int64_t st[4], en[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int64_t l = 4 * r + k;
        st[k] = l ? nl[l - 1] + 1 : 0;
        en[k] = l < n_nl ? nl[l] : n;
    }
    fpl_fastq_record o;
    o.name_off = st[0]; o.seq_off = st[1]; o.plus_off = st[2]; o.qual_off = st[3];
    o.name_len = (int32_t)(en[0] - st[0]); o.seq_len = (int32_t)(en[1] - st[1]);
    o.plus_len = (int32_t)(en[2] - st[2]); o.reserved = 0;
    const bool ok = o.name_len >= 1 && text[st[0]] == '@' && o.plus_len >= 1 && text[st[2]] == '+' &&
                    (en[3] - st[3]) == (en[1] - st[1]) && (en[1] - st[1]) < (1ll << 31);
    if (!ok) atomicMin(first_bad, (unsigned long long)r);
    rec[r] = o;
    lens[r] = o.seq_len;
    slots[r] = ((int64_t)o.seq_len + FPL_SLOT_ALIGN - 1) / FPL_SLOT_ALIGN * FPL_SLOT_ALIGN;
}

// dst is 4-byte aligned (slots are FPL_SLOT_ALIGN-aligned); src is arbitrary: each lane assembles whole words
__device__ __forceinline__ void copy_line(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int n, int lane) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(src);
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const unsigned sh = (unsigned)(a & 3) * 8;
    uint32_t* dw = reinterpret_cast<uint32_t*>(dst);
    const int nw = n >> 2;
    for (int k = lane; k < nw; k += 32) {
        const uint32_t lo = __ldg(sw + k);
        dw[k] = sh ? __funnelshift_r(lo, __ldg(sw + k + 1), sh) : lo;
    }
    const int tail = nw << 2;
    if (tail + lane < n) dst[tail + lane] = src[tail + lane];   // < 4 bytes
}

__global__ void __launch_bounds__(256)
k_fastq_pack(const uint8_t* __restrict__ text, const fpl_fastq_record* __restrict__ rec, const int64_t* __restrict__ offsets,
             int64_t n_records, uint8_t* __restrict__ seq, uint8_t* __restrict__ qual) {
    const int lane = lane_id();
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_records; r += nwarps) {
        const fpl_fastq_record o = rec[r];
        copy_line(seq + offsets[r], text + o.seq_off, o.seq_len, lane);
        copy_line(qual + offsets[r], text + o.qual_off, o.seq_len, lane);
    }
}

}  // namespace

int fpl_ingest_index(FplIngest* g, const uint8_t* h_text, int64_t n, int is_last, cudaStream_t s, int64_t* n_records,
                     int64_t* consumed, char* err, size_t errlen) {
    *n_records = 0; *consumed = 0;
    if (n == 0) return 0;
    FPL_CK_ERR(g->d_text.grow(n + 64, FPL_INGEST_FIRST_BYTES));
    FPL_CK_ERR(cudaMemcpyAsync(g->d_text, h_text, (size_t)n, cudaMemcpyHostToDevice, s));
    FPL_CK_ERR(cudaMemsetAsync(g->d_text + n, 0, 64, s));
    // misc: [0] newline count, [1] count written by cub, [2] first bad record, [4] CR flag
    FPL_CK_ERR(g->d_misc.grow_exact(8));
    FPL_CK_ERR(cudaMemsetAsync(g->d_misc, 0, 64, s));
    FPL_CK_ERR(cudaMemsetAsync(g->d_misc + 2, 0xFF, 8, s));   // first_bad = ~0
    k_count_lines<<<(unsigned)((n + 16 * 256 - 1) / (16 * 256)), 256, 0, s>>>(g->d_text, n, g->d_misc);
    struct { int64_t n_nl; int has_cr; int pad; } h;
    FPL_CK_ERR(cudaMemcpyAsync(&h.n_nl, g->d_misc, 8, cudaMemcpyDeviceToHost, s));
    FPL_CK_ERR(cudaMemcpyAsync(&h.has_cr, g->d_misc + 4, 4, cudaMemcpyDeviceToHost, s));
    FPL_CK_ERR(cudaStreamSynchronize(s));
    if (h.has_cr) return 1;   // CR line ends: the reference's getLine() has its own rules for them
    g->n_nl = h.n_nl;
    FPL_CK_ERR(g->d_nl.grow(h.n_nl + 1, FPL_INGEST_FIRST_BYTES));
    cub::CountingInputIterator<int64_t> idx(0);
    IsNewline pred{g->d_text};
    FPL_CK_ERR(cub_call(g->d_tmp, [&](void* t, size_t& b) {
        return cub::DeviceSelect::If(t, b, idx, g->d_nl.get(), (int64_t*)(g->d_misc + 1), n, pred, s);
    }, FPL_INGEST_FIRST_BYTES));
    // complete lines: every newline ends one; at the end of the input an unterminated last line counts too
    uint8_t lastc = h_text[n - 1];
    int64_t n_lines = h.n_nl + ((is_last && lastc != '\n') ? 1 : 0);
    const int64_t nrec = n_lines / 4;
    if (is_last && n_lines % 4 != 0) return 1;        // trailing partial record / blank lines: let the reference decide
    if (nrec == 0) return 0;
    FPL_CK_ERR(g->d_rec.grow(nrec, FPL_INGEST_FIRST_BYTES));
    FPL_CK_ERR(g->d_lens.grow(nrec, FPL_INGEST_FIRST_BYTES));
    FPL_CK_ERR(g->d_slots.grow(nrec + 1, FPL_INGEST_FIRST_BYTES));
    FPL_CK_ERR(g->d_offsets.grow(nrec + 1, FPL_INGEST_FIRST_BYTES));
    k_fastq_records<<<(unsigned)((nrec + 255) / 256), 256, 0, s>>>(g->d_text, n, g->d_nl, h.n_nl, nrec, g->d_rec, g->d_lens,
                                                                  g->d_slots, g->d_misc + 2);
    FPL_CK_ERR(cudaMemsetAsync(g->d_slots + nrec, 0, 8, s));
    FPL_CK_ERR(cub_call(g->d_tmp, [&](void* t, size_t& b) {
        return cub::DeviceScan::ExclusiveSum(t, b, g->d_slots.get(), g->d_offsets.get(), nrec + 1, s);
    }, FPL_INGEST_FIRST_BYTES));
    unsigned long long first_bad = 0;
    int64_t total = 0;
    FPL_CK_ERR(cudaMemcpyAsync(&first_bad, g->d_misc + 2, 8, cudaMemcpyDeviceToHost, s));
    FPL_CK_ERR(cudaMemcpyAsync(&total, g->d_offsets + nrec, 8, cudaMemcpyDeviceToHost, s));
    FPL_CK_ERR(cudaStreamSynchronize(s));
    if (first_bad != ~0ull) return 1;   // a record the strict layout does not describe
    g->packed_bytes = total;
    *n_records = nrec;
    // bytes consumed = through the newline that ends the last complete record (or the whole input)
    int64_t last_nl_idx = 4 * nrec - 1;
    if (last_nl_idx < h.n_nl) {
        int64_t pos = 0;
        FPL_CK_ERR(cudaMemcpy(&pos, g->d_nl + last_nl_idx, 8, cudaMemcpyDeviceToHost));
        *consumed = pos + 1;
    } else {
        *consumed = n;
    }
    return 0;
}

int fpl_ingest_pack(FplIngest* g, int64_t nrec, uint8_t* d_seq, uint8_t* d_qual, cudaStream_t s, char* err, size_t errlen) {
    if (nrec == 0) return 0;
    const int64_t want = (nrec + 7) / 8;
    k_fastq_pack<<<(unsigned)(want < FPL_NUM_SMS * 32 ? want : FPL_NUM_SMS * 32), 256, 0, s>>>(g->d_text, g->d_rec, g->d_offsets, nrec, d_seq, d_qual);
    FPL_CK_ERR(cudaGetLastError());
    return 0;
}
