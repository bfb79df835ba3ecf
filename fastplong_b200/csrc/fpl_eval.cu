// SURVEY §8f row 4: the counting half of Evaluator::evalAdapterAndReadNum (src/evaluator.cpp:105-265) on the device.
// The reference walks the first (side 0) or last (side 1) 128 ten-mer positions of up to 64 Ki reads and fills two
// tables indexed by the 2-bit-packed ten-mer (A 0, T/U 1, C 2, G 3, first base most significant; seq2int :503-560):
// counts[key] and positionAcc[key] (sum of pos, or of len - pos at the read end).  seq2int's rolling form is the
// closed form "all ten bases of [pos, pos + 10) are A/C/G/T/U".  One warp per read, one position per lane and round,
// global atomics into the two 4^10-entry tables (8 M updates for 64 Ki reads: microseconds).  Choosing the top key and
// growing it into the adapter stays on the host (fastplong_b200/evaluator.py), as O(4^10) table work.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "fplgpu.h"
#include "fpl_buf.h"

namespace {
constexpr int KEYLEN = 10;

__device__ __forceinline__ int base_code(uint32_t b) {
    return b == 'A' ? 0 : (b == 'T' || b == 'U') ? 1 : b == 'C' ? 2 : b == 'G' ? 3 : -1;
}

__global__ void __launch_bounds__(256)
k_eval_kmers(const uint8_t* __restrict__ seq, const int64_t* __restrict__ offsets, const int32_t* __restrict__ lens, int64_t n_reads,
             int shift_tail, int side, unsigned int* __restrict__ counts, unsigned long long* __restrict__ pos_acc,
             unsigned long long* __restrict__ total) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n_reads) return;
    const int len = lens[r];
    const uint8_t* s = seq + offsets[r];
    const int last = len - KEYLEN - shift_tail;                      // the loops run while pos <= last
    int p0, p1;                                                      // [p0, p1]
    if (side == 0) { p0 = 0; p1 = min(last, 127); }
    else { p0 = max(0, last - 128); p1 = last; }
    unsigned long long mine = 0;
    for (int pos = p0 + lane; pos <= p1; pos += 32) {
        int key = 0;
        bool ok = true;
#pragma unroll
        for (int i = 0; i < KEYLEN; i++) {
            const int c = base_code(s[pos + i]);
            ok = ok && c >= 0;
            key = (key << 2) | (c & 3);
        }
        if (ok) {
            atomicAdd(&counts[key], 1u);
            atomicAdd(&pos_acc[key], (unsigned long long)(side == 0 ? pos : len - pos));
            mine++;
        }
    }
    mine = __reduce_add_sync(0xffffffffu, (unsigned)mine);
    if (lane == 0 && mine) atomicAdd(total, mine);
}
}  // namespace

extern "C" int fpl_eval_adapter_kmers(int device, const fpl_batch* b, int32_t shift_tail, int32_t side, uint32_t* counts,
                                      uint64_t* position_acc, int64_t* total) {
    if (!b || !counts || !position_acc || !total || side < 0 || side > 1 || shift_tail < 0 || b->n_reads < 0) return -1;
    if (cudaSetDevice(device) != cudaSuccess) return -2;
    const size_t size = (size_t)1 << (2 * KEYLEN);
    DevBuf<uint8_t> d_seq; DevBuf<int64_t> d_off; DevBuf<int32_t> d_len;
    DevBuf<unsigned int> d_cnt; DevBuf<unsigned long long> d_acc, d_tot;
    const int64_t n = b->n_reads;
    // only the two ends of every read are looked at, but the packed layout is uploaded as it is (64 Ki reads at most)
    if (d_seq.grow_exact(b->n_bytes + 64) || d_off.grow_exact(n + 1) || d_len.grow_exact(n + 1) || d_cnt.grow_exact(size) ||
        d_acc.grow_exact(size) || d_tot.grow_exact(1))
        return -3;
    cudaMemcpy(d_seq, b->seq, (size_t)b->n_bytes, cudaMemcpyHostToDevice);
    cudaMemcpy(d_off, b->offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice);
    cudaMemcpy(d_len, b->lens, sizeof(int32_t) * n, cudaMemcpyHostToDevice);
    cudaMemset(d_cnt, 0, sizeof(unsigned int) * size);
    cudaMemset(d_acc, 0, sizeof(unsigned long long) * size);
    cudaMemset(d_tot, 0, sizeof(unsigned long long));
    if (n) k_eval_kmers<<<(unsigned)((n * 32 + 255) / 256), 256>>>(d_seq, d_off, d_len, n, shift_tail, side, d_cnt, d_acc, d_tot);
    unsigned long long t = 0;
    int rc = 0;
    if (cudaMemcpy(counts, d_cnt, sizeof(unsigned int) * size, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(position_acc, d_acc, sizeof(unsigned long long) * size, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(&t, d_tot, sizeof(t), cudaMemcpyDeviceToHost) != cudaSuccess)
        rc = -4;
    *total = (int64_t)t;
    return rc;
}

// ---- the table half (host only): Evaluator::getTopKey + the acceptance rule + Evaluator::extendKeyToAdapter ----
namespace {
constexpr int EV_SIZE = 1 << (2 * KEYLEN);
constexpr int EV_MAX_LEN = 64;

// src/evaluator.cpp:266-322.  `val` is the COUNT: the reference's "neighbouring bases differ" loop shifts it, not the key.
int ev_top_key(const uint32_t* counts) {
    int top = -1;
    uint32_t topCount = 0;
    for (int k = 1; k < EV_SIZE; k++) {                   // k == 0 (AAAAAAAAAA) is never a top key (:310, and its count is ignored)
        const uint32_t val = counts[k];
        if (val <= topCount) continue;                    // only a strictly larger count can replace the top key
        int n[4] = {0, 0, 0, 0};
        for (int i = 0; i < KEYLEN; i++) n[(k >> (2 * i)) & 3]++;
        int zero = 0;
        bool low = false;
        for (int b = 0; b < 4; b++) { low = low || n[b] >= KEYLEN - 4; zero += n[b] == 0; }
        low = low || zero >= 2 || (k >> KEYLEN) == (k & ((1 << KEYLEN) - 1));
        int diff = 0;
        for (int s = 0; s < KEYLEN - 1; s++)
            diff += ((val >> ((KEYLEN - s) * 2)) & 3u) != ((val >> ((KEYLEN - s - 1) * 2)) & 3u);
        if (diff < 3 || low) continue;
        if (n[2] + n[3] >= KEYLEN - 2) continue;          // too many C/G
        if ((k >> 12) == 0xff) continue;                  // starts with GGGG
        topCount = val;
        top = k;
    }
    return top;
}

// src/evaluator.cpp:324-407; returns the length written into out (<= EV_MAX_LEN).
int ev_extend(int key, const uint32_t* counts, const uint64_t* acc, bool rna, char* out) {
    const char bases[4] = {'A', rna ? 'U' : 'T', 'C', 'G'};
    const int mask = EV_SIZE - 1;
    char buf[2 * EV_MAX_LEN + KEYLEN];                    // grows to both sides of the middle
    int lo = EV_MAX_LEN, hi = EV_MAX_LEN;
    for (int i = 0; i < KEYLEN; i++) buf[hi++] = bases[(key >> (2 * (KEYLEN - 1 - i))) & 3];
    bool leftDone = false, rightDone = false, left = true;
    while (true) {
        int cur = key;
        while (hi - lo < EV_MAX_LEN) {
            int nk[4];
            long long totalCount = 0;
            uint32_t cnk[4];                                  // the reference zeroes counts[AAAAAAAAAA] before all of this (:195)
            for (int b = 0; b < 4; b++) {
                nk[b] = left ? ((b << ((KEYLEN - 1) * 2)) | (cur >> 2)) : (b | (mask & (cur << 2)));
                cnk[b] = nk[b] == 0 ? 0u : counts[nk[b]];
                totalCount += cnk[b];
            }
            bool extended = false;
            for (int b = 0; b < 4 && !extended; b++) {
                const uint32_t cn = cnk[b];
                if (cn == 0) continue;
                const double offset = (double)acc[nk[b]] / cn - (double)acc[cur] / counts[cur];
                if ((double)cn / (double)totalCount < 0.7) continue;
                if ((double)cn / (double)counts[key] < 0.5) continue;
                if (offset > 2 || offset < -4) continue;
                cur = nk[b];
                extended = true;
                if (left) buf[--lo] = bases[b]; else buf[hi++] = bases[b];
            }
            if (!extended) { (left ? leftDone : rightDone) = true; break; }
            if (hi - lo == EV_MAX_LEN) { leftDone = rightDone = true; break; }
        }
        left = !left;
        if (leftDone && rightDone) break;
    }
    const int n = hi - lo;
    for (int i = 0; i < n; i++) out[i] = buf[lo + i];
    return n;
}
}  // namespace

extern "C" int fpl_eval_pick_adapter(const uint32_t* counts, const uint64_t* position_acc, int64_t total, int32_t is_rna,
                                     char* adapter, int32_t cap) {
    if (!counts || !position_acc || !adapter || cap < EV_MAX_LEN + 1 || total < 0) return -1;
    adapter[0] = 0;
    long long keys = 0;                                   // src/evaluator.cpp:190-193 (before AAAAAAAAAA is zeroed)
    for (int k = 0; k < EV_SIZE; k++) keys += counts[k] > 0;
    const int key = ev_top_key(counts);
    if (key < 0) return 0;
    const long long count = counts[key];
    if (!(count > 10 && (double)(count * keys) > (double)total * 100.0)) return 0;
    char buf[EV_MAX_LEN + 1];
    const int n = ev_extend(key, counts, position_acc, is_rna != 0, buf);
    if (n <= 16) return 0;                                // "too short" (:203): the option stays "auto"
    for (int i = 0; i < n; i++) adapter[i] = buf[i];
    adapter[n] = 0;
    return n;
}

