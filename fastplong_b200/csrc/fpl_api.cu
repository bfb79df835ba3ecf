// C-ABI implementation of include/fplgpu.h: context management, device tables, batch tiling and kernel sequencing.
// No CPU fallback anywhere: every entry point fails loudly when CUDA is unusable.
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <algorithm>
#include <map>
#include <string>
#include <vector>
#include <dlfcn.h>
#include <nccl.h>
#include <cub/device/device_scan.cuh>
#include "fpl_device.cuh"
#include "fpl_scanplan.h"
#include "fpl_stats.h"
#include "fpl_jit.h"
#include "fpl_ingest.h"
#include "fpl_ext.h"
#include "fpl_emit.h"
#include "fpl_buf.h"

static_assert(sizeof(fpl_options) == 144, "fpl_options ABI size");
static_assert(sizeof(fpl_segment) == 20 && sizeof(fpl_region) == 12, "segment / region ABI size");
static_assert(sizeof(fpl_read_result) == 64, "fpl_read_result ABI size");
static_assert(sizeof(ReadState) == 64, "ReadState size");
static_assert(sizeof(StatSeg) == 24, "StatSeg size");

#define QH_STRIPES 128      // stripes of k_scan_jit's histogram sums (fpl_scan_jit2_src.h)

// kernel launchers (fpl_trim.cu, fpl_scan.cu, fpl_stats.cu)
void launch_trim(const DevParams&, const DevBatch&, ReadState*, fpl_read_result*, unsigned long long*, cudaStream_t);
void launch_scan(const DevParams&, const DevBatch&, ReadState*, cudaStream_t);
void launch_scan_fast(const DevParams&, const ScanPlan&, const DevBatch&, ReadState*, cudaStream_t);
void launch_final(const DevParams&, const DevBatch&, const ReadState*, fpl_read_result*, StatSeg*, int32_t*, int*, cudaStream_t);
void launch_count(const fpl_read_result*, int64_t, unsigned long long*, bool, const int32_t*, unsigned long long*, unsigned long long*,
                  int64_t, cudaStream_t);
int launch_cycle_stats(CycleWs*, const uint8_t*, const uint8_t*, const StatSeg*, int64_t, int64_t, unsigned long long*, int64_t,
                        bool, unsigned long long*, bool, const StatSeg*, unsigned long long*, const StatSeg*, cudaStream_t);
void launch_kmer_fix(const DevBatch&, const fpl_read_result*, unsigned long long*, cudaStream_t);
void launch_read_qual(const DevBatch&, unsigned long long*, unsigned long long*, int64_t, fpl_read_result*, bool, cudaStream_t);
void launch_read_qual_exc(const DevBatch&, const ReadState*, const int32_t*, const int*, unsigned long long*, unsigned long long*, int64_t,
                          fpl_read_result*, cudaStream_t);
void launch_qhist_fold(const unsigned long long*, int, unsigned long long*, unsigned long long*, int64_t, cudaStream_t);
void launch_make_preseg(const DevBatch&, StatSeg*, cudaStream_t);
void launch_report_cycles(const unsigned long long*, const unsigned long long*, int64_t, unsigned long long*, cudaStream_t);
void launch_report_sizes(const ReportCurves&, int64_t*, cudaStream_t);
void launch_report_text(const ReportCurves&, const int64_t*, const uint8_t*, const int64_t*, const int64_t*, int, uint8_t*, cudaStream_t);
void launch_html_capture(const fpl_read_result*, const int32_t*, int64_t, const fpl_segment*, int64_t, HtmlEntry*, HtmlEntry*, cudaStream_t);
void launch_html_hist(const HtmlEntry*, int64_t, int64_t, long long*, cudaStream_t);
void launch_html_scatter(const HtmlEntry*, int64_t, int64_t, const long long*, HtmlEntry*, cudaStream_t);
void launch_html_lenhist(const HtmlEntry*, int64_t, unsigned long long*, cudaStream_t);
void launch_html_lenprod(const unsigned long long*, int64_t, long long*, cudaStream_t);
void launch_html_lensearch(const unsigned long long*, const long long*, const long long*, const long long*, int64_t, long long,
                           unsigned long long, int*, cudaStream_t);
void launch_html_bins(const unsigned long long*, int64_t, int64_t, unsigned long long*, cudaStream_t);
void launch_html_values(const unsigned long long*, int64_t, int64_t, int, double*, cudaStream_t);
void launch_html_sums(const double*, int64_t, const long long*, int64_t, double*, cudaStream_t);
void launch_html_sizes(const HtmlText&, int64_t*, cudaStream_t);
void launch_html_text(const HtmlText&, const int64_t*, const uint8_t*, const int64_t*, const int64_t*, int, uint8_t*, cudaStream_t);

static thread_local char g_err[512] = "";

static int fail(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return -1;
}

#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) return fail("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

enum { K_PRESEG, K_CYCLE_PRE, K_QUAL_PRE, K_TRIM, K_SCAN, K_FINAL, K_COUNT, K_CYCLE_POST, K_QUAL_POST, K_KMER_FIX, K_ALLREDUCE,
       K_EMIT_BATCH_SIZES, K_EMIT_BATCH_COPY, K_REPORT_CYCLES, K_REPORT_SIZES, K_REPORT_TEXT, K_QUAL_EXC, K_QHIST_FOLD,
       K_HTML_CAPTURE, K_HTML_CYCLES, K_HTML_GROUP_HIST, K_HTML_GROUP_SCATTER, K_HTML_LENGTHS, K_HTML_VALUES, K_HTML_SUMS,
       K_HTML_SIZES, K_HTML_TEXT, K_MERGE_STATS, K_NKERNELS };
// K_CYCLE_PRE: the fused pass (both Stats blocks) without --mask/--break, the pre-filter pass with it; K_CYCLE_POST: the
// post-filter segments the fused pass did not take, or the whole --mask/--break post-filter list.  K_QUAL_EXC and
// K_QHIST_FOLD replace K_QUAL_PRE where k_scan_jit counts the quality histograms.
static const char* const kKernelNames[K_NKERNELS] = {"k_make_preseg", "k_cycle_stats(pre+post)", "k_read_qual(pre+post)",
                                                     "k_trim", "k_scan", "k_final", "k_count",
                                                     "k_cycle_stats(post residual)", "k_read_qual(post)", "k_kmer_fix",
                                                     "nccl_allreduce(stats)", "k_emit_batch(sizes)", "k_emit_batch(copy)",
                                                     "k_report(cycles)", "k_report(sizes)", "k_report(text)",
                                                     "k_read_qual(exceptions)", "k_qhist_fold",
                                                     "k_html(capture)", "k_html(cycles)", "k_html(group hist)", "k_html(group scatter)",
                                                     "k_html(lengths)", "k_html(values)", "k_html(sums)", "k_html(sizes)",
                                                     "k_html(text)", "k_merge_stats"};
// K_HTML_CYCLES: k_report_cycles + k_html_bins; K_HTML_LENGTHS: k_html_lenhist, k_html_lenprod, k_html_lensearch

// fpl_keep_read_lists: the (length, median) lists of both Stats blocks
struct FplLists {
    DevBuf<HtmlEntry> d[2];
    int64_t n[2] = {0, 0};
    bool keep = false;                  // capture on
    bool complete = true;               // every fpl_process_* call since fpl_create / fpl_reset captured
    bool merged = false;                // fpl_allreduce_stats over more than one rank since then
};

// fpl_report_html: the text and its work buffers
struct FplHtml {
    DevBuf<HtmlEntry> d_grp[2];
    DevBuf<long long> d_mat;            // grouping histograms, then their exclusive sum in place
    DevBuf<long long> d_moff;
    DevBuf<unsigned long long> d_hist;  // length histogram
    DevBuf<long long> d_lwork;          // count scan, products, product scan
    DevBuf<int> d_lstat;                // min, max, median, N50 of each block
    DevBuf<unsigned long long> d_sum;   // k_report_cycles' 6 words, then 16 base-bin counts
    DevBuf<long long> d_x;
    DevBuf<double> d_vals;
    DevBuf<double> d_sums;
    DevBuf<int64_t> d_size;
    DevBuf<int64_t> d_off;
    DevBuf<uint8_t> d_tmp;
    DevBuf<uint8_t> d_frame;
    DevBuf<uint8_t> d_text;
    std::vector<uint8_t> h_frame;
    bool built = false;
    std::string key;
    int64_t n_bytes = 0;
};

// fpl_report_json: the report text of the accumulators as they were when it was built, kept in HBM until a call changes them
struct FplReport {
    DevBuf<unsigned long long> d_sum;   // k_report_cycles: total_cycles, bases, G+C of each block
    DevBuf<int64_t> d_size;             // bytes of every value
    DevBuf<int64_t> d_off;              // their exclusive sum
    DevBuf<uint8_t> d_tmp;
    DevBuf<uint8_t> d_frame;            // piece tables + the host-built frame
    DevBuf<uint8_t> d_text;
    std::vector<uint8_t> h_frame;
    bool built = false;
    std::string key;                                // version, command and is_rna of the built text
    int64_t n_bytes = 0;
};

// the context's NCCL communicator, released by ncclCommDestroy (defined where nccl() is)
struct CommRelease { void operator()(ncclComm_t m) const; };

// The owners of the streams come first: they go last, after everything that work queued on them uses.  fpl_destroy
// synchronises both streams before the context goes.
struct fpl_ctx {
    int device = 0;
    Stream stream;
    // fpl_process_host: the upload runs on its own stream, piece by piece, and the kernels of a piece start as soon
    // as its bytes have arrived (copy/compute overlap inside one call)
    Stream copy_stream;
    DevParams P;
    ScanPlan plan;
    FplJitKernel jit;   // specialised scan kernel (NVRTC), fn == nullptr if not used
    FplIngest ingest;   // device-side FASTQ parsing state
    FplExt ext;         // --mask / --break state (variable number of output reads)
    FplEmit emit;       // device-side output text of the last fpl_process_fastq_host chunk (fpl_emit_fastq_host)
    bool emit_valid = false;            // the last call was a successful fpl_process_fastq_host: chunk + records + results in HBM
    int64_t emit_n = 0;
    FplBatchEmit bemit;                 // fpl_emit_batch_device: sizes of the output batches of the last fpl_process_* call
    bool bemit_valid = false;           // the last fpl_process_* call succeeded: bsrc + last_results + ext lists describe it
    DevBatch bsrc = {};                 // the batch that call processed (the context's staging or the caller's buffers)
    int64_t last_bytes = 0;
    bool slots16 = false;               // this batch's read offsets are multiples of 16 (checked: host and device batches)
    int n_adapters = 0;
    std::vector<std::string> adapter_str;   // fpl_adapters order (the report's adapter names and counted substrings)
    FplReport rep;
    FplLists lists;
    FplHtml html;
    DevBuf<uint8_t> d_adapters;
    DevBuf<int> d_alen;
    DevBuf<uint4> d_peq;
    DevBuf<uint32_t> d_peq16;
    DevBuf<uint32_t> d_acode;
    DevBuf<unsigned long long> d_peq_long;
    DevBuf<int> d_pf_order;
    // accumulators
    int64_t C = 0;
    DevBuf<unsigned long long> d_stats[2];
    DevBuf<unsigned long long> d_counters;
    int64_t counter_words = 0;
    // per-read work buffers
    int64_t cap_reads = 0;
    DevBuf<ReadState> d_state;
    DevBuf<fpl_read_result> d_results;
    CycleWs cycle_ws;
    DevBuf<StatSeg> d_preseg;
    DevBuf<StatSeg> d_postseg;
    // k_scan_jit with the quality histograms (jit.qhist): their striped sums, and k_final's list of the reads whose one
    // passing segment is not their window (k_read_qual_exc)
    DevBuf<unsigned long long> d_qstripes;
    DevBuf<int32_t> d_exc;
    DevBuf<int> d_nexc;
    int64_t last_n = 0;
    fpl_read_result* last_results = nullptr;  // where the last call's records live (device)
    // staging for host batches
    DevBuf<uint8_t> d_seq;
    DevBuf<uint8_t> d_qual;
    DevBuf<int64_t> d_offsets;
    DevBuf<int32_t> d_lens;
    std::vector<int32_t> h_lens;
    // tiling + measurement
    int64_t tile_bases = 0;
    DevBuf<int> d_minmax;               // fpl_process_device: min / max read length of the batch
    PinnedHost<int> h_minmax;
    std::vector<Event> piece_events;
    int64_t piece_bytes = 16ll << 20;
    bool timing = false;
    float kernel_ms[K_NKERNELS];
    int64_t kernel_n[K_NKERNELS];
    int64_t launches = 0;
    // multi-GPU merge (fpl_comm_init / fpl_allreduce_stats): one NCCL communicator per context
    Owned<ncclComm_t, CommRelease> comm;
    int comm_rank = 0, comm_size = 1;
    int64_t used_cycles = 0;            // longest read accumulated since the last fpl_reset
    int64_t reduced_rows = 0;           // widest fpl_allreduce_stats since then: other ranks' reads may fill rows past used_cycles
    DevBuf<long long> d_agree;          // device word for the all-reduce(max) of the cycle count
    PinnedHost<long long> h_agree;
    // fpl_merge_stats: the sources' table (k_merge_stats) and the event that orders the streams
    DevBuf<MergeSrc> d_merge;
    Event merge_ev;
    DevBuf<unsigned long long> d_state_stage;   // fpl_state_merge: the images' Stats and counter sections

    // timing (Timed): the recorded start / end pairs not yet collected, and the collected events for reuse
    struct Ev { int k; Event a, b; };
    std::vector<Ev> events;
    std::vector<Event> pool;
};

static int ensure_reads(fpl_ctx* c, int64_t n) {
    if (n <= c->cap_reads) return 0;
    int64_t cap = c->cap_reads ? c->cap_reads : 1024;
    while (cap < n) cap *= 2;
    c->cap_reads = 0;
    c->d_state.reset(); c->d_results.reset(); c->d_preseg.reset(); c->d_postseg.reset(); c->d_exc.reset();
    CK(c->d_state.grow_exact(cap));
    CK(c->d_results.grow_exact(cap));
    CK(c->d_preseg.grow_exact(cap));
    CK(c->d_postseg.grow_exact(2 * cap));
    if (c->jit.qhist) CK(c->d_exc.grow_exact(cap));
    c->cap_reads = cap;
    return 0;
}

// Both blocks re-laid out at capacity nc, or (on any failure) the context as it was: the new blocks are allocated and filled
// before they replace the old ones.
static int reserve_cycles(fpl_ctx* c, int64_t need) {
    if (need <= c->C) return 0;
    c->rep.built = false; c->html.built = false;
    int64_t nc = c->C ? c->C : 1024;
    while (nc < need) nc *= 2;
    DevBuf<unsigned long long> nb[2];
    for (int w = 0; w < 2; w++) CK(nb[w].grow_exact(FPL_STATS_WORDS(nc)));
    for (int w = 0; w < 2; w++) {
        CK(cudaMemsetAsync(nb[w], 0, sizeof(unsigned long long) * FPL_STATS_WORDS(nc), c->stream));
        if (c->C) {
            // rows b*C + c move to b*nc + c; the tail moves to 16*nc
            CK(cudaMemcpy2DAsync(nb[w], sizeof(unsigned long long) * nc, c->d_stats[w], sizeof(unsigned long long) * c->C,
                                 sizeof(unsigned long long) * c->C, 16, cudaMemcpyDeviceToDevice, c->stream));
            CK(cudaMemcpyAsync(nb[w] + 16 * nc, c->d_stats[w] + 16 * c->C, sizeof(unsigned long long) * FPL_STATS_TAIL,
                               cudaMemcpyDeviceToDevice, c->stream));
        }
    }
    if (c->C) CK(cudaStreamSynchronize(c->stream));
    for (int w = 0; w < 2; w++) c->d_stats[w].swap(nb[w]);      // nb frees the old blocks
    c->C = nc;
    return 0;
}

// list w holds at least `need` entries, its entries kept
static int grow_list(fpl_ctx* c, int w, int64_t need) {
    FplLists& L = c->lists;
    CK(L.d[w].grow_keep(need, L.n[w], c->stream, (int64_t)sizeof(HtmlEntry) << 16));
    return 0;
}

// the staging batch of host input: n_bytes in each of seq and qual, n_reads offsets and lengths, each at exactly that size when
// it grows
static int reserve_staging(fpl_ctx* c, int64_t n_bytes, int64_t n_reads) {
    CK(c->d_seq.grow_exact(n_bytes));
    CK(c->d_qual.grow_exact(n_bytes));
    CK(c->d_offsets.grow_exact(n_reads));
    CK(c->d_lens.grow_exact(n_reads));
    return 0;
}

// a timing event from the pool, or a new one; empty when none can be created
static Event get_event(fpl_ctx* c) {
    Event e;
    if (c->pool.empty()) { create_event(e, true); return e; }
    e = std::move(c->pool.back());
    c->pool.pop_back();
    return e;
}

// A launch timed when timing is on and both its events exist; without them it runs untimed.  It is counted either way.
struct Timed {
    fpl_ctx* c; int k; bool ours; Event a, b;
    Timed(fpl_ctx* c_, int k_, bool ours_ = true) : c(c_), k(k_), ours(ours_) {   // ours = false: a library kernel (NCCL), timed but not counted
        if (c->timing) { a = get_event(c); b = get_event(c); }
        if (a && b) cudaEventRecord(a, c->stream);
    }
    ~Timed() {
        if (ours) c->launches++;
        if (a && b) { cudaEventRecord(b, c->stream); c->events.push_back({k, std::move(a), std::move(b)}); }
    }
};

// Harvest the event pairs that have completed; pending ones stay queued (kernel_ms accumulates until
// fpl_set_timing() resets it).
static void collect_times(fpl_ctx* c) {
    size_t keep = 0;
    for (auto& e : c->events) {
        if (cudaEventQuery(e.b) != cudaSuccess) { c->events[keep++] = std::move(e); continue; }
        float ms = 0;
        if (cudaEventElapsedTime(&ms, e.a, e.b) == cudaSuccess) { c->kernel_ms[e.k] += ms; c->kernel_n[e.k]++; }
        c->pool.push_back(std::move(e.a)); c->pool.push_back(std::move(e.b));
    }
    c->events.resize(keep);
}

// min and max of the read lengths (fpl_process_device)
// ... and the OR of the low four bits of the slot offsets (out[2]): 0 <=> every read starts on a 16-byte boundary
__global__ void k_lens_minmax(const int32_t* __restrict__ lens, const int64_t* __restrict__ offsets, int64_t n, int* __restrict__ out) {
    int lo = INT_MAX, hi = INT_MIN;
    unsigned mis = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int v = lens[i];
        lo = min(lo, v); hi = max(hi, v);
        mis |= (unsigned)offsets[i] & 15u;
    }
    lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi); mis = __reduce_or_sync(0xffffffffu, mis);
    if ((threadIdx.x & 31) == 0) { atomicMin(&out[0], lo); atomicMax(&out[1], hi); if (mis) atomicOr(&out[2], (int)mis); }
}

// Runs every kernel over reads [0, n) of a device-resident batch whose lens are known on the host.
// cuts/arrived (optional): the batch arrives in pieces — reads [cuts[j], cuts[j+1]) are on the device once event
// arrived[j] has fired; the kernels then run piece by piece.
// h_lens may be null when the caller knows the longest read (known_max_len >= 0) and nothing below needs the individual
// lengths (no tiling, no pieces): a device-resident batch then never waits for the host to walk a million lengths.
static int run_batch(fpl_ctx* c, const DevBatch& full, const int32_t* h_lens, fpl_read_result* d_res_out, int64_t n_bytes,
                     const std::vector<int64_t>* cuts = nullptr, const Event* arrived = nullptr,
                     int64_t known_max_len = -1) {
    const int64_t n = full.n_reads;
    CK(cudaSetDevice(c->device));
    collect_times(c);
    c->emit_valid = false; c->emit.built = false;
    c->bemit_valid = false; c->bemit.built = false;
    c->rep.built = false; c->html.built = false;
    c->bsrc = full;
    c->last_n = n;
    if (ensure_reads(c, n)) return -1;
    fpl_read_result* d_res = d_res_out ? d_res_out : c->d_results;
    c->last_results = d_res;
    int64_t max_len = 0;
    if (h_lens) {
        for (int64_t i = 0; i < n; i++) {
            if (h_lens[i] < 0) return fail("read %lld has a negative length", (long long)i);
            if (h_lens[i] > max_len) max_len = h_lens[i];
        }
    } else {
        max_len = known_max_len;
    }
    if (reserve_cycles(c, max_len > 0 ? max_len : 1)) return -1;
    if (max_len > c->used_cycles) c->used_cycles = max_len;
    // tiles of reads whose payload stays L2-resident across the kernels that revisit it
    const bool ext = c->P.opt.mask_enabled || c->P.opt.break_enabled;   // variable number of output reads: one tile
    c->ext.n_segs = 0; c->ext.n_regs = 0;
    // the scan counts the quality histograms (k_scan_jit built with them; never with --mask/--break): k_final lists the
    // exceptions, k_read_qual_exc treats them, k_count adds the per-read sums and the striped sums are folded at the end
    const bool qhist = c->jit.fn && c->jit.qhist;
    if (qhist && n > 0) CK(cudaMemsetAsync(c->d_qstripes, 0, sizeof(unsigned long long) * QH_STRIPES * 256, c->stream));
    int64_t r0 = 0;
    size_t piece = 0;
    while (r0 < n) {
        int64_t r1 = r0, bases = 0, tmax = 0;
        if (cuts) {
            if (ext) {       // one tile: wait for everything
                for (size_t j = 0; j + 1 < cuts->size(); j++) CK(cudaStreamWaitEvent(c->stream, arrived[j], 0));
                r1 = n;
            } else {
                CK(cudaStreamWaitEvent(c->stream, arrived[piece], 0));
                r1 = (*cuts)[piece + 1];
                piece++;
            }
            for (int64_t i = r0; i < r1; i++) if (h_lens[i] > tmax) tmax = h_lens[i];
        } else if (!h_lens || ext || c->tile_bases >= (1ll << 61)) {
            r1 = n; tmax = max_len;      // one tile
        } else {
            while (r1 < n && (r1 == r0 || ext || bases + h_lens[r1] <= c->tile_bases)) {
                bases += h_lens[r1];
                if (h_lens[r1] > tmax) tmax = h_lens[r1];
                r1++;
            }
        }
        DevBatch b = full;
        b.offsets = full.offsets + r0; b.lens = full.lens + r0; b.n_reads = r1 - r0;
        ReadState* st = c->d_state + r0;
        fpl_read_result* res = d_res + r0;
        StatSeg* pre = c->d_preseg + r0;
        StatSeg* post = c->d_postseg + 2 * r0;
        cudaStream_t s = c->stream;
        { Timed t(c, K_PRESEG); launch_make_preseg(b, pre, s); }
        { Timed t(c, K_TRIM); launch_trim(c->P, b, st, res, c->d_counters, s);
          if (c->P.opt.adapter_enabled && c->n_adapters > 2) c->launches++; }   // + k_trim_fasta
        if (ext) {
            Timed t(c, K_CYCLE_PRE);
            if (launch_cycle_stats(&c->cycle_ws, full.seq, full.qual, pre, b.n_reads, tmax, c->d_stats[0], c->C, true, nullptr,
                                   c->slots16, nullptr, nullptr, nullptr, s))
                return fail("out of device memory (cycle stats workspace)");
            c->launches += 2;   // + k_cs_keys and k_cs_gather around the (library) radix sort
        }
        {
            Timed t(c, K_SCAN);
            if (c->jit.fn) { if (fpl_jit_launch_scan(&c->jit, b, st, s)) return fail("launching k_scan_jit failed"); }
            else if (c->plan.fast) launch_scan_fast(c->P, c->plan, b, st, s);
            else launch_scan(c->P, b, st, s);
        }
        int32_t* exc = qhist ? c->d_exc + r0 : nullptr;
        if (qhist) CK(cudaMemsetAsync(c->d_nexc, 0, sizeof(int), s));
        { Timed t(c, K_FINAL); launch_final(c->P, b, st, res, post, exc, c->d_nexc, s); }
        if (!ext) {
            if (qhist) { Timed t(c, K_QUAL_EXC); launch_read_qual_exc(b, st, exc, c->d_nexc, c->d_stats[0], c->d_stats[1], c->C, res, s); }
            { Timed t(c, K_COUNT);
              launch_count(res, b.n_reads, c->d_counters, true, b.lens, qhist ? c->d_stats[0].get() : nullptr, c->d_stats[1], c->C, s); }
            // one pass over the reads counts the pre-filter Stats and, for the read's slot-0 passing segment, the
            // post-filter per-cycle counters; the residual pass counts the passing segments it did not take
            { Timed t(c, K_CYCLE_PRE);
              if (launch_cycle_stats(&c->cycle_ws, full.seq, full.qual, pre, b.n_reads, tmax, c->d_stats[0], c->C, true,
                                     c->d_stats[1] + 16 * c->C + FPL_STATS_KMER, c->slots16, post, c->d_stats[1], nullptr, s))
                  return fail("out of device memory (cycle stats workspace)");
              c->launches += 2; }   // + k_cs_keys and k_cs_gather around the (library) radix sort
            { Timed t(c, K_CYCLE_POST);
              if (launch_cycle_stats(&c->cycle_ws, full.seq, full.qual, post, 2 * b.n_reads, tmax, c->d_stats[1], c->C, false, nullptr,
                                     false, nullptr, nullptr, pre, s))
                  return fail("out of device memory (cycle stats workspace)");
              c->launches += 2; }   // + k_cs_keys and k_cs_gather around the (library) radix sort
            { Timed t(c, K_KMER_FIX); launch_kmer_fix(b, res, c->d_stats[1] + 16 * c->C + FPL_STATS_KMER, s); }
            if (!qhist) { Timed t(c, K_QUAL_PRE); launch_read_qual(b, c->d_stats[0], c->d_stats[1], c->C, res, false, s); }
        } else {
            // --mask / --break: k_final left the output reads of the adapter stage in the records; fpl_ext_run breaks /
            // masks / filters them (variable count) and the post-filter Stats run over its segment list
            char xerr[256] = "";
            const uint8_t* fseq = full.seq;
            { Timed t(c, K_QUAL_PRE); launch_read_qual(b, c->d_stats[0], c->d_stats[1], c->C, res, true, s); }
            { Timed t(c, K_COUNT); launch_count(res, b.n_reads, c->d_counters, false, nullptr, nullptr, nullptr, 0, s); }
            if (fpl_ext_run(&c->ext, c->P, b, n_bytes, res, c->d_counters, c->d_stats[1], c->C, &fseq, s, xerr, sizeof(xerr)))
                return fail("--mask/--break stage: %s", xerr);
            { Timed t(c, K_CYCLE_POST);
              if (launch_cycle_stats(&c->cycle_ws, fseq, full.qual, c->ext.d_stat, c->ext.n_segs, tmax, c->d_stats[1], c->C, true, nullptr, false,
                                     nullptr, nullptr, nullptr, s))
                  return fail("out of device memory (cycle stats workspace)");
          c->launches += 2; }   // + k_cs_keys and k_cs_gather around the (library) radix sort
        }
        r0 = r1;
    }
    if (qhist && n > 0) { Timed t(c, K_QHIST_FOLD); launch_qhist_fold(c->d_qstripes, QH_STRIPES, c->d_stats[0], c->d_stats[1], c->C, c->stream); }
    if (c->lists.keep) {
        // after every kernel that writes a median: the call's entries behind the lists' ends.  Without --mask/--break the
        // post-filter list takes two slots per read (their segments), with them one per output read (ext.n_segs)
        FplLists& L = c->lists;
        const int64_t n_post = ext ? c->ext.n_segs : 2 * n;
        if (grow_list(c, 0, L.n[0] + n) || grow_list(c, 1, L.n[1] + n_post)) return -1;
        if (n || n_post) {
            Timed t(c, K_HTML_CAPTURE);
            launch_html_capture(d_res, full.lens, n, ext ? c->ext.d_segs.get() : nullptr, ext ? n_post : 0, L.d[0] + L.n[0], L.d[1] + L.n[1],
                                c->stream);
        }
        L.n[0] += n; L.n[1] += n_post;
        c->html.built = false;
    } else {
        c->lists.complete = false;
    }
    CK(cudaGetLastError());
    return 0;
}

extern "C" {

const char* fpl_last_error(void) { return g_err; }
int fpl_abi_version(void) { return FPL_ABI_VERSION; }

int fpl_create(const fpl_options* opt, const fpl_adapters* ad, fpl_ctx** out) {
    g_err[0] = 0;
    if (!opt || !ad || !out) return fail("fpl_create: null argument");
    if (opt->struct_size != (int32_t)sizeof(fpl_options))
        return fail("fpl_create: fpl_options.struct_size %d != %d (ABI mismatch)", opt->struct_size, (int)sizeof(fpl_options));
    if (opt->ed_max < 0 || opt->ed_max > 1.0) return fail("fpl_create: ed_max must be within 0..1");
    if (opt->trim_front < 0 || opt->trim_tail < 0) return fail("fpl_create: trim_front/trim_tail must be >= 0");
    if ((opt->cut_front_enabled && (opt->cut_front_window < 1 || opt->cut_front_window > FPL_MAX_WINDOW)) ||
        (opt->cut_tail_enabled && (opt->cut_tail_window < 1 || opt->cut_tail_window > FPL_MAX_WINDOW)))
        return fail("fpl_create: cut window size must be within 1..%d", FPL_MAX_WINDOW);
    const int n = 2 + (ad->n_fasta > 0 ? ad->n_fasta : 0);
    if (n > FPL_MAX_ADAPTERS) return fail("fpl_create: %d adapters exceed FPL_MAX_ADAPTERS=%d", n, FPL_MAX_ADAPTERS);
    // FPL_TIMING=1: where the start-up time goes (stderr)
    const bool tlog = getenv("FPL_TIMING") != nullptr;
    auto now = [] { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; };
    double t_last = now();
    auto stamp = [&](const char* what) {
        if (!tlog) return;
        const double t = now();
        fprintf(stderr, "[libfplgpu] fpl_create: %-28s %7.3f s\n", what, t - t_last);
        t_last = t;
    };
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail("fpl_create: no usable CUDA device (%s); libfplgpu has no CPU fallback", cudaGetErrorString(e));
    if (opt->device < 0 || opt->device >= ndev) return fail("fpl_create: device %d out of range (%d devices)", opt->device, ndev);
    CK(cudaSetDevice(opt->device));
    CK(cudaDeviceSynchronize());        // the first call that needs the device context creates it
    stamp("driver + device context");
    std::unique_ptr<fpl_ctx> c(new fpl_ctx());     // released to the caller on success, freed on every failure
    c->device = opt->device;
    c->n_adapters = n;
    // host tables
    std::vector<uint8_t> h_ad((size_t)n * FPL_MAX_ADAPTER_LEN, 0);
    std::vector<int> h_alen(n, 0);
    std::vector<uint4> h_peq((size_t)n * 256, make_uint4(0, 0, 0, 0));
    std::vector<uint32_t> h_peq16((size_t)n * 512, 0);   // [adapter][prefix | suffix][byte]
    std::vector<uint32_t> h_acode((size_t)n * 4, 0);
    size_t maxlen = 0;
    for (int k = 0; k < n; k++) {
        const char* s = k == 0 ? ad->start : k == 1 ? ad->end : ad->fasta[k - 2];
        if (s && strlen(s) > maxlen) maxlen = strlen(s);
    }
    // adapters longer than 128 bp: multi-word match masks for myers_long (the 128-bit table below stays as it is)
    const int peq_words = maxlen > 128 ? (int)((maxlen + 63) / 64) + 1 : 0;
    std::vector<unsigned long long> h_peq_long((size_t)n * 256 * peq_words, 0ull);
    for (int k = 0; k < n; k++) {
        const char* s = k == 0 ? ad->start : k == 1 ? ad->end : ad->fasta[k - 2];
        if (!s) s = "";
        size_t len = strlen(s);
        if (len > FPL_MAX_ADAPTER_LEN)
            return fail("fpl_create: adapter %d is %zu bp, longer than FPL_MAX_ADAPTER_LEN=%d", k, len, FPL_MAX_ADAPTER_LEN);
        h_alen[k] = (int)len;
        c->adapter_str.push_back(s);
        memcpy(&h_ad[(size_t)k * FPL_MAX_ADAPTER_LEN], s, len);
        const int plen = (int)len < FPL_PATTERN_LEN ? (int)len : FPL_PATTERN_LEN;
        {   // packed 2-bit form for the windowed Hamming search (k_trim), only for ACGT-only adapters of <= 32 bp
            bool ok = len >= 1 && len <= 32;
            unsigned long long code = 0, mask = 0;
            for (size_t j = 0; j < len && ok; j++) {
                const char ch = s[j];
                if (ch != 'A' && ch != 'C' && ch != 'G' && ch != 'T') ok = false;
                code |= (unsigned long long)((ch >> 1) & 3) << (2 * j);
                mask |= 1ull << (2 * j);
            }
            if (ok) {
                h_acode[(size_t)k * 4 + 0] = (uint32_t)code; h_acode[(size_t)k * 4 + 1] = (uint32_t)(code >> 32);
                h_acode[(size_t)k * 4 + 2] = (uint32_t)mask; h_acode[(size_t)k * 4 + 3] = (uint32_t)(mask >> 32);
            }
        }
        for (size_t j = 0; j < len; j++) {
            uint8_t ch = (uint8_t)s[j];
            uint32_t* w = reinterpret_cast<uint32_t*>(&h_peq[(size_t)k * 256 + ch]);
            if (j < 128) w[j >> 5] |= 1u << (j & 31);
            if (peq_words) h_peq_long[((size_t)k * 256 + ch) * peq_words + (j >> 6)] |= 1ull << (j & 63);
            if ((int)j < plen) h_peq16[(size_t)k * 512 + ch] |= 1u << j;                            // first plen chars
            if ((int)j >= (int)len - plen) h_peq16[(size_t)k * 512 + 256 + ch] |= 1u << (j - (len - plen));  // last plen chars
        }
    }
    memset(&c->P, 0, sizeof(c->P));
    c->P.opt = *opt;
    c->P.one = 1u;
    {
        auto cls = [](int a) { return a <= 32 ? 0 : a <= 64 ? 1 : 2; };
        c->P.small_adapters = std::max(cls(h_alen[0]), cls(h_alen[1]));
        int fc = 0;
        for (int k = 2; k < n; k++) fc = std::max(fc, cls(h_alen[k]));
        c->P.fasta_class = fc;
    }
    c->P.n_adapters = n;
    // plan for the bit-sliced middle-adapter scan (k_scan_fast); anything it cannot express uses k_scan
    memset(&c->plan, 0, sizeof(c->plan));
    {
        bool fast = getenv("FPL_FORCE_GENERIC_SCAN") == nullptr;
        int maxa = 1;
        for (int k = 0; k < 2 && fast && opt->adapter_enabled; k++) {
            const char* s = k == 0 ? ad->start : ad->end;
            const int len = h_alen[k];
            if (len < 1 || len > 128) { fast = false; break; }   // bit-sliced counters: up to 8 planes, 4 halo words
            if (len > maxa) maxa = len;
            for (int i = 0; i < len; i++) {
                const char ch = s[i];
                if (ch != 'A' && ch != 'C' && ch != 'G' && ch != 'T') { fast = false; break; }
                c->plan.hm[k][i] = (ch & 2) ? 0xFFFFFFFFu : 0u;   // code bit HI = byte bit 1
                c->plan.lm[k][i] = (ch & 4) ? 0xFFFFFFFFu : 0u;   // code bit LO = byte bit 2
                c->plan.vm[k][i] = 0xFFFFFFFFu;
            }
        }
        c->plan.fast = fast ? 1 : 0;
        c->plan.npl = maxa <= 31 ? 5 : maxa <= 63 ? 6 : maxa <= 127 ? 7 : 8;
        c->plan.halo_words = ((maxa - 1) >> 5) + 1;
    }
    for (int i = 0; i <= FPL_MAX_ADAPTER_LEN; i++) c->P.thr[i] = (short)(int)round(opt->ed_max * i);  // src/adaptertrimmer.cpp:73
    CK(create_stream(c->stream));
    CK(c->d_adapters.grow_exact((int64_t)h_ad.size()));
    CK(c->d_alen.grow_exact(n));
    CK(c->d_peq.grow_exact((int64_t)h_peq.size()));
    CK(c->d_peq16.grow_exact((int64_t)h_peq16.size()));
    CK(c->d_acode.grow_exact((int64_t)h_acode.size()));
    CK(cudaMemcpy(c->d_acode, h_acode.data(), sizeof(uint32_t) * h_acode.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_adapters, h_ad.data(), h_ad.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_alen, h_alen.data(), sizeof(int) * n, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_peq, h_peq.data(), sizeof(uint4) * h_peq.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_peq16, h_peq16.data(), sizeof(uint32_t) * h_peq16.size(), cudaMemcpyHostToDevice));
    if (peq_words) {
        CK(c->d_peq_long.grow_exact((int64_t)h_peq_long.size()));
        CK(cudaMemcpy(c->d_peq_long, h_peq_long.data(), sizeof(unsigned long long) * h_peq_long.size(), cudaMemcpyHostToDevice));
    }
    c->P.peq_long = c->d_peq_long; c->P.peq_words = peq_words;
    if (n > 2) {
        // k_trim's many-adapter pre-filter works on 32 (adapter, side) pairs at a time and uses 64-bit bit-vectors for a
        // round as soon as one of its adapters is longer than 32 bp: group the adapters by width class
        std::vector<int> order;
        for (int cls = 0; cls < 3; cls++)
            for (int k = 2; k < n; k++) {
                const int kc = h_alen[k] <= 32 ? 0 : h_alen[k] <= 64 ? 1 : 2;
                if (kc == cls) order.push_back(k);
            }
        CK(c->d_pf_order.grow_exact((int64_t)order.size()));
        CK(cudaMemcpy(c->d_pf_order, order.data(), sizeof(int) * order.size(), cudaMemcpyHostToDevice));
    }
    c->P.pf_order = c->d_pf_order;
    c->P.adapters = c->d_adapters; c->P.alen = c->d_alen; c->P.peq = c->d_peq; c->P.peq16 = c->d_peq16; c->P.acode = c->d_acode;
    c->counter_words = FPL_COUNTER_WORDS(n);
    CK(c->d_counters.grow_exact(c->counter_words));
    CK(cudaMemset(c->d_counters, 0, sizeof(unsigned long long) * c->counter_words));
    stamp("tables");
    // specialise the scan kernel on the adapters (NVRTC); FPL_NO_JIT=1 keeps the precompiled k_scan_fast
    if (c->plan.fast && getenv("FPL_NO_JIT") == nullptr) {
        char jerr[512] = "";
        const bool doCounts = opt->qual_filter_enabled || opt->length_filter_enabled;
        // the quality histograms ride on the scan where it loads the quality bytes anyway (the quality or the length
        // filter) and without --mask/--break (whose post-filter reads are not the windows).  With -Q -L the scan would
        // load them for the histograms alone: measured on an H100 (profiles/README.md), that loses on 1 kb reads
        const bool doQhist = doCounts && !(opt->mask_enabled || opt->break_enabled);
        if (fpl_jit_build_scan(c->device, ad->start ? ad->start : "", ad->end ? ad->end : "", opt->adapter_enabled != 0,
                               doCounts, opt->complexity_enabled != 0, doQhist, opt->qualified_qual, &c->jit, jerr, sizeof(jerr))) {
            fprintf(stderr, "libfplgpu: run-time specialisation unavailable (%s); using the precompiled k_scan_fast\n", jerr);
            c->jit.fn = nullptr;
            c->jit.qhist = false;
        }
    }
    if (c->jit.qhist) {
        CK(c->d_qstripes.grow_exact(QH_STRIPES * 256));
        CK(c->d_nexc.grow_exact(1));
        c->P.qstripes = c->d_qstripes;
    }
    stamp("scan kernel specialisation");
    const char* tb = getenv("FPL_TILE_MBASES");
    // 0 (default) = no tiling: every kernel streams the whole batch from HBM (L2-sized tiles make launches too small
    // to fill the GPU)
    c->tile_bases = (tb && atoll(tb) > 0) ? atoll(tb) * 1000000ll : (1ll << 62);
    // fpl_process_host uploads in pieces of this many MiB per buffer and overlaps them with the kernels (0 = one piece)
    const char* pm = getenv("FPL_PIECE_MB");
    if (pm) c->piece_bytes = atoll(pm) > 0 ? atoll(pm) << 20 : 0;
    for (int k = 0; k < K_NKERNELS; k++) { c->kernel_ms[k] = 0; c->kernel_n[k] = 0; }
    if (reserve_cycles(c.get(), 1024)) return -1;
    CK(cudaStreamSynchronize(c->stream));
    stamp("accumulators");
    *out = c.release();
    return 0;
}

void fpl_destroy(fpl_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    collect_times(c);
    delete c;                           // every resource goes with its owner
}

int fpl_process_device(fpl_ctx* c, const fpl_batch* b, fpl_read_result* results_dev) {
    g_err[0] = 0;
    if (!c || !b) return fail("fpl_process_device: null argument");
    c->bemit_valid = false;
    CK(cudaSetDevice(c->device));
    const int64_t n = b->n_reads;
    if (n < 0) return fail("fpl_process_device: negative n_reads");
    DevBatch d = {b->seq, b->qual, b->offsets, b->lens, n};
    // the extremes of the lengths (Stats capacity, grid sizes) and the alignment of the offsets are all the host needs
    // to know: reduce them on the side stream, which does not wait for the kernels of the previous batch still running
    // on the compute stream
    if (!c->copy_stream) CK(create_stream(c->copy_stream));
    CK(c->d_minmax.grow_exact(4));
    if (!c->h_minmax) CK(create_pinned(c->h_minmax, 4));
    c->h_minmax[0] = 0; c->h_minmax[1] = 0; c->h_minmax[2] = 0;
    if (n) {
        const int init[3] = {INT_MAX, INT_MIN, 0};
        CK(cudaMemcpyAsync(c->d_minmax, init, sizeof(init), cudaMemcpyHostToDevice, c->copy_stream));
        const unsigned blocks = (unsigned)((n + 1023) / 1024 < 1184 ? (n + 1023) / 1024 : 1184);
        k_lens_minmax<<<blocks, 256, 0, c->copy_stream>>>(b->lens, b->offsets, n, c->d_minmax);
        CK(cudaMemcpyAsync(c->h_minmax, c->d_minmax, 3 * sizeof(int), cudaMemcpyDeviceToHost, c->copy_stream));
        CK(cudaStreamSynchronize(c->copy_stream));
        if (c->h_minmax[0] < 0) return fail("fpl_process_device: a read has a negative length");
        if (c->h_minmax[2]) return fail("fpl_process_device: a read offset is not a multiple of 16 (see fpl_batch)");
    }
    c->slots16 = true;
    if (c->tile_bases < (1ll << 61)) {       // read tiling was asked for: the tile boundaries need every length
        c->h_lens.resize((size_t)n);
        if (n) {
            CK(cudaMemcpyAsync(c->h_lens.data(), b->lens, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
        }
        if (run_batch(c, d, c->h_lens.data(), results_dev, b->n_bytes)) return -1;
    } else if (run_batch(c, d, nullptr, results_dev, b->n_bytes, nullptr, nullptr, n ? c->h_minmax[1] : 0)) {
        return -1;
    }
    c->bemit_valid = true;
    return 0;
}

void* fpl_stream(fpl_ctx* c) { return c ? (void*)c->stream : nullptr; }

int fpl_sync(fpl_ctx* c) {
    if (!c) return fail("fpl_sync: null context");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    return 0;
}

int fpl_process_host(fpl_ctx* c, const fpl_batch* b, fpl_read_result* results) {
    g_err[0] = 0;
    if (!c || !b) return fail("fpl_process_host: null argument");
    c->bemit_valid = false;
    CK(cudaSetDevice(c->device));
    const int64_t n = b->n_reads;
    if (n < 0 || b->n_bytes < 0) return fail("fpl_process_host: negative size");
    if (n > 0 && !results) return fail("fpl_process_host: results is null");
    // validate the slot layout on the host (cheap, O(reads))
    bool monotonic = true;
    for (int64_t i = 0; i < n; i++) {
        const int64_t o = b->offsets[i];
        if (i > 0 && o < b->offsets[i - 1] + b->lens[i - 1]) monotonic = false;
        if (o < 0 || (o & 15) || b->lens[i] < 0 || o + b->lens[i] > b->n_bytes)
            return fail("fpl_process_host: read %lld has a bad slot (offset %lld, len %d, n_bytes %lld; offsets must be multiples of 16)",
                        (long long)i, (long long)o, b->lens[i], (long long)b->n_bytes);
    }
    const int64_t need = FPL_BATCH_BYTES(b->n_bytes);  // the tail the kernels' whole-vector reads may touch
    if (reserve_staging(c, need, n)) return -1;
    // pieces of about piece_bytes, cut at read boundaries (slots in increasing order; otherwise one piece)
    std::vector<int64_t> cuts(1, 0);
    if (monotonic && c->piece_bytes > 0) {
        int64_t start = 0;
        for (int64_t i = 1; i < n; i++)
            if (b->offsets[i] - start >= c->piece_bytes) { cuts.push_back(i); start = b->offsets[i]; }
    }
    cuts.push_back(n);
    const size_t np = cuts.size() - 1;
    if (!c->copy_stream) CK(create_stream(c->copy_stream));
    while (c->piece_events.size() < np) {
        Event e;
        CK(create_event(e, false));
        c->piece_events.push_back(std::move(e));
    }
    // every call ends with a synchronize of the compute stream, so the device buffers are free to overwrite here
    cudaStream_t cs = c->copy_stream;
    if (n) {
        CK(cudaMemcpyAsync(c->d_offsets, b->offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, cs));
        CK(cudaMemcpyAsync(c->d_lens, b->lens, sizeof(int32_t) * n, cudaMemcpyHostToDevice, cs));
    }
    for (size_t j = 0; j < np; j++) {
        const int64_t lo = j == 0 ? 0 : b->offsets[cuts[j]];
        const int64_t hi = j + 1 == np ? b->n_bytes : b->offsets[cuts[j + 1]];
        if (hi > lo) {
            CK(cudaMemcpyAsync(c->d_seq + lo, b->seq + lo, hi - lo, cudaMemcpyHostToDevice, cs));
            CK(cudaMemcpyAsync(c->d_qual + lo, b->qual + lo, hi - lo, cudaMemcpyHostToDevice, cs));
        }
        if (j + 1 == np) {
            CK(cudaMemsetAsync(c->d_seq + b->n_bytes, 0, need - b->n_bytes, cs));
            CK(cudaMemsetAsync(c->d_qual + b->n_bytes, 0, need - b->n_bytes, cs));
        }
        CK(cudaEventRecord(c->piece_events[j], cs));
    }
    DevBatch d = {c->d_seq, c->d_qual, c->d_offsets, c->d_lens, n};
    c->slots16 = true;          // checked above: every offset is a multiple of 16
    if (run_batch(c, d, b->lens, nullptr, b->n_bytes, &cuts, c->piece_events.data())) return -1;
    if (n) CK(cudaMemcpyAsync(results, c->d_results, sizeof(fpl_read_result) * n, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    c->bemit_valid = true;
    return 0;
}

int fpl_process_fastq_host(fpl_ctx* c, const uint8_t* text, int64_t n_bytes, int is_last, fpl_fastq_record* records,
                           fpl_read_result* results, int64_t max_records, int64_t* n_records, int64_t* consumed) {
    g_err[0] = 0;
    if (!c || !n_records || !consumed || (n_bytes > 0 && !text)) return fail("fpl_process_fastq_host: null argument");
    // the ingest below overwrites the record table and offsets the batch emit of the last call reads, even when it then
    // refuses the chunk: nothing is left to emit from until this call succeeds
    c->bemit_valid = false; c->bemit.built = false;
    if (n_bytes < 0 || n_bytes >= (1ll << 40)) return fail("fpl_process_fastq_host: bad chunk size");
    CK(cudaSetDevice(c->device));
    char err[256] = "";
    int64_t nrec = 0;
    int rc = fpl_ingest_index(&c->ingest, text, n_bytes, is_last, c->stream, &nrec, consumed, err, sizeof(err));
    if (rc < 0) return fail("fpl_process_fastq_host: %s", err);
    if (rc > 0) return 1;
    *n_records = nrec;
    c->emit_valid = false; c->emit.built = false;
    if (nrec == 0) {
        c->emit_valid = true; c->emit_n = 0;
        c->bsrc = DevBatch{}; c->bemit_valid = true;
        return 0;
    }
    if (nrec > max_records) return 1;
    if (!records || !results) return fail("fpl_process_fastq_host: records/results is null");
    FplIngest& g = c->ingest;
    const int64_t need = FPL_BATCH_BYTES(g.packed_bytes);
    if (reserve_staging(c, need, 0)) return -1;
    // slot padding is never interpreted, but keep it defined for whole-vector reads past a read's end
    CK(cudaMemsetAsync(c->d_seq, 0, need, c->stream));
    CK(cudaMemsetAsync(c->d_qual, 0, need, c->stream));
    if (fpl_ingest_pack(&g, nrec, c->d_seq, c->d_qual, c->stream, err, sizeof(err))) return fail("fpl_process_fastq_host: %s", err);
    c->h_lens.resize((size_t)nrec);
    CK(cudaMemcpyAsync(c->h_lens.data(), g.d_lens, sizeof(int32_t) * nrec, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(records, g.d_rec, sizeof(fpl_fastq_record) * nrec, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    DevBatch d = {c->d_seq, c->d_qual, g.d_offsets, g.d_lens, nrec};
    c->slots16 = false;         // the device packer's slots are aligned, but nothing here depends on it
    if (run_batch(c, d, c->h_lens.data(), nullptr, g.packed_bytes)) return -1;
    CK(cudaMemcpyAsync(results, c->d_results, sizeof(fpl_read_result) * nrec, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    c->emit_valid = true; c->emit_n = nrec;
    c->bemit_valid = true;
    return 0;
}

int fpl_emit_fastq_host(fpl_ctx* c, int want_failed, uint8_t* out, int64_t out_cap, int64_t* out_bytes, uint8_t* failed,
                        int64_t failed_cap, int64_t* failed_bytes) {
    g_err[0] = 0;
    if (!c || !out_bytes || !failed_bytes) return fail("fpl_emit_fastq_host: null argument");
    *out_bytes = *failed_bytes = 0;
    if (!c->emit_valid)
        return fail("fpl_emit_fastq_host: the last call on this context was not a successful fpl_process_fastq_host");
    CK(cudaSetDevice(c->device));
    FplEmit& e = c->emit;
    if (!e.built || e.with_failed != (want_failed != 0)) {
        const bool ext = c->P.opt.mask_enabled || c->P.opt.break_enabled;
        EmitSource src = {};
        src.text = c->ingest.d_text; src.rec = c->ingest.d_rec; src.res = c->last_results; src.n_reads = c->emit_n;
        src.segs = ext ? c->ext.d_segs.get() : nullptr;
        src.seg_off = ext ? c->ext.d_off.get() : nullptr;
        src.mseq = (c->P.opt.mask_enabled && c->ext.n_segs > 0) ? c->ext.d_mseq.get() : nullptr;   // fpl_ext_run made the masked copy
        src.offsets = c->ingest.d_offsets;
        char err[256] = "";
        if (fpl_emit_build(&e, src, want_failed != 0, c->stream, err, sizeof(err))) return fail("fpl_emit_fastq_host: %s", err);
        if (c->emit_n) c->launches += 2;
    }
    *out_bytes = e.out_bytes;
    *failed_bytes = e.failed_bytes;
    if (e.out_bytes > out_cap || e.failed_bytes > failed_cap) return 1;     // the text stays built: call again with room
    if ((e.out_bytes && !out) || (e.failed_bytes && !failed)) return fail("fpl_emit_fastq_host: null output buffer");
    if (e.out_bytes) CK(cudaMemcpyAsync(out, e.d_out, (size_t)e.out_bytes, cudaMemcpyDeviceToHost, c->stream));
    if (e.failed_bytes) CK(cudaMemcpyAsync(failed, e.d_failed, (size_t)e.failed_bytes, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}

// is `o` (an output with n_reads reads in n_bytes bytes) writable?  0 = yes, 1 = too small / missing buffers, -1 = misaligned
static int out_fits(const fpl_out_batch* o, int64_t n_reads, int64_t n_bytes) {
    if (n_reads == 0) return 0;
    if (!o->seq || !o->qual || !o->offsets || !o->lens || o->cap_reads < n_reads || o->cap_bytes < FPL_BATCH_BYTES(n_bytes)) return 1;
    if ((reinterpret_cast<uintptr_t>(o->seq) | reinterpret_cast<uintptr_t>(o->qual)) & 15) return -1;
    return 0;
}

int fpl_emit_batch_device(fpl_ctx* c, fpl_out_batch* out, fpl_out_batch* failed) {
    g_err[0] = 0;
    if (!c || !out) return fail("fpl_emit_batch_device: null argument");
    out->n_reads = out->n_bytes = 0;
    if (failed) failed->n_reads = failed->n_bytes = 0;
    if (!c->bemit_valid) return fail("fpl_emit_batch_device: no successful fpl_process_* call to emit from");
    CK(cudaSetDevice(c->device));
    const bool ext = c->P.opt.mask_enabled || c->P.opt.break_enabled;
    EmitSource src = {};
    src.res = c->last_results; src.n_reads = c->bsrc.n_reads;
    src.segs = ext ? c->ext.d_segs.get() : nullptr;
    src.seg_off = ext ? c->ext.d_off.get() : nullptr;
    src.mseq = (c->P.opt.mask_enabled && c->ext.n_segs > 0) ? c->ext.d_mseq.get() : nullptr;   // fpl_ext_run made the masked copy
    src.offsets = c->bsrc.offsets; src.seq = c->bsrc.seq; src.qual = c->bsrc.qual;
    FplBatchEmit& e = c->bemit;
    if (!e.built) {
        e.n_out = e.out_bytes = e.n_failed = e.failed_bytes = 0;
        if (src.n_reads) {
            char err[256] = "";
            if (fpl_emit_batch_reserve(&e, src.n_reads, err, sizeof(err))) return fail("fpl_emit_batch_device: %s", err);
            { Timed t(c, K_EMIT_BATCH_SIZES); launch_emit_batch_sizes(src, e.d_cnt, c->stream); }
            if (fpl_emit_batch_scan(&e, src.n_reads, c->stream, err, sizeof(err))) return fail("fpl_emit_batch_device: %s", err);
        }
        e.built = true;
    }
    out->n_reads = e.n_out; out->n_bytes = e.out_bytes;
    if (failed) { failed->n_reads = e.n_failed; failed->n_bytes = e.failed_bytes; }
    const int fo = out_fits(out, e.n_out, e.out_bytes), ff = failed ? out_fits(failed, e.n_failed, e.failed_bytes) : 0;
    if (fo < 0 || ff < 0) return fail("fpl_emit_batch_device: seq and qual must be 16-byte aligned");
    if (fo || ff) return 1;                 // the sizes stay built: call again with room
    const bool do_out = e.n_out > 0, do_failed = failed && e.n_failed > 0;
    if (!do_out && !do_failed) return 0;
    EmitBatchOut o = {}, f = {};
    if (do_out) o = EmitBatchOut{out->seq, out->qual, out->offsets, out->lens, out->segs};
    if (do_failed) f = EmitBatchOut{failed->seq, failed->qual, failed->offsets, failed->lens, failed->segs};
    // the tail pads; the slots (padding included) are the kernel's
    if (do_out) {
        CK(cudaMemsetAsync(out->seq + e.out_bytes, 0, FPL_TAIL_PAD, c->stream));
        CK(cudaMemsetAsync(out->qual + e.out_bytes, 0, FPL_TAIL_PAD, c->stream));
    }
    if (do_failed) {
        CK(cudaMemsetAsync(failed->seq + e.failed_bytes, 0, FPL_TAIL_PAD, c->stream));
        CK(cudaMemsetAsync(failed->qual + e.failed_bytes, 0, FPL_TAIL_PAD, c->stream));
    }
    { Timed t(c, K_EMIT_BATCH_COPY); launch_emit_batch_copy(src, e.d_off, o, f, c->stream); }
    CK(cudaGetLastError());
    return 0;
}

int fpl_last_segments(fpl_ctx* c, fpl_segment* out, int64_t cap, int64_t* n) {
    if (!c || !n) return fail("fpl_last_segments: null argument");
    *n = c->ext.n_segs;
    if (*n == 0) return 0;
    if (!out || cap < *n) return fail("fpl_last_segments: %lld entries, capacity %lld", (long long)*n, (long long)cap);
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(out, c->ext.d_segs, sizeof(fpl_segment) * *n, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}

int fpl_last_mask_regions(fpl_ctx* c, fpl_region* out, int64_t cap, int64_t* n) {
    if (!c || !n) return fail("fpl_last_mask_regions: null argument");
    *n = c->ext.n_regs;
    if (*n == 0) return 0;
    if (!out || cap < *n) return fail("fpl_last_mask_regions: %lld entries, capacity %lld", (long long)*n, (long long)cap);
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(out, c->ext.d_regs, sizeof(fpl_region) * *n, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}

int fpl_fetch_results(fpl_ctx* c, fpl_read_result* results, int64_t n) {
    if (!c || !results) return fail("fpl_fetch_results: null argument");
    if (n > c->last_n) return fail("fpl_fetch_results: only %lld records available", (long long)c->last_n);
    CK(cudaSetDevice(c->device));
    if (n) CK(cudaMemcpyAsync(results, c->last_results, sizeof(fpl_read_result) * n, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    return 0;
}

int64_t fpl_stats_cycles(fpl_ctx* c) { return c ? c->C : 0; }

int fpl_stats_reserve(fpl_ctx* c, int64_t cycles) {
    if (!c) return fail("fpl_stats_reserve: null context");
    CK(cudaSetDevice(c->device));
    if (reserve_cycles(c, cycles)) return -1;
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}

int fpl_stats_download(fpl_ctx* c, int which, int64_t* out, int64_t n_words) {
    if (!c || !out || which < 0 || which > 1) return fail("fpl_stats_download: bad argument");
    if (n_words != FPL_STATS_WORDS(c->C)) return fail("fpl_stats_download: n_words %lld != FPL_STATS_WORDS(%lld)", (long long)n_words, (long long)c->C);
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(out, c->d_stats[which], sizeof(int64_t) * n_words, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}

int fpl_stats_device_ptr(fpl_ctx* c, int which, void** dptr, int64_t* n_words) {
    if (!c || !dptr || !n_words || which < 0 || which > 1) return fail("fpl_stats_device_ptr: bad argument");
    *dptr = c->d_stats[which];
    *n_words = FPL_STATS_WORDS(c->C);
    return 0;
}

int64_t fpl_counter_words(fpl_ctx* c) { return c ? c->counter_words : 0; }

int fpl_counters_download(fpl_ctx* c, int64_t* out, int64_t n_words) {
    if (!c || !out) return fail("fpl_counters_download: bad argument");
    if (n_words != c->counter_words) return fail("fpl_counters_download: n_words %lld != %lld", (long long)n_words, (long long)c->counter_words);
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(out, c->d_counters, sizeof(int64_t) * n_words, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}

int fpl_counters_device_ptr(fpl_ctx* c, void** dptr, int64_t* n_words) {
    if (!c || !dptr || !n_words) return fail("fpl_counters_device_ptr: bad argument");
    *dptr = c->d_counters;
    *n_words = c->counter_words;
    return 0;
}

int fpl_reset(fpl_ctx* c) {
    if (!c) return fail("fpl_reset: null context");
    CK(cudaSetDevice(c->device));
    for (int w = 0; w < 2; w++)
        CK(cudaMemsetAsync(c->d_stats[w], 0, sizeof(unsigned long long) * FPL_STATS_WORDS(c->C), c->stream));
    CK(cudaMemsetAsync(c->d_counters, 0, sizeof(unsigned long long) * c->counter_words, c->stream));
    c->used_cycles = 0; c->reduced_rows = 0;
    c->rep.built = false; c->html.built = false;
    c->lists.n[0] = c->lists.n[1] = 0;
    c->lists.complete = true; c->lists.merged = false;
    return 0;
}

int fpl_last_kernel_times(fpl_ctx* c, const char** names, float* ms, int64_t* launches, int cap) {
    if (!c) return 0;
    collect_times(c);
    for (int k = 0; k < K_NKERNELS && k < cap; k++) {
        if (names) names[k] = kKernelNames[k];
        if (ms) ms[k] = c->kernel_ms[k];
        if (launches) launches[k] = c->kernel_n[k];
    }
    return K_NKERNELS;
}

int64_t fpl_launch_count(fpl_ctx* c) { return c ? c->launches : 0; }

int fpl_set_timing(fpl_ctx* c, int enabled) {
    if (!c) return fail("fpl_set_timing: null context");
    c->timing = enabled != 0;
    collect_times(c);
    for (int k = 0; k < K_NKERNELS; k++) { c->kernel_ms[k] = 0; c->kernel_n[k] = 0; }
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// Multi-GPU merge: the replacement of Stats::merge (src/stats.cpp:1013-1082) and FilterResult::merge
// (src/filterresult.cpp:28-61) for one process per GPU.  NCCL is resolved at run time (dlopen of libnccl.so.2: inside
// a torch process that is the copy torch already loaded), so the library stays loadable without it; the collectives
// run on the context's own stream, after the kernels that fill the blocks, with no host synchronisation.
// ------------------------------------------------------------------------------------------------------------------
namespace {
struct Nccl {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
    Nccl() {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        GetUniqueId = (decltype(GetUniqueId))dlsym(h, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(h, "ncclCommInitRank");
        CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
        AllReduce = (decltype(AllReduce))dlsym(h, "ncclAllReduce");
        GroupStart = (decltype(GroupStart))dlsym(h, "ncclGroupStart");
        GroupEnd = (decltype(GroupEnd))dlsym(h, "ncclGroupEnd");
        GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
        ok = GetUniqueId && CommInitRank && CommDestroy && AllReduce && GroupStart && GroupEnd && GetErrorString;
    }
};
Nccl& nccl() { static Nccl n; return n; }
}  // namespace

void CommRelease::operator()(ncclComm_t m) const { nccl().CommDestroy(m); }

#define CKN(call)                                                                                        \
    do {                                                                                                 \
        ncclResult_t r_ = (call);                                                                        \
        if (r_ != ncclSuccess) return fail("%s failed: %s", #call, nccl().GetErrorString(r_));          \
    } while (0)

static_assert(sizeof(ncclUniqueId) == FPL_COMM_ID_BYTES, "FPL_COMM_ID_BYTES must be sizeof(ncclUniqueId)");

extern "C" {

int fpl_comm_unique_id(uint8_t* id) {
    g_err[0] = 0;
    if (!id) return fail("fpl_comm_unique_id: null argument");
    if (!nccl().ok) return fail("fpl_comm_unique_id: libnccl.so.2 is not loadable");
    ncclUniqueId u;
    CKN(nccl().GetUniqueId(&u));
    memcpy(id, &u, sizeof(u));
    return 0;
}

int fpl_comm_init(fpl_ctx* c, const uint8_t* id, int rank, int n_ranks) {
    g_err[0] = 0;
    if (!c || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail("fpl_comm_init: bad argument");
    if (!nccl().ok) return fail("fpl_comm_init: libnccl.so.2 is not loadable");
    if (c->comm) return fail("fpl_comm_init: the context already has a communicator");
    CK(cudaSetDevice(c->device));
    ncclUniqueId u;
    memcpy(&u, id, sizeof(u));
    ncclComm_t m = nullptr;
    CKN(nccl().CommInitRank(&m, n_ranks, u, rank));
    c->comm.reset(m);
    c->comm_rank = rank; c->comm_size = n_ranks;
    CK(c->d_agree.grow_exact(1));
    if (!c->h_agree) CK(create_pinned(c->h_agree, 1));
    return 0;
}

int fpl_comm_destroy(fpl_ctx* c) {
    if (!c || !c->comm) return 0;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->comm.reset();
    c->comm_size = 1; c->comm_rank = 0;
    return 0;
}

int fpl_comm_size(fpl_ctx* c) { return c ? c->comm_size : 0; }

int fpl_comm_agree_cycles(fpl_ctx* c, int64_t* cycles) {
    g_err[0] = 0;
    if (!c || !c->comm) return fail("fpl_comm_agree_cycles: no communicator (fpl_comm_init first)");
    CK(cudaSetDevice(c->device));
    *c->h_agree = (long long)c->used_cycles;
    CK(cudaMemcpyAsync(c->d_agree, c->h_agree, sizeof(long long), cudaMemcpyHostToDevice, c->stream));
    CKN(nccl().AllReduce(c->d_agree, c->d_agree, 1, ncclInt64, ncclMax, c->comm, c->stream));
    CK(cudaMemcpyAsync(c->h_agree, c->d_agree, sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    const int64_t agreed = (int64_t)*c->h_agree;
    if (reserve_cycles(c, agreed > 0 ? agreed : 1)) return -1;      // every rank now holds at least `agreed` columns
    CK(cudaStreamSynchronize(c->stream));
    if (cycles) *cycles = agreed;
    return 0;
}

int fpl_allreduce_stats(fpl_ctx* c, int64_t cycles) {
    g_err[0] = 0;
    if (!c || !c->comm) return fail("fpl_allreduce_stats: no communicator (fpl_comm_init first)");
    CK(cudaSetDevice(c->device));
    if (cycles <= 0 && fpl_comm_agree_cycles(c, &cycles)) return -1;
    if (cycles > c->C) return fail("fpl_allreduce_stats: %lld cycles exceed this rank's capacity %lld (fpl_stats_reserve first)",
                                   (long long)cycles, (long long)c->C);
    if (cycles < c->used_cycles) return fail("fpl_allreduce_stats: %lld cycles do not cover this rank's longest read (%lld)",
                                             (long long)cycles, (long long)c->used_cycles);
    // rows [b*C, b*C + cycles) of the 16 per-cycle arrays, then the tail; the row pointers depend on this rank's C, the
    // counts do not, so ranks need not share a capacity.  One group = one fused launch.
    c->rep.built = false; c->html.built = false;
    if (c->comm_size > 1) c->lists.merged = true;
    if (cycles > c->reduced_rows) c->reduced_rows = cycles;
    Timed t(c, K_ALLREDUCE, false);
    CKN(nccl().GroupStart());
    for (int w = 0; w < 2; w++) {
        unsigned long long* blk = c->d_stats[w];
        if (cycles > 0)
            for (int b = 0; b < 16; b++)
                CKN(nccl().AllReduce(blk + (int64_t)b * c->C, blk + (int64_t)b * c->C, (size_t)cycles, ncclInt64, ncclSum, c->comm, c->stream));
        CKN(nccl().AllReduce(blk + 16 * c->C, blk + 16 * c->C, FPL_STATS_TAIL, ncclInt64, ncclSum, c->comm, c->stream));
    }
    CKN(nccl().AllReduce(c->d_counters, c->d_counters, (size_t)c->counter_words, ncclInt64, ncclSum, c->comm, c->stream));
    CKN(nccl().GroupEnd());
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// fpl_report_json: JsonReporter::report (src/jsonreporter.cpp:11-94) from the device accumulators.  The host builds the
// frame — every line but the 22 per-cycle curves, from a few hundred scalars — and the kernels of fpl_stats.cu print the
// curves (O(total_cycles) text) into the same device buffer, between the frame's pieces.
// ------------------------------------------------------------------------------------------------------------------
namespace {

struct RepBlock {                      // Stats::summarize's scalars of one block (src/stats.cpp:150-263)
    long long reads, bases, q20, q30, gc, cycles, lensum;
    const long long* tail;             // FPL_STATS_TAIL words
};

std::string gfmt(double v) {           // ostream << double
    char b[32];
    snprintf(b, sizeof(b), "%g", v);
    return b;
}

std::string dec(long long v) { return std::to_string(v); }

double ratio(long long a, long long b) { return b == 0 ? 0.0 : (double)a / (double)b; }

void summary_part(std::string& s, const char* key, const RepBlock& b) {
    s += std::string("\t\t\"") + key + "\": {\n";
    s += "\t\t\t\"total_reads\":" + dec(b.reads) + ",\n";
    s += "\t\t\t\"total_bases\":" + dec(b.bases) + ",\n";
    s += "\t\t\t\"q20_bases\":" + dec(b.q20) + ",\n";
    s += "\t\t\t\"q30_bases\":" + dec(b.q30) + ",\n";
    s += "\t\t\t\"q20_rate\":" + gfmt(ratio(b.q20, b.bases)) + ",\n";
    s += "\t\t\t\"q30_rate\":" + gfmt(ratio(b.q30, b.bases)) + ",\n";
    s += "\t\t\t\"read_mean_length\":" + dec(b.reads == 0 ? 0 : (int)(b.lensum / b.reads)) + ",\n";   // Stats::getMeanLength: int
    s += "\t\t\t\"gc_content\":" + gfmt(ratio(b.gc, b.bases)) + "\n";
}

// Stats::reportJson's lines in front of the first curve ("A":[)
void stats_head(std::string& s, const char* key, const RepBlock& b) {
    s += std::string("\t\"") + key + "\": {\n";
    s += "\t\t\"total_reads\": " + dec(b.reads) + ",\n";
    s += "\t\t\"total_bases\": " + dec(b.bases) + ",\n";
    s += "\t\t\"q20_bases\": " + dec(b.q20) + ",\n";
    s += "\t\t\"q30_bases\": " + dec(b.q30) + ",\n";
    s += "\t\t\"total_cycles\": " + dec(b.cycles) + ",\n";
    s += "\t\t\"quality_curves\": {\n\t\t\t\"A\":[";
}

// ... and behind the last one (the content curve "GC"): the 5-mer table (Stats::kmer3 / kmer2 names)
void stats_tail(std::string& s, const RepBlock& b, bool is_rna) {
    const char bases[4] = {'A', is_rna ? 'U' : 'T', 'C', 'G'};
    s += "]\n\t\t},\n\t\t\"kmer_count\": {\n";
    for (int i = 0; i < 64; i++) {
        for (int j = 0; j < 16; j++) {
            const char key[6] = {bases[(i >> 4) & 3], bases[(i >> 2) & 3], bases[i & 3], bases[(j >> 2) & 3], bases[j & 3], 0};
            s += std::string("\t\t\t\"") + key + "\":" + dec(b.tail[FPL_STATS_KMER + (i << 4) + j]);
            if (j != 15) s += ",";
        }
        s += i != 63 ? ",\n" : "\n";
    }
    s += "\t\t}\n\t},\n";
}

struct ClassComp {                     // classcomp (src/filterresult.h:14-23): by length, then lexicographically
    bool operator()(const std::string& a, const std::string& b) const {
        return a.size() != b.size() ? a.size() < b.size() : a < b;
    }
};

// The 23 frame pieces around the 22 curves (pre quality A,T,C,G,mean, content A,T,C,G,N,GC, then post): piece j comes
// in front of curve j, piece 22 behind the last.
std::vector<std::string> report_frame(const fpl_options& o, const std::vector<std::string>& ad, const long long* cnt,
                                      const RepBlock b[2], const char* version, const char* command, bool is_rna) {
    std::vector<std::string> p(23);
    std::string& s = p[0];
    s = "{\n\t\"summary\": {\n";
    s += std::string("\t\t\"fastplong_version\": \"") + version + "\",\n";
    summary_part(s, "before_filtering", b[0]);
    s += "\t\t},\n";
    summary_part(s, "after_filtering", b[1]);
    s += "\t\t}\n\t},\n";
    // FilterResult::reportJson (src/filterresult.cpp:120-132)
    s += "\t\"filtering_result\": {\n";
    s += "\t\t\"passed_filter_reads\": " + dec(cnt[FPL_CNT_FILTER + FPL_PASS_FILTER]) + ",\n";
    s += "\t\t\"low_quality_reads\": " + dec(cnt[FPL_CNT_FILTER + FPL_FAIL_QUALITY]) + ",\n";
    s += "\t\t\"too_many_N_reads\": " + dec(cnt[FPL_CNT_FILTER + FPL_FAIL_N_BASE]) + ",\n";
    if (o.complexity_enabled) s += "\t\t\"low_complexity_reads\": " + dec(cnt[FPL_CNT_FILTER + FPL_FAIL_COMPLEXITY]) + ",\n";
    s += "\t\t\"too_short_reads\": " + dec(cnt[FPL_CNT_FILTER + FPL_FAIL_LENGTH]) + ",\n";
    s += "\t\t\"too_long_reads\": " + dec(cnt[FPL_CNT_FILTER + FPL_FAIL_TOO_LONG]) + "\n";
    s += "\t},\n";
    // Options::adapterCuttingEnabled (src/options.cpp:27-33): the FASTA alone does not turn the section on
    if (o.adapter_enabled && (!ad[0].empty() || !ad[1].empty())) {
        auto name = [](const std::string& a) { return a.empty() || a == "auto" ? std::string("unspecified") : a; };   // :247-259
        s += "\t\"adapter_cutting\": {\n";
        s += "\t\t\"adapter_trimmed_reads\": " + dec(cnt[FPL_CNT_ADAPTER_READS]) + ",\n";
        s += "\t\t\"adapter_trimmed_bases\": " + dec(cnt[FPL_CNT_ADAPTER_BASES]) + ",\n";
        s += "\t\t\"read_start_adapter\": \"" + name(ad[0]) + "\",\n";
        s += "\t\t\"read_end_adapter\": \"" + name(ad[1]) + "\",\n";
        s += "\t\t\"read_adapter_counts\": {";
        // FilterResult::mAdapter from the event table, then outputAdaptersJson (src/filterresult.cpp:134-169)
        std::map<std::string, long long, ClassComp> m;
        for (size_t k = 0; k < ad.size(); k++)
            for (int side = 0; side < 2; side++)
                for (int len = 1; len <= (int)ad[k].size(); len++) {
                    const long long v = cnt[FPL_CNT_FIXED + ((int64_t)k * 2 + side) * (FPL_MAX_ADAPTER_LEN + 1) + len];
                    if (v) m[side == 0 ? ad[k].substr(ad[k].size() - len) : ad[k].substr(0, len)] += v;
                }
        long long total = 0, reported = 0;
        for (auto& kv : m) total += kv.second;
        if (total) {
            const double dtotal = (double)total;
            bool first = true;
            for (auto& kv : m) {
                if (kv.second / dtotal < 0.01) continue;
                if (!first) s += ", ";
                first = false;
                s += "\"" + kv.first + "\":" + dec(kv.second);
                reported += kv.second;
            }
            if (total - reported > 0) s += std::string(first ? "" : ", ") + "\"others\":" + dec(total - reported);
        }
        s += "}\n\t},\n";
    }
    // FilterResult::reportPolyXTrimJson (src/filterresult.cpp:187-204): keys are ATCG_BASES, never U
    if (o.polyx_enabled) {
        s += "\t\"polyx_trimming\": \t{\n";
        for (int which = 0; which < 2; which++) {
            const char* key = which ? "polyx_trimmed_bases" : "polyx_trimmed_reads";
            const long long* v = cnt + (which ? FPL_CNT_POLYX_BASES : FPL_CNT_POLYX_READS);
            s += std::string("\t\t\"total_") + key + "\": " + dec(v[0] + v[1] + v[2] + v[3]) + ",\n";
            s += std::string("\t\t\"") + key + "\":{\"A\": " + dec(v[0]) + ", \"T\": " + dec(v[1]) + ", \"C\": " + dec(v[2]) +
                 ", \"G\": " + dec(v[3]) + "}";
            s += which ? "\n\t},\n" : ",\n";
        }
    }
    const std::string t = is_rna ? "U" : "T";
    const std::string qual_names[5] = {"A", t, "C", "G", "mean"}, content_names[6] = {"A", t, "C", "G", "N", "GC"};
    for (int w = 0; w < 2; w++) {
        std::string& head = p[11 * w];
        stats_head(head, w ? "read_after_filtering" : "read_before_filtering", b[w]);
        for (int k = 1; k < 11; k++) {
            std::string& q = p[11 * w + k];
            if (k < 5) q = "],\n\t\t\t\"" + qual_names[k] + "\":[";
            else if (k == 5) q = "]\n\t\t},\n\t\t\"content_curves\": {\n\t\t\t\"A\":[";
            else q = "],\n\t\t\t\"" + content_names[k - 5] + "\":[";
        }
        stats_tail(p[11 * w + 11], b[w], is_rna);
    }
    p[22] += std::string("\t\"command\": \"") + command + "\"\n}";
    return p;
}

// the text of the accumulators as they are now, into c->rep
int report_build(fpl_ctx* c, const char* version, const char* command, bool is_rna) {
    FplReport& r = c->rep;
    r.built = false;
    const int64_t C = c->C;
    cudaStream_t s = c->stream;
    // 1. total_cycles, bases and G+C of both blocks; the tails and the counters come to the host
    CK(r.d_sum.grow_exact(6));
    unsigned long long sum[6] = {(unsigned long long)C, 0, 0, (unsigned long long)C, 0, 0};
    CK(cudaMemcpyAsync(r.d_sum, sum, sizeof(sum), cudaMemcpyHostToDevice, s));
    { Timed t(c, K_REPORT_CYCLES); launch_report_cycles(c->d_stats[0], c->d_stats[1], C, r.d_sum, s); }
    std::vector<long long> tails(2 * FPL_STATS_TAIL), cnt((size_t)c->counter_words);
    for (int w = 0; w < 2; w++)
        CK(cudaMemcpyAsync(tails.data() + w * FPL_STATS_TAIL, c->d_stats[w] + 16 * C, sizeof(long long) * FPL_STATS_TAIL,
                           cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(cnt.data(), c->d_counters, sizeof(long long) * c->counter_words, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(sum, r.d_sum, sizeof(sum), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    RepBlock b[2];
    for (int w = 0; w < 2; w++) {
        const long long* tl = tails.data() + w * FPL_STATS_TAIL;
        long long q20 = 0, q30 = 0;
        for (int i = 33 + 20; i < 127; i++) q20 += tl[FPL_STATS_QUALHIST + i];      // Stats::summarize :176-186: c + 33, c < 94
        for (int i = 33 + 30; i < 127; i++) q30 += tl[FPL_STATS_QUALHIST + i];
        b[w] = RepBlock{tl[FPL_STATS_READS], (long long)sum[3 * w + 1], q20, q30, (long long)sum[3 * w + 2], (long long)sum[3 * w],
                        tl[FPL_STATS_LENSUM], tl};
    }
    const std::vector<std::string> frame = report_frame(c->P.opt, c->adapter_str, cnt.data(), b, version, command, is_rna);
    // 2. the size of every value, their exclusive sum (the n + 1st entry: the curves' total)
    ReportCurves R = {};
    R.blk[0] = c->d_stats[0]; R.blk[1] = c->d_stats[1]; R.C = C; R.T[0] = b[0].cycles; R.T[1] = b[1].cycles;
    R.is_rna = is_rna ? 1 : 0;
    const int64_t n = 11 * (R.T[0] + R.T[1]);
    CK(r.d_size.grow(n + 1));
    CK(r.d_off.grow(n + 1));
    CK(cudaMemsetAsync(r.d_size + n, 0, sizeof(int64_t), s));
    { Timed t(c, K_REPORT_SIZES); launch_report_sizes(R, r.d_size, s); }
    CK(cub_call(r.d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, r.d_size.get(), r.d_off.get(), n + 1, s); }));
    int64_t end[22];                   // the running sum behind curve j
    for (int j = 0; j < 22; j++) {
        const int w = j / 11, k = j % 11;
        CK(cudaMemcpyAsync(&end[j], r.d_off + (w ? 11 * R.T[0] : 0) + (int64_t)(k + 1) * R.T[w], sizeof(int64_t),
                           cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    // 3. the frame pieces at their places, the curves between them
    std::vector<int64_t> src(24), dst(23);
    int64_t fbytes = 0, shift = 0;
    for (int j = 0; j < 23; j++) {
        src[j] = fbytes;
        dst[j] = (j ? end[j - 1] : 0) + shift;      // behind curve j - 1
        shift += (int64_t)frame[j].size();
        fbytes += (int64_t)frame[j].size();
        if (j < 22) R.shift[j] = shift;
    }
    src[23] = fbytes;
    const int64_t total = end[21] + shift;
    const size_t tables = sizeof(int64_t) * (24 + 23);
    r.h_frame.resize(tables + (size_t)fbytes);
    memcpy(r.h_frame.data(), src.data(), sizeof(int64_t) * 24);
    memcpy(r.h_frame.data() + sizeof(int64_t) * 24, dst.data(), sizeof(int64_t) * 23);
    for (int j = 0; j < 23; j++) memcpy(r.h_frame.data() + tables + src[j], frame[j].data(), frame[j].size());
    CK(r.d_frame.grow((int64_t)r.h_frame.size()));
    CK(r.d_text.grow(total));
    CK(cudaMemcpyAsync(r.d_frame, r.h_frame.data(), r.h_frame.size(), cudaMemcpyHostToDevice, s));
    {
        Timed t(c, K_REPORT_TEXT);
        const int64_t* d_src = reinterpret_cast<const int64_t*>(r.d_frame.get());
        launch_report_text(R, r.d_off, r.d_frame + tables, d_src, d_src + 24, 23, r.d_text, s);
        c->launches++;                 // + k_report_frame
    }
    CK(cudaGetLastError());
    r.n_bytes = total;
    r.built = true;
    return 0;
}

}  // namespace

extern "C" int fpl_report_json(fpl_ctx* c, const fpl_report_info* info, uint8_t* out, int64_t cap, int64_t* n_bytes) {
    g_err[0] = 0;
    if (!c || !info || !n_bytes) return fail("fpl_report_json: null argument");
    *n_bytes = 0;
    if (info->struct_size != (int32_t)sizeof(fpl_report_info))
        return fail("fpl_report_json: fpl_report_info.struct_size %d != %d (ABI mismatch)", info->struct_size, (int)sizeof(fpl_report_info));
    if (!info->version || !info->command) return fail("fpl_report_json: version and command must not be null");
    CK(cudaSetDevice(c->device));
    std::string key = std::string(info->version) + '\0' + info->command + '\0' + (info->is_rna ? "U" : "T");
    if (!c->rep.built || c->rep.key != key) {
        if (report_build(c, info->version, info->command, info->is_rna != 0)) { c->rep.built = false; return -1; }
        c->rep.key.swap(key);
    }
    *n_bytes = c->rep.n_bytes;
    if (!out || cap < c->rep.n_bytes) return 1;     // the text stays built: call again with room
    CK(cudaMemcpyAsync(out, c->rep.d_text, (size_t)c->rep.n_bytes, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// fpl_report_html: HtmlReporter::report (src/htmlreporter.cpp:75-253) from the device accumulators and read lists.  The host
// builds the frame — everything O(1), O(128), O(1024) or O(log total_cycles) — with the reference's own expressions; the
// kernels of fpl_stats.cu print the density lists and the down-sampled curves into the same device buffer, between its pieces.
// ------------------------------------------------------------------------------------------------------------------
namespace {

std::string to_str(double v) { return std::to_string(v); }        // to_string(double): "%f"

std::string format_number(long number) {                          // HtmlReporter::formatNumber
    double num = (double)number;
    const std::string unit[6] = {"", "K", "M", "G", "T", "P"};
    int order = 0;
    while (num > 1000.0) {
        order += 1;
        num /= 1000.0;
    }
    if (order == 0) return std::to_string(number);
    return std::to_string(num) + " " + unit[order];
}

std::string get_percents(long numerator, long denominator) {       // HtmlReporter::getPercents
    if (denominator == 0) return "0.0";
    return std::to_string((double)numerator * 100.0 / (double)denominator);
}

std::string row(const std::string& key, const std::string& v) {
    return "<tr><td class='col1'>" + key + "</td><td class='col2'>" + v + "</td></tr>\n";
}

std::string replace_all(std::string s, const std::string& a, const std::string& b) {
    for (size_t p = s.find(a); p != std::string::npos; p = s.find(a, p + b.size())) s.replace(p, a.size(), b);
    return s;
}

struct HtmlBlock {                     // the merged Stats' scalars the frame prints
    long reads, bases, lensum, cycles;
    long base_contents[8];
    int min_len, max_len, median_len, n50_len;
    const long long* tail;
    std::vector<long long> x;          // the curves' x list
};

std::vector<long long> curve_x(long cycles) {   // Stats::reportHtmlQuality / reportHtmlContents
    std::vector<long long> x;
    if (cycles <= 300) {
        for (int i = 0; i < cycles; i++) x.push_back(i + 1);
        return x;
    }
    for (int i = 0; i < 40 && i < cycles; i++) x.push_back(i + 1);
    double pos = 40;
    while (true) {
        pos *= 1.05;
        if (pos >= cycles) break;
        x.push_back((int)pos);
    }
    if (x.back() != cycles) x.push_back(cycles);
    return x;
}

std::string join_long(const std::vector<long long>& v) {
    std::string s;
    for (size_t i = 0; i < v.size(); i++) { if (i) s += ","; s += std::to_string(v[i]); }
    return s;
}

std::string gjoin(const std::vector<double>& v) {
    std::string s;
    for (size_t i = 0; i < v.size(); i++) { if (i) s += ","; s += gfmt(v[i]); }
    return s;
}

void basic_info(std::string& s, const std::string& type, const HtmlBlock& b) {   // Stats::reportHtmlBasicInfo
    const long* bc = b.base_contents;
    const long long* qh = b.tail + FPL_STATS_QUALHIST;
    long q[7];                         // Q40, Q30, Q20, Q15, Q10, Q7, Q5 as Stats::summarize adds them
    long acc = 0;
    for (int c = 40; c < 127 - 33; c++) acc += qh[c + 33];
    q[0] = acc;
    const int lo[6] = {30, 20, 15, 10, 7, 5}, hi[6] = {40, 30, 20, 15, 10, 7};
    for (int k = 0; k < 6; k++) {
        for (int c = lo[k]; c < hi[k]; c++) acc += qh[c + 33];
        q[k + 1] = acc;
    }
    const long gc = bc['G' & 7] + bc['C' & 7];
    s += "<div class='subsection_title'>" + type + ": Basic statistics</div>\n";
    s += "<table>\n";
    s += row("total reads:", format_number(b.reads));
    s += row("total bases:", format_number(b.bases));
    s += row("minimum length:", format_number(b.min_len));
    s += row("maximum length:", format_number(b.max_len));
    s += row("median length:", format_number(b.median_len));
    s += row("mean length:", format_number(b.reads == 0 ? 0 : (int)(b.lensum / b.reads)));
    s += row("N50 length:", format_number(b.n50_len));
    s += row("GC content:", get_percents(gc, b.bases) + "%");
    const char* names[7] = {"Q5", "Q7", "Q10", "Q15", "Q20", "Q30", "Q40"};
    for (int k = 0; k < 7; k++) {
        const long v = q[6 - k];
        s += row(std::string(names[k]) + " bases:", format_number(v) + " (" + get_percents(v, b.bases) + "%)");
    }
    s += "</table>\n";
}

void median_hist(std::string& s, const std::string& type, const HtmlBlock& b) {   // Stats::reporHtmlMedianQualHist
    const std::string sub = type + ": Read median quality statistics", div = replace_all(sub, " ", "_");
    const long long* hist = b.tail + FPL_STATS_MEDHIST;
    const long long* bases = b.tail + FPL_STATS_MEDBASES;
    s += "<div class='subsection_title'>" + sub + "</div>\n";
    int minVal = 0, maxVal = 0;
    for (int i = 0; i < 127 - 33; i++) {
        if (bases[i + 33] == 0) minVal++;
        else break;
    }
    for (int i = 127 - 33; i >= 0; i--)
        if (bases[i + 33] > 0) { maxVal = i; break; }
    const int offset = std::max(0, minVal - 1);
    int total = std::min(127 - 33, maxVal - minVal + 2);
    total = std::max(0, total);
    std::vector<long long> x(total);
    std::vector<double> pr(total), pb(total);
    for (int i = 0; i < total; i++) {
        x[i] = i + offset;
        pr[i] = (double)hist[i + offset + 33] * 100.0 / (double)b.reads;
        pb[i] = (double)bases[i + offset + 33] * 100.0 / (double)b.bases;
    }
    s += "<div id='mean_qual_length_histogram_figure'>\n";
    s += "<div class='figure' id='plot_median_qual_hist_" + div + "' style='height:400px;'></div>\n";
    s += "</div>\n";
    s += "\n<script type=\"text/javascript\">\n";
    s += "var readNum={x:[" + join_long(x) + "],y:[" + gjoin(pr) + "],name: '% reads',type:'bar',line:{color:'rgba(128,0,128,1.0)', width:1}\n};\n";
    s += "var baseNum={x:[" + join_long(x) + "],y:[" + gjoin(pb) +
         "],name: '% accumulated bases',type:'bar',line:{color:'rgba(128,128,0,1.0)', width:1}\n};\n";
    s += "var data = [readNum, baseNum];;\n";
    s += "var layout={legend: {x: 0, y: 1.0},title:'Read median quality distribution', xaxis:{title:'read median quality score'}, "
         "yaxis:{title:'Percent (%)'}};\n";
    s += "Plotly.newPlot('plot_median_qual_hist_" + div + "', data, layout);\n";
    s += "</script>\n";
}

std::string kmer_td(const HtmlBlock& b, int i, int j, const char* letters) {   // Stats::makeKmerTD
    const long val = b.tail[FPL_STATS_KMER + (i << 4) + j];
    const char kmer[6] = {letters[(i >> 4) & 3], letters[(i >> 2) & 3], letters[i & 3], letters[(j >> 2) & 3], letters[j & 3], 0};
    const double meanBases = (double)(b.bases + 1) / 2048;     // mKmerBufLen = 2 << (5 * 2): twice the 5-mers
    const double prop = val / meanBases;
    int r = 0, g = 0, bl = 0;
    if (prop <= 0.3) {
        const double frac = prop * 2.0;
        bl = 255 - 256 * frac;
        g = 255 * frac;
        r = bl * frac;
    } else if (prop > 3.0) {
        const double frac = 2.0 / prop;
        r = 255 - 128 * frac;
        g = 128 * frac;
        bl = r * frac;
    } else {
        r = g = bl = 196;
    }
    char col[32];
    snprintf(col, sizeof(col), "%s%x%s%x%s%x", r < 16 ? "0" : "", r, g < 16 ? "0" : "", g, bl < 16 ? "0" : "", bl);
    return std::string("<td style='background:#") + col + "' title='" + kmer + ": " + std::to_string(val) + "\n" + gfmt(prop) +
           " times as mean value'>" + kmer + "</td>";
}

void kmer_table(std::string& s, const std::string& type, const HtmlBlock& b, bool is_rna) {   // Stats::reportHtmlKMER
    const std::string sub = type + ": KMER counting", div = replace_all(replace_all(sub, " ", "_"), ":", "_");
    const char letters[4] = {'A', is_rna ? 'U' : 'T', 'C', 'G'};
    s += "<div class='subsection_title'>" + sub + "</div>\n";
    s += "<div  id='" + div + "'>\n";
    s += "<div class='sub_section_tips'>Darker background means larger counts. The count will be shown on mouse over.</div>\n";
    s += "<table class='kmer_table' style='width:680px;'>\n";
    s += "<tr><td></td>";
    for (int h = 0; h < 16; h++) s += std::string("<td style='color:#333333'>") + letters[(h >> 2) & 3] + letters[h & 3] + "</td>";
    s += "</tr>\n";
    for (int i = 0; i < 64; i++) {
        s += std::string("<tr><td style='color:#333333'>") + letters[(i >> 4) & 3] + letters[(i >> 2) & 3] + letters[i & 3] + "</td>";
        for (int j = 0; j < 16; j++) s += kmer_td(b, i, j, letters);
        s += "</tr>\n";
    }
    s += "</table>\n</div>\n";
}

std::string section_open(const char* id, const char* title) {
    return std::string("<div class='section_div'>\n<div class='section_title' onclick=showOrHide('") + id + "')><a name='summary'>" + title +
           "</a></div>\n<table id='" + id + "' class='section_table'>\n<tr><td>\n";
}

const char* const kSectionMid = "</td><td>\n";
const char* const kSectionClose = "</td></tr>\n</table>\n</div>\n";

// The HTML_SEGS + 1 frame pieces: piece j in front of segment j, the last behind them all
std::vector<std::string> html_frame(const fpl_options& o, const long long* cnt, const HtmlBlock b[2], const fpl_report_html_info& info) {
    std::vector<std::string> p(1);
    auto hole = [&] { p.emplace_back(); };
    const std::string time_text = info.time_text, version = info.version;
    const bool rna = info.is_rna != 0;
    const char* type[2] = {"Before filtering", "After filtering"};
    std::string* s = &p.back();
    // printHeader: printJS, printCSS
    *s += "<html><head><meta http-equiv=\"content-type\" content=\"text/html;charset=utf-8\" />";
    *s += "<title>fastplong report at " + time_text + " </title>";
    *s += "<script src='https://opengene.org/plotly-1.2.0.min.js'></script>\n";
    *s += "\n<script type='text/javascript'>\n";
    *s += "    window.Plotly || document.write('<script src=\"https://cdn.plot.ly/plotly-1.2.0.min.js\"><\\/script>')\n";
    *s += "</script>\n";
    *s += "\n<script type=\"text/javascript\">\n";
    *s += "    function showOrHide(divname) {\n";
    *s += "        div = document.getElementById(divname);\n";
    *s += "        if(div.style.display == 'none')\n";
    *s += "            div.style.display = 'block';\n";
    *s += "        else\n";
    *s += "            div.style.display = 'none';\n";
    *s += "    }\n";
    *s += "</script>\n";
    static const char* const css[] = {
        "<style type=\"text/css\">",
        "td {border:1px solid #dddddd;padding:5px;font-size:12px;}",
        "table {border:1px solid #999999;padding:2x;border-collapse:collapse;width:100%}",
        ".col1 {width:240px; font-weight:bold;}",
        ".adapter_col {width:500px; font-size:10px;}",
        "img {padding:30px;}",
        "#menu {font-family:Consolas, 'Liberation Mono', Menlo, Courier, monospace;}",
        "#menu a {color:#0366d6; font-size:18px;font-weight:600;line-height:28px;text-decoration:none;font-family:-apple-system, "
        "BlinkMacSystemFont, 'Segoe UI', Helvetica, Arial, sans-serif, 'Apple Color Emoji', 'Segoe UI Emoji', 'Segoe UI Symbol'}",
        "a:visited {color: #999999}",
        ".alignleft {text-align:left;}",
        ".alignright {text-align:right;}",
        ".figure {width:680px;height:600px;}",
        ".header {color:#ffffff;padding:1px;height:20px;background:#000000;}",
        ".section_title {color:#ffffff;font-size:20px;padding:5px;text-align:left;background:#663355; margin-top:10px;}",
        ".section_table {width:100%;}",
        ".subsection_title {font-size:16px;padding:5px;margin-top:10px;text-align:left;color:#663355}",
        "#container {text-align:center;padding:3px 3px 3px 10px;font-family:Arail,'Liberation Mono', Menlo, Courier, monospace;}",
        ".menu_item {text-align:left;padding-top:5px;font-size:18px;}",
        ".highlight {text-align:left;padding-top:30px;padding-bottom:30px;font-size:20px;line-height:35px;}",
        "#helper {text-align:left;border:1px dotted #fafafa;color:#777777;font-size:12px;}",
        "#footer {text-align:left;padding:15px;color:#ffffff;font-size:10px;background:#663355;font-family:Arail,'Liberation Mono', Menlo, "
        "Courier, monospace;}",
        ".kmer_table {text-align:center;font-size:8px;padding:2px;}",
        ".kmer_table td{text-align:center;font-size:8px;padding:0px;color:#ffffff}",
        ".sub_section_tips {color:#999999;font-size:10px;padding-left:5px;padding-bottom:3px;}",
        "</style>"};
    for (const char* line : css) *s += std::string(line) + "\n";
    *s += "</head>";
    *s += "<body><div id='container'>";
    // printSummary, FilterResult::reportHtml (src/filterresult.cpp:227-242)
    *s += "\n";
    *s += "<h3 style='text-align:left;'><a href='https://github.com/OpenGene/fastplong' target='_blank' style='color:#663355;"
          "text-decoration:none;'>" + std::string(info.title) + "</a><a href='https://github.com/OpenGene/fastplong' target='_blank' "
          "style='font-size:-2;text-decoration:none;'>(fastplong version v" + version + ")</a></h3>\n";
    *s += "<div class='section_div'>\n";
    *s += "<div class='section_title' onclick=showOrHide('summary')><a name='summary'>Summary</a> </div>\n";
    *s += "<div id='summary'>\n";
    *s += "<div class='subsection_title'>Filtering result</div>\n";
    *s += "<div id='filtering_result'>\n";
    {
        const double total = (double)b[0].reads;
        const long long* f = cnt + FPL_CNT_FILTER;
        auto fr = [&](const char* key, int code) {
            *s += row(key, format_number(f[code]) + " (" + to_str(f[code] * 100.0 / total) + "%)");
        };
        *s += "<table class='summary_table'>\n";
        fr("reads passed filters:", FPL_PASS_FILTER);
        fr("reads with low quality:", FPL_FAIL_QUALITY);
        fr("reads with too many N:", FPL_FAIL_N_BASE);
        if (o.length_filter_enabled) {
            fr("reads too short:", FPL_FAIL_LENGTH);
            if (o.length_max > 0) fr("reads too long:", FPL_FAIL_TOO_LONG);
        }
        if (o.complexity_enabled) fr("reads with low complexity:", FPL_FAIL_COMPLEXITY);
        *s += "</table>\n";
    }
    *s += "</div>\n";
    *s += "</div>\n";
    *s += "</div>\n";
    *s += section_open("basic_stat", "Basic statistics");
    basic_info(*s, type[0], b[0]);
    *s += kSectionMid;
    basic_info(*s, type[1], b[1]);
    *s += kSectionClose;
    *s += section_open("median_qual_stat", "Median qual histogram");
    median_hist(*s, type[0], b[0]);
    *s += kSectionMid;
    median_hist(*s, type[1], b[1]);
    *s += kSectionClose;
    // Stats::reporHtmlMedianQualLengthDensity: segments 0..3
    *s += section_open("median_qual_length_density", "Median qual length density");
    for (int w = 0; w < 2; w++) {
        const std::string sub = std::string(type[w]) + ": Density plot of read median quality and read length", div = replace_all(sub, " ", "_");
        if (w) *s += kSectionMid;
        *s += "<div class='subsection_title'>" + sub + "</div>\n";
        *s += "<div id='mean_qual_length_density_figure'>\n";
        *s += "<div class='figure' id='plot_median_qual_length_density_" + div + "' style='height:400px;'></div>\n";
        *s += "</div>\n";
        *s += "\n<script type=\"text/javascript\">\n";
        *s += "var density={x:[";
        hole(); s = &p.back();
        *s += "],y:[";
        hole(); s = &p.back();
        *s += "],name: '% reads',type:'histogram2dcontour',line:{color:'rgba(128,0,128,1.0)', width:1}\n};\n";
        *s += "var data = [density];\n";
        *s += "var layout={legend: {x: 0, y: 1.0},title:' Density plot of read median quality and read length', xaxis:{title:'read median "
              "quality score'}, yaxis:{title:'Read length', type:'log'}};\n";
        *s += "Plotly.newPlot('plot_median_qual_length_density_" + div + "', data, layout);\n";
        *s += "</script>\n";
    }
    *s += kSectionClose;
    // Stats::reportHtmlQuality / reportHtmlContents: segments 4..25
    const std::string t = rna ? "U" : "T";
    const std::string qnames[5] = {"A", t, "C", "G", "mean"}, cnames[6] = {"A", t, "C", "G", "N", "GC"};
    const char* const qcolors[5] = {"rgba(128,128,0,1.0)", "rgba(128,0,128,1.0)", "rgba(0,255,0,1.0)", "rgba(0,0,255,1.0)", "rgba(20,20,20,1.0)"};
    const char* const ccolors[6] = {"rgba(128,128,0,1.0)", "rgba(128,0,128,1.0)", "rgba(0,255,0,1.0)", "rgba(0,0,255,1.0)",
                                    "rgba(255, 0, 0, 1.0)", "rgba(20,20,20,1.0)"};
    for (int content = 0; content < 2; content++) {
        *s += content ? section_open("contents_stat", "Base contents statistics") : section_open("quality_stat", "Quality statistics");
        for (int w = 0; w < 2; w++) {
            const HtmlBlock& B = b[w];
            const std::string sub = std::string(type[w]) + (content ? ": base contents" : ": quality");
            const std::string div = replace_all(replace_all(sub, " ", "_"), ":", "_");
            if (w) *s += kSectionMid;
            *s += "<div class='subsection_title'>" + sub + "</div>\n";
            *s += "<div id='" + div + "'>\n";
            *s += "<div class='sub_section_tips'>Value of each position will be shown on mouse over.</div>\n";
            *s += "<div class='figure' id='plot_" + div + "'></div>\n";
            *s += "</div>\n";
            *s += "\n<script type=\"text/javascript\">\n";
            *s += "var data=[";
            const std::string xs = join_long(B.x);
            for (int k = 0; k < (content ? 6 : 5); k++) {
                std::string name = content ? cnames[k] : qnames[k];
                if (content) {
                    const long count = k < 5 ? B.base_contents[cnames[k][0] & 7] : B.base_contents['G' & 7] + B.base_contents['C' & 7];
                    std::string percentage = std::to_string((double)count * 100.0 / B.bases);
                    if (percentage.length() > 5) percentage = percentage.substr(0, 5);
                    name = cnames[k] + "(" + percentage + "%)";
                }
                *s += "{x:[" + xs + "],y:[";
                hole(); s = &p.back();
                *s += "],name: '" + name + "',mode:'lines',line:{color:'" + (content ? ccolors[k] : qcolors[k]) + "', width:1}\n},";
            }
            *s += "];\n";
            *s += "var layout={title:'', xaxis:{title:'position'";
            if (B.cycles > 300) *s += ",type:'log'";
            *s += content ? "}, yaxis:{title:'base content ratios'}};\n" : "}, yaxis:{title:'quality'}};\n";
            *s += "Plotly.newPlot('plot_" + div + "', data, layout);\n";
            *s += "</script>\n";
        }
        *s += kSectionClose;
    }
    *s += section_open("kmer_stat", "k-mer statistics");
    kmer_table(*s, type[0], b[0], rna);
    *s += kSectionMid;
    kmer_table(*s, type[1], b[1], rna);
    *s += kSectionClose;
    // printFooter
    *s += "\n</div>\n";
    *s += "<div id='footer'> ";
    *s += "<p>" + std::string(info.command) + "</p>";
    *s += "fastplong " + version + ", at " + time_text + " </div>";
    *s += "</body></html>";
    return p;
}

int html_build(fpl_ctx* c, const fpl_report_html_info& info) {
    FplHtml& h = c->html;
    FplLists& L = c->lists;
    h.built = false;
    const int64_t C = c->C;
    cudaStream_t s = c->stream;
    // 1. total_cycles, bases and G+C (k_report_cycles), then the base-bin counts below total_cycles
    CK(h.d_sum.grow_exact(22));
    CK(h.d_lstat.grow_exact(8));
    unsigned long long sum[22] = {(unsigned long long)C, 0, 0, (unsigned long long)C, 0, 0};
    CK(cudaMemcpyAsync(h.d_sum, sum, sizeof(sum), cudaMemcpyHostToDevice, s));
    { Timed t(c, K_HTML_CYCLES); launch_report_cycles(c->d_stats[0], c->d_stats[1], C, h.d_sum, s); }
    std::vector<long long> tails(2 * FPL_STATS_TAIL), cnt((size_t)c->counter_words);
    for (int w = 0; w < 2; w++)
        CK(cudaMemcpyAsync(tails.data() + w * FPL_STATS_TAIL, c->d_stats[w] + 16 * C, sizeof(long long) * FPL_STATS_TAIL,
                           cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(cnt.data(), c->d_counters, sizeof(long long) * c->counter_words, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(sum, h.d_sum, 6 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const int64_t T[2] = {(int64_t)sum[0], (int64_t)sum[3]};
    {
        Timed t(c, K_HTML_CYCLES);
        for (int w = 0; w < 2; w++) launch_html_bins(c->d_stats[w], C, T[w], h.d_sum + 6 + 8 * w, s);
        c->launches += (T[0] > 0) + (T[1] > 0) - 1;  // one k_html_bins per block with cycles
    }
    // 2. each list grouped by median: the entries of bins 0..127 are the density pairs, bin 128 the empty reads
    int64_t M[2] = {0, 0}, NE[2] = {0, 0};
    for (int w = 0; w < 2; w++) {
        const int64_t n = L.n[w], nch = (n + HTML_CHUNK - 1) / HTML_CHUNK;
        if (!n) continue;
        const int64_t m = HTML_BINS * nch + 1;
        CK(h.d_mat.grow(m));
        CK(h.d_moff.grow(m));
        CK(h.d_grp[w].grow(n));
        CK(cudaMemsetAsync(h.d_mat + m - 1, 0, sizeof(long long), s));
        { Timed t(c, K_HTML_GROUP_HIST); launch_html_hist(L.d[w], n, nch, h.d_mat, s); }
        CK(cub_call(h.d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, h.d_mat.get(), h.d_moff.get(), m, s); }));
        { Timed t(c, K_HTML_GROUP_SCATTER); launch_html_scatter(L.d[w], n, nch, h.d_moff, h.d_grp[w], s); }
        CK(cudaMemcpyAsync(&NE[w], h.d_moff + 128 * nch, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&M[w], h.d_moff + 129 * nch, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    // 3. Stats::calcLengthHistogram over [0, longest read]
    const int64_t H = c->used_cycles + 1;
    CK(h.d_hist.grow(2 * H));
    CK(h.d_lwork.grow(6 * H));
    CK(cudaMemsetAsync(h.d_hist, 0, sizeof(unsigned long long) * 2 * H, s));
    const int init[8] = {INT_MAX, -1, INT_MAX, INT_MAX, INT_MAX, -1, INT_MAX, INT_MAX};
    CK(cudaMemcpyAsync(h.d_lstat, init, sizeof(init), cudaMemcpyHostToDevice, s));
    for (int w = 0; w < 2; w++) {
        unsigned long long* hist = h.d_hist + w * H;
        long long *ccum = h.d_lwork + 3 * w * H, *prod = ccum + H, *pcum = prod + H;
        Timed t(c, K_HTML_LENGTHS);
        launch_html_lenhist(L.d[w], L.n[w], hist, s);
        launch_html_lenprod(hist, H, prod, s);
        CK(cub_call(h.d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, hist, ccum, H, s); }));
        CK(cub_call(h.d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, prod, pcum, H, s); }));
        const long long lensum = tails[w * FPL_STATS_TAIL + FPL_STATS_LENSUM];
        launch_html_lensearch(hist, ccum, prod, pcum, H, lensum / 2, (unsigned long long)M[w] / 2, h.d_lstat + 4 * w, s);
        c->launches += L.n[w] ? 2 : 1;               // k_html_lenhist (with entries), k_html_lenprod, k_html_lensearch
    }
    int lstat[8];
    CK(cudaMemcpyAsync(lstat, h.d_lstat, sizeof(lstat), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(sum + 6, h.d_sum + 6, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    HtmlBlock b[2];
    for (int w = 0; w < 2; w++) {
        const long long* tl = tails.data() + w * FPL_STATS_TAIL;
        if (M[w] != tl[FPL_STATS_READS])
            return fail("fpl_report_html: the %s read list holds %lld reads, the Stats block %lld", w ? "post-filter" : "pre-filter",
                        (long long)M[w], tl[FPL_STATS_READS]);
        HtmlBlock& B = b[w];
        B.reads = tl[FPL_STATS_READS]; B.bases = (long)sum[3 * w + 1]; B.lensum = tl[FPL_STATS_LENSUM]; B.cycles = (long)T[w];
        for (int k = 0; k < 8; k++) B.base_contents[k] = (long)sum[6 + 8 * w + k];
        const int* ls = lstat + 4 * w;
        B.min_len = ls[0] == INT_MAX ? 0 : ls[0];
        B.max_len = ls[1] < 0 ? 0 : ls[1];
        B.median_len = ls[2] == INT_MAX ? 0 : ls[2];
        B.n50_len = ls[3] == INT_MAX ? 0 : ls[3];
        B.tail = tl;
        B.x = curve_x(B.cycles);
    }
    // 4. the per-cycle values, then the down-sampled means
    const int64_t R[2] = {(int64_t)b[0].x.size(), (int64_t)b[1].x.size()};
    CK(h.d_x.grow(R[0] + R[1] + 1));
    CK(h.d_vals.grow(11 * (T[0] + T[1]) + 1));
    CK(h.d_sums.grow(11 * (R[0] + R[1]) + 1));
    std::vector<long long> xs(b[0].x);
    xs.insert(xs.end(), b[1].x.begin(), b[1].x.end());
    if (!xs.empty()) CK(cudaMemcpyAsync(h.d_x, xs.data(), sizeof(long long) * xs.size(), cudaMemcpyHostToDevice, s));
    for (int w = 0; w < 2; w++) {
        double* vals = h.d_vals + (w ? 11 * T[0] : 0);
        if (T[w]) { Timed t(c, K_HTML_VALUES); launch_html_values(c->d_stats[w], C, T[w], info.is_rna != 0, vals, s); }
        if (R[w]) { Timed t(c, K_HTML_SUMS); launch_html_sums(vals, T[w], h.d_x + (w ? R[0] : 0), R[w], h.d_sums + (w ? 11 * R[0] : 0), s); }
    }
    // 5. the frame, the size of every value and their exclusive sum
    const std::vector<std::string> frame = html_frame(c->P.opt, cnt.data(), b, info);
    if ((int)frame.size() != HTML_SEGS + 1) return fail("fpl_report_html: internal error (%d frame pieces)", (int)frame.size());
    HtmlText X = {};
    int64_t items = 0;
    for (int j = 0; j < HTML_SEGS; j++) {
        X.start[j] = items;
        if (j < 4) {                   // density x, y of block j / 2
            const int w = j / 2;
            X.kind[j] = j % 2; X.blk[j] = w;
            items += M[w];
        } else {                       // quality: 4..13 = curves 0..4 of block 0, then of block 1; content: 14..25 = curves 5..10
            const int q = j - 4, content = q >= 10;
            const int w = content ? (q - 10) / 6 : q / 5, k = content ? 5 + (q - 10) % 6 : q % 5;
            X.kind[j] = 2; X.blk[j] = w;
            X.base[j] = (int64_t)k * R[w];
            items += R[w];
        }
    }
    X.start[HTML_SEGS] = items;
    for (int w = 0; w < 2; w++) {
        X.grp[w] = h.d_grp[w]; X.nonempty[w] = NE[w];
        X.sums[w] = h.d_sums + (w ? 11 * R[0] : 0);
        X.x[w] = h.d_x + (w ? R[0] : 0);
    }
    CK(h.d_size.grow(items + 1));
    CK(h.d_off.grow(items + 1));
    CK(cudaMemsetAsync(h.d_size + items, 0, sizeof(int64_t), s));
    if (items) { Timed t(c, K_HTML_SIZES); launch_html_sizes(X, h.d_size, s); }
    CK(cub_call(h.d_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, h.d_size.get(), h.d_off.get(), items + 1, s); }));
    int64_t end[HTML_SEGS];            // the running sum behind segment j
    for (int j = 0; j < HTML_SEGS; j++)
        CK(cudaMemcpyAsync(&end[j], h.d_off + X.start[j + 1], sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    // 6. the frame pieces at their places, the values between them
    const int np = HTML_SEGS + 1;
    std::vector<int64_t> src(np + 1), dst(np);
    int64_t fbytes = 0, shift = 0;
    for (int j = 0; j < np; j++) {
        src[j] = fbytes;
        dst[j] = (j ? end[j - 1] : 0) + shift;
        shift += (int64_t)frame[j].size();
        fbytes += (int64_t)frame[j].size();
        if (j < HTML_SEGS) X.shift[j] = shift;
    }
    src[np] = fbytes;
    const int64_t total = end[HTML_SEGS - 1] + shift;
    const size_t tables = sizeof(int64_t) * (2 * np + 1);
    h.h_frame.resize(tables + (size_t)fbytes);
    memcpy(h.h_frame.data(), src.data(), sizeof(int64_t) * (np + 1));
    memcpy(h.h_frame.data() + sizeof(int64_t) * (np + 1), dst.data(), sizeof(int64_t) * np);
    for (int j = 0; j < np; j++) memcpy(h.h_frame.data() + tables + src[j], frame[j].data(), frame[j].size());
    CK(h.d_frame.grow((int64_t)h.h_frame.size()));
    CK(h.d_text.grow(total));
    CK(cudaMemcpyAsync(h.d_frame, h.h_frame.data(), h.h_frame.size(), cudaMemcpyHostToDevice, s));
    {
        Timed t(c, K_HTML_TEXT);
        const int64_t* d_src = reinterpret_cast<const int64_t*>(h.d_frame.get());
        launch_html_text(X, h.d_off, h.d_frame + tables, d_src, d_src + np + 1, np, h.d_text, s);
        if (items) c->launches++;      // k_report_frame + k_html_text (only with values to print)
    }
    CK(cudaGetLastError());
    h.n_bytes = total;
    h.built = true;
    return 0;
}

}  // namespace

extern "C" int fpl_keep_read_lists(fpl_ctx* c, int enabled) {
    g_err[0] = 0;
    if (!c) return fail("fpl_keep_read_lists: null context");
    c->lists.keep = enabled != 0;
    return 0;
}

extern "C" int fpl_report_html(fpl_ctx* c, const fpl_report_html_info* info, uint8_t* out, int64_t cap, int64_t* n_bytes) {
    g_err[0] = 0;
    if (!c || !info || !n_bytes) return fail("fpl_report_html: null argument");
    *n_bytes = 0;
    if (info->struct_size != (int32_t)sizeof(fpl_report_html_info))
        return fail("fpl_report_html: fpl_report_html_info.struct_size %d != %d (ABI mismatch)", info->struct_size,
                    (int)sizeof(fpl_report_html_info));
    if (!info->version || !info->command || !info->title || !info->time_text)
        return fail("fpl_report_html: version, command, title and time_text must not be null");
    if (!c->lists.complete)
        return fail("fpl_report_html: read-list capture (fpl_keep_read_lists) was off for an fpl_process_* call since fpl_create "
                    "or fpl_reset: the lists are incomplete");
    if (c->lists.merged)
        return fail("fpl_report_html: fpl_allreduce_stats merged the Stats over several ranks, but not the read lists");
    CK(cudaSetDevice(c->device));
    std::string key = std::string(info->version) + '\0' + info->command + '\0' + info->title + '\0' + info->time_text + '\0' +
                      (info->is_rna ? "U" : "T");
    if (!c->html.built || c->html.key != key) {
        if (html_build(c, *info)) { c->html.built = false; return -1; }
        c->html.key.swap(key);
    }
    *n_bytes = c->html.n_bytes;
    if (!out || cap < c->html.n_bytes) return 1;     // the text stays built: call again with room
    CK(cudaMemcpyAsync(out, c->html.d_text, (size_t)c->html.n_bytes, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// fpl_merge_stats: Stats::merge / FilterResult::merge over [dst, src...] on one device (SingleEndProcessor::process,
// src/seprocessor.cpp:108-121).  The accumulators are summed by k_merge_stats, the read lists appended by device copies; all of
// it on dst's stream, between an event wait on every source's stream and a wait of every source's stream on dst's.
// ------------------------------------------------------------------------------------------------------------------
extern "C" int fpl_merge_stats(fpl_ctx* c, fpl_ctx* const* src, int n_src) {
    g_err[0] = 0;
    if (!c) return fail("fpl_merge_stats: null destination context");
    if (n_src < 0) return fail("fpl_merge_stats: negative number of sources (%d)", n_src);
    if (n_src > 0 && !src) return fail("fpl_merge_stats: null source list");
    // every fpl_options field but struct_size (the first) and reserved (the last)
    const size_t ob = offsetof(fpl_options, device), oe = offsetof(fpl_options, reserved);
    for (int k = 0; k < n_src; k++) {
        const fpl_ctx* s = src[k];
        if (!s) return fail("fpl_merge_stats: source %d is null", k);
        if (s == c) return fail("fpl_merge_stats: source %d is the destination itself", k);
        if (s->device != c->device)
            return fail("fpl_merge_stats: source %d is on device %d, the destination on device %d (merging across devices is not "
                        "supported)", k, s->device, c->device);
        if (memcmp(reinterpret_cast<const char*>(&s->P.opt) + ob, reinterpret_cast<const char*>(&c->P.opt) + ob, oe - ob))
            return fail("fpl_merge_stats: source %d was created with other options than the destination", k);
        if (s->adapter_str != c->adapter_str)
            return fail("fpl_merge_stats: source %d was created with another adapter list than the destination", k);
    }
    if (n_src == 0) return 0;
    CK(cudaSetDevice(c->device));
    FplLists& L = c->lists;
    int64_t rows = 0, used = c->used_cycles, reduced = c->reduced_rows, total[2] = {L.n[0], L.n[1]};
    bool complete = L.complete, merged = L.merged;
    std::vector<MergeSrc> tab((size_t)n_src);
    for (int k = 0; k < n_src; k++) {
        const fpl_ctx* s = src[k];
        const int64_t r = std::max(s->used_cycles, s->reduced_rows);
        tab[k] = MergeSrc{{s->d_stats[0], s->d_stats[1]}, s->d_counters, s->C, r};
        rows = std::max(rows, r);
        used = std::max(used, s->used_cycles);
        reduced = std::max(reduced, s->reduced_rows);
        complete = complete && s->lists.complete;
        merged = merged || s->lists.merged;
        for (int w = 0; w < 2; w++) total[w] += s->lists.n[w];
    }
    // the capacities first: they synchronise dst's stream when they grow
    if (reserve_cycles(c, rows)) return -1;
    if (L.keep && (grow_list(c, 0, total[0]) || grow_list(c, 1, total[1]))) return -1;
    CK(c->d_merge.grow(n_src));
    if (!c->merge_ev) CK(create_event(c->merge_ev, false));
    for (int k = 0; k < n_src; k++) {         // behind everything queued on the sources
        CK(cudaEventRecord(c->merge_ev, src[k]->stream));
        CK(cudaStreamWaitEvent(c->stream, c->merge_ev, 0));
    }
    CK(cudaMemcpyAsync(c->d_merge, tab.data(), sizeof(MergeSrc) * n_src, cudaMemcpyHostToDevice, c->stream));
    {
        Timed t(c, K_MERGE_STATS);
        launch_merge_stats(c->d_stats[0], c->d_stats[1], c->d_counters, c->C, rows, c->counter_words, c->d_merge, n_src, c->stream);
    }
    if (L.keep) {
        for (int w = 0; w < 2; w++) {
            int64_t at = L.n[w];
            for (int k = 0; k < n_src; k++) {
                const int64_t n = src[k]->lists.n[w];
                if (n) CK(cudaMemcpyAsync(L.d[w] + at, src[k]->lists.d[w], sizeof(HtmlEntry) * n, cudaMemcpyDeviceToDevice, c->stream));
                at += n;
            }
            L.n[w] = at;
        }
    } else {
        complete = false;                     // the sources' entries were not captured, as in a call with capture off
    }
    CK(cudaEventRecord(c->merge_ev, c->stream));
    for (int k = 0; k < n_src; k++) CK(cudaStreamWaitEvent(src[k]->stream, c->merge_ev, 0));   // before the sources' next work
    c->used_cycles = used; c->reduced_rows = reduced;
    L.complete = complete; L.merged = merged;
    c->rep.built = false; c->html.built = false;
    CK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// fpl_state_export / fpl_state_merge: a context's state as a byte image (layout: include/fplgpu.h) and images merged with
// fpl_merge_stats' semantics (Stats::merge, src/stats.cpp:1013-1082; FilterResult::merge, src/filterresult.cpp:28-61).  The
// images' Stats and counter sections are staged in one device buffer, where each image's compact blocks (capacity = rows) are a
// k_merge_stats source as they are; the read-list entries are copied behind dst's.
// ------------------------------------------------------------------------------------------------------------------
#if defined(__BYTE_ORDER__) && __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "state images are little-endian: the library supports little-endian hosts only"
#endif

namespace {

enum { SI_MAGIC, SI_FORMAT, SI_ABI, SI_TOTAL, SI_N_ADAPTERS, SI_ADAPTER_BYTES, SI_COUNTER_WORDS, SI_ROWS, SI_USED, SI_REDUCED,
       SI_KEEP, SI_COMPLETE, SI_MERGED, SI_LIST0, SI_LIST1, SI_WORDS };
// the fpl_options bytes in the image: what fpl_merge_stats compares (device up to reserved) but device
const size_t kOptBegin = offsetof(fpl_options, trim_front), kOptEnd = offsetof(fpl_options, reserved);
const int64_t kOptAt = 8 * SI_WORDS;
static_assert(offsetof(fpl_options, device) + sizeof(int32_t) == offsetof(fpl_options, trim_front), "device precedes trim_front");
static_assert(kOptAt + (int64_t)(kOptEnd - kOptBegin) + 4 == FPL_STATE_HEADER_BYTES, "FPL_STATE_HEADER_BYTES");
static_assert(sizeof(HtmlEntry) == 8, "list entries are 8 bytes in the image");

int64_t pad8(int64_t n) { return (n + 7) & ~(int64_t)7; }

int64_t adapter_section_bytes(const std::vector<std::string>& a) {
    int64_t n = 0;
    for (const std::string& s : a) n += 8 + pad8((int64_t)s.size());
    return n;
}

// one validated image: its flags, list lengths and where its sections are
struct StateImage {
    int64_t rows, used, reduced, n[2];
    bool complete, merged;
    const uint8_t* stats;                   // pre and post Stats, then the counters: contiguous
    const uint8_t* list[2];
};

// Validation of image i against dst, on the host, reading nothing outside [p, p + n)
int parse_image(const fpl_ctx* c, int i, const uint8_t* p, int64_t n, StateImage& im) {
    if (!p) return fail("fpl_state_merge: image %d is null", i);
    if (n < 0) return fail("fpl_state_merge: image %d has a negative size (%lld)", i, (long long)n);
    if (n < FPL_STATE_HEADER_BYTES)
        return fail("fpl_state_merge: image %d is truncated: %lld bytes, the header alone is %d", i, (long long)n, FPL_STATE_HEADER_BYTES);
    int64_t h[SI_WORDS];
    memcpy(h, p, sizeof(h));
    if ((uint64_t)h[SI_MAGIC] != FPL_STATE_MAGIC) return fail("fpl_state_merge: image %d is not a state image (bad magic number)", i);
    if (h[SI_FORMAT] != FPL_STATE_FORMAT)
        return fail("fpl_state_merge: image %d has image format %lld, this library reads format %d", i, (long long)h[SI_FORMAT],
                    FPL_STATE_FORMAT);
    if (h[SI_ABI] != FPL_ABI_VERSION)
        return fail("fpl_state_merge: image %d was written with FPL_ABI_VERSION %lld, this library is %d", i, (long long)h[SI_ABI],
                    FPL_ABI_VERSION);
    if (h[SI_TOTAL] != n)
        return fail("fpl_state_merge: image %d: its header says %lld bytes, %lld were given (truncated, or trailing bytes)", i,
                    (long long)h[SI_TOTAL], (long long)n);
    for (int k = SI_N_ADAPTERS; k < SI_WORDS; k++)
        if (h[k] < 0) return fail("fpl_state_merge: image %d: header word %d is negative (%lld)", i, k, (long long)h[k]);
    for (int k = SI_KEEP; k <= SI_MERGED; k++)
        if (h[k] > 1) return fail("fpl_state_merge: image %d: header word %d is a flag, not %lld", i, k, (long long)h[k]);
    const int64_t A = h[SI_ADAPTER_BYTES], cw = h[SI_COUNTER_WORDS], rows = h[SI_ROWS], n0 = h[SI_LIST0], n1 = h[SI_LIST1];
    if (rows != std::max(h[SI_USED], h[SI_REDUCED]))
        return fail("fpl_state_merge: image %d: rows %lld != max(used_cycles, reduced_rows)", i, (long long)rows);
    // each length within the image before any product of them: the sum below cannot overflow
    if (A > n || cw > n / 8 || rows > n / 256 || n0 > n / 8 || n1 > n / 8 ||
        FPL_STATE_HEADER_BYTES + A + 8 * (2 * FPL_STATS_WORDS(rows) + cw + n0 + n1) != n)
        return fail("fpl_state_merge: image %d: the section lengths do not add up to its %lld bytes", i, (long long)n);
    if (memcmp(p + kOptAt, reinterpret_cast<const char*>(&c->P.opt) + kOptBegin, kOptEnd - kOptBegin))
        return fail("fpl_state_merge: image %d was created with other options than the destination", i);
    // A == dst's adapter section and the sum above hold: walking dst's lengths stays inside the section
    if (h[SI_N_ADAPTERS] != (int64_t)c->adapter_str.size() || A != adapter_section_bytes(c->adapter_str))
        return fail("fpl_state_merge: image %d was created with another adapter list than the destination", i);
    const uint8_t* q = p + FPL_STATE_HEADER_BYTES;
    for (const std::string& s : c->adapter_str) {
        int64_t len;
        memcpy(&len, q, 8);
        if (len != (int64_t)s.size() || memcmp(q + 8, s.data(), s.size()))
            return fail("fpl_state_merge: image %d was created with another adapter list than the destination", i);
        q += 8 + pad8(len);
    }
    if (cw != c->counter_words)
        return fail("fpl_state_merge: image %d has %lld counter words, the destination %lld", i, (long long)cw,
                    (long long)c->counter_words);
    im.rows = rows; im.used = h[SI_USED]; im.reduced = h[SI_REDUCED];
    im.n[0] = n0; im.n[1] = n1;
    im.complete = h[SI_COMPLETE] != 0; im.merged = h[SI_MERGED] != 0;
    im.stats = q;
    im.list[0] = q + 8 * (2 * FPL_STATS_WORDS(rows) + cw);
    im.list[1] = im.list[0] + 8 * n0;
    return 0;
}

}  // namespace

extern "C" int fpl_state_export(fpl_ctx* c, uint8_t* out, int64_t cap, int64_t* n_bytes) {
    g_err[0] = 0;
    if (!c || !n_bytes) return fail("fpl_state_export: null argument");
    const FplLists& L = c->lists;
    const int64_t rows = std::max(c->used_cycles, c->reduced_rows), sw = FPL_STATS_WORDS(rows), cw = c->counter_words;
    const int64_t A = adapter_section_bytes(c->adapter_str);
    const int64_t total = FPL_STATE_HEADER_BYTES + A + 8 * (2 * sw + cw + L.n[0] + L.n[1]);
    *n_bytes = total;
    if (!out || cap < total) return 1;
    CK(cudaSetDevice(c->device));
    memset(out, 0, (size_t)(FPL_STATE_HEADER_BYTES + A));
    const int64_t h[SI_WORDS] = {(int64_t)FPL_STATE_MAGIC, FPL_STATE_FORMAT, FPL_ABI_VERSION, total, (int64_t)c->adapter_str.size(), A, cw,
                                 rows, c->used_cycles, c->reduced_rows, L.keep, L.complete, L.merged, L.n[0], L.n[1]};
    memcpy(out, h, sizeof(h));
    memcpy(out + kOptAt, reinterpret_cast<const char*>(&c->P.opt) + kOptBegin, kOptEnd - kOptBegin);
    uint8_t* q = out + FPL_STATE_HEADER_BYTES;
    for (const std::string& s : c->adapter_str) {
        const int64_t len = (int64_t)s.size();
        memcpy(q, &len, 8);
        memcpy(q + 8, s.data(), s.size());
        q += 8 + pad8(len);
    }
    const size_t W = sizeof(unsigned long long);
    for (int w = 0; w < 2; w++) {
        uint8_t* blk = q + W * sw * w;
        if (rows)       // rows b*C + c of the block go to b*rows + c
            CK(cudaMemcpy2DAsync(blk, W * rows, c->d_stats[w], W * c->C, W * rows, 16, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(blk + W * 16 * rows, c->d_stats[w] + 16 * c->C, W * FPL_STATS_TAIL, cudaMemcpyDeviceToHost, c->stream));
    }
    q += W * 2 * sw;
    CK(cudaMemcpyAsync(q, c->d_counters, W * cw, cudaMemcpyDeviceToHost, c->stream));
    q += W * cw;
    for (int w = 0; w < 2; w++) {
        if (L.n[w]) CK(cudaMemcpyAsync(q, L.d[w], sizeof(HtmlEntry) * L.n[w], cudaMemcpyDeviceToHost, c->stream));
        q += sizeof(HtmlEntry) * L.n[w];
    }
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    return 0;
}

extern "C" int fpl_state_merge(fpl_ctx* c, const uint8_t* const* images, const int64_t* n_bytes, int n_images) {
    g_err[0] = 0;
    if (!c) return fail("fpl_state_merge: null destination context");
    if (n_images < 0) return fail("fpl_state_merge: negative number of images (%d)", n_images);
    if (n_images > 0 && (!images || !n_bytes)) return fail("fpl_state_merge: null image or size list");
    std::vector<StateImage> im((size_t)n_images);
    for (int k = 0; k < n_images; k++)
        if (parse_image(c, k, images[k], n_bytes[k], im[k])) return -1;
    if (n_images == 0) return 0;
    CK(cudaSetDevice(c->device));
    FplLists& L = c->lists;
    const int64_t cw = c->counter_words;
    int64_t rows = 0, used = c->used_cycles, reduced = c->reduced_rows, total[2] = {L.n[0], L.n[1]}, words = 0;
    bool complete = L.complete, merged = L.merged;
    for (const StateImage& s : im) {
        rows = std::max(rows, s.rows);
        used = std::max(used, s.used);
        reduced = std::max(reduced, s.reduced);
        complete = complete && s.complete;
        merged = merged || s.merged;
        for (int w = 0; w < 2; w++) total[w] += s.n[w];
        words += 2 * FPL_STATS_WORDS(s.rows) + cw;
    }
    // the capacities first, as fpl_merge_stats grows them
    if (reserve_cycles(c, rows)) return -1;
    if (L.keep && (grow_list(c, 0, total[0]) || grow_list(c, 1, total[1]))) return -1;
    CK(c->d_state_stage.grow(words));
    CK(c->d_merge.grow(n_images));
    std::vector<MergeSrc> tab((size_t)n_images);
    int64_t at = 0;
    for (int k = 0; k < n_images; k++) {
        const int64_t sw = FPL_STATS_WORDS(im[k].rows);
        unsigned long long* d = c->d_state_stage + at;
        CK(cudaMemcpyAsync(d, im[k].stats, sizeof(unsigned long long) * (2 * sw + cw), cudaMemcpyHostToDevice, c->stream));
        // the compact blocks as a source of capacity rows: k_merge_stats reads b * rows + c for c < rows, the tail at 16 * rows
        tab[k] = MergeSrc{{d, d + sw}, d + 2 * sw, im[k].rows, im[k].rows};
        at += 2 * sw + cw;
    }
    CK(cudaMemcpyAsync(c->d_merge, tab.data(), sizeof(MergeSrc) * n_images, cudaMemcpyHostToDevice, c->stream));
    {
        Timed t(c, K_MERGE_STATS);
        launch_merge_stats(c->d_stats[0], c->d_stats[1], c->d_counters, c->C, rows, cw, c->d_merge, n_images, c->stream);
    }
    if (L.keep) {
        for (int w = 0; w < 2; w++)
            for (const StateImage& s : im) {
                if (s.n[w])
                    CK(cudaMemcpyAsync(L.d[w] + L.n[w], s.list[w], sizeof(HtmlEntry) * s.n[w], cudaMemcpyHostToDevice, c->stream));
                L.n[w] += s.n[w];
            }
    } else {
        complete = false;                     // the images' entries were not taken, as in a call with capture off
    }
    c->used_cycles = used; c->reduced_rows = reduced;
    L.complete = complete; L.merged = merged;
    c->rep.built = false; c->html.built = false;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->stream));
    collect_times(c);
    return 0;
}
