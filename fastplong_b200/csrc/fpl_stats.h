// fpl_stats.cu's launchers, each adding the kernels it enqueues to its last argument, and the descriptors they take.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>
#include "fpl_buf.h"
#include "fpl_device.cuh"

// Workspace of launch_cycle_stats (the length-sorted segment list), owned by a context: one stream, one workspace.

struct SegD;
struct CycleWs {
    DevBuf<uint8_t> tmp;
    DevBuf<uint32_t> k_in, k_out;
    DevBuf<int32_t> v_in, v_out;
    DevBuf<SegD> sorted;
    int64_t cap = 0;                    // segments every list above holds
};

// fpl_report_json: the two Stats blocks whose curves k_report_sizes / k_report_text print
struct ReportCurves {
    const unsigned long long* blk[2];   // pre, post (FPL_STATS_WORDS(C) each)
    int64_t C;
    int64_t T[2];                       // total_cycles of each block
    int64_t shift[22];                  // curve j's text starts shift[j] bytes of frame behind its place in the scanned sizes
    int is_rna;
};

// fpl_merge_stats: one source context's accumulators, as k_merge_stats reads them
struct MergeSrc {
    const unsigned long long* blk[2];   // pre, post (FPL_STATS_WORDS(C) each)
    const unsigned long long* cnt;      // counter block (the destination's counter_words)
    int64_t C;                          // the source's capacity
    int64_t rows;                       // rows [0, rows) of its per-cycle arrays may be non-zero
};
// k_merge_stats: rows [0, rows) and the tail of dst's two blocks (capacity C), and its cnt_words counters, += each of the n_src
// sources' (a device table), in table order; one launch
void launch_merge_stats(unsigned long long* pre, unsigned long long* post, unsigned long long* cnt, int64_t C, int64_t rows,
                        int64_t cnt_words, const MergeSrc* src, int n_src, cudaStream_t stream, int& launched);

// fpl_keep_read_lists: one entry per read of a Stats block, in the order Stats::statRead saw them.  A post-filter slot that
// holds no output read (a failing or missing segment) has len = -1; the report drops it.
struct HtmlEntry {
    int32_t len;
    int32_t med;                        // the read's median quality char
};

#define HTML_CHUNK 2048                 // list entries per warp of the grouping by median
#define HTML_BINS 130                   // its bins: medians 0..127, 128: empty reads, 129: no output read

// fpl_report_html: the device-printed lists of the report, in text order — per Stats block the density x and y lists, then
// the 5 quality and the 6 content curves of each block — between HTML_SEGS + 1 host-built frame pieces
#define HTML_SEGS 26
struct HtmlText {
    int64_t start[HTML_SEGS + 1];       // index of each segment's first value; start[HTML_SEGS] = all values
    int64_t shift[HTML_SEGS];           // frame bytes in front of the segment
    int kind[HTML_SEGS];                // 0: density x (median - 33), 1: density y (length), 2: down-sampled curve value
    int blk[HTML_SEGS];                 // Stats block
    int64_t base[HTML_SEGS];            // kind 2: index of the segment's first value in sums[blk]
    const HtmlEntry* grp[2];            // each block's list grouped by median
    int64_t nonempty[2];                // entries of grp that are density pairs (reads with bases); the rest print 0
    const double* sums[2];              // curve values
    const long long* x[2];              // each block's x list: range i is [x[i - 1], x[i]), x[-1] = 0
};

int launch_cycle_stats(CycleWs*, const uint8_t*, const uint8_t*, const StatSeg*, int64_t, int64_t, unsigned long long*, int64_t,
                       bool, unsigned long long*, bool, const StatSeg*, unsigned long long*, const StatSeg*, cudaStream_t, int&);
void launch_kmer_fix(const DevBatch&, const fpl_read_result*, unsigned long long*, cudaStream_t, int&);
void launch_read_qual(const DevBatch&, unsigned long long*, unsigned long long*, int64_t, fpl_read_result*, bool, cudaStream_t, int&);
void launch_read_qual_exc(const DevBatch&, const ReadState*, const int32_t*, const int*, unsigned long long*, unsigned long long*, int64_t,
                          fpl_read_result*, cudaStream_t, int&);
void launch_qhist_fold(const unsigned long long*, int, unsigned long long*, unsigned long long*, int64_t, cudaStream_t, int&);
void launch_make_preseg(const DevBatch&, StatSeg*, cudaStream_t, int&);
void launch_report_cycles(const unsigned long long*, const unsigned long long*, int64_t, unsigned long long*, cudaStream_t, int&);
void launch_report_sizes(const ReportCurves&, int64_t*, cudaStream_t, int&);
void launch_report_text(const ReportCurves&, const int64_t*, const uint8_t*, const int64_t*, const int64_t*, int, uint8_t*, cudaStream_t,
                        int&);
void launch_html_capture(const fpl_read_result*, const int32_t*, int64_t, const fpl_segment*, int64_t, HtmlEntry*, HtmlEntry*, cudaStream_t,
                         int&);
void launch_html_hist(const HtmlEntry*, int64_t, int64_t, long long*, cudaStream_t, int&);
void launch_html_scatter(const HtmlEntry*, int64_t, int64_t, const long long*, HtmlEntry*, cudaStream_t, int&);
void launch_html_lenhist(const HtmlEntry*, int64_t, unsigned long long*, cudaStream_t, int&);
void launch_html_lenprod(const unsigned long long*, int64_t, long long*, cudaStream_t, int&);
void launch_html_lensearch(const unsigned long long*, const long long*, const long long*, const long long*, int64_t, long long,
                           unsigned long long, int*, cudaStream_t, int&);
void launch_html_bins(const unsigned long long*, int64_t, int64_t, unsigned long long*, cudaStream_t, int&);
void launch_html_values(const unsigned long long*, int64_t, int64_t, int, double*, cudaStream_t, int&);
void launch_html_sums(const double*, int64_t, const long long*, int64_t, double*, cudaStream_t, int&);
void launch_html_sizes(const HtmlText&, int64_t*, cudaStream_t, int&);
void launch_html_text(const HtmlText&, const int64_t*, const uint8_t*, const int64_t*, const int64_t*, int, uint8_t*, cudaStream_t, int&);
