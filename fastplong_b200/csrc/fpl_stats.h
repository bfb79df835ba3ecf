// Workspace of launch_cycle_stats (the length-sorted segment list), owned by a context: one stream, one workspace.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

struct CycleWs {
    void* tmp = nullptr; size_t tmp_bytes = 0;
    uint32_t *k_in = nullptr, *k_out = nullptr;
    int32_t *v_in = nullptr, *v_out = nullptr;
    void* sorted = nullptr;
    int64_t cap = 0;
};
void fpl_cycle_ws_free(CycleWs* ws);

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
                        int64_t cnt_words, const MergeSrc* src, int n_src, cudaStream_t stream);

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
