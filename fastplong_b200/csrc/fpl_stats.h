// Workspace of launch_cycle_stats (the length-sorted segment list), owned by a context: one stream, one workspace.
#pragma once
#include <cstddef>
#include <cstdint>

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
