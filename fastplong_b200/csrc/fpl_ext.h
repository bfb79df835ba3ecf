#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fpl_device.cuh"
#include "fpl_buf.h"

struct FplExt {
    DevBuf<int32_t> d_cnt;              // pieces per initial segment (2 per read)
    DevBuf<int32_t> d_off;
    DevBuf<fpl_segment> d_segs;
    DevBuf<StatSeg> d_stat;
    DevBuf<int32_t> d_rcnt;             // mask regions per piece
    DevBuf<int32_t> d_roff;
    DevBuf<fpl_region> d_regs;
    DevBuf<uint8_t> d_mseq;             // private, masked copy of the sequence buffer
    DevBuf<uint8_t> d_tmp;
    int64_t n_segs = 0, n_regs = 0;
};

int fpl_ext_run(FplExt* x, const DevParams& P, const DevBatch& b, int64_t n_bytes, fpl_read_result* res,
                unsigned long long* counters, unsigned long long* stats_post, int64_t C, const uint8_t** fseq_out,
                cudaStream_t s, char* err, size_t errlen);
