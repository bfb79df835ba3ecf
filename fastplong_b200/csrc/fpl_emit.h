#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fplgpu.h"
#include "fpl_buf.h"

// Device half of SURVEY §8f row 2 (output assembly): state of fpl_emit_fastq_host.
struct FplEmit {
    DevBuf<int64_t> d_size;             // [0, n]: --out bytes of read r; [n+1, 2n+1]: --failed_out bytes
    DevBuf<int64_t> d_off;              // exclusive sums of the two halves
    DevBuf<uint8_t> d_out, d_failed;
    DevBuf<uint8_t> d_tmp;
    int64_t out_bytes = 0, failed_bytes = 0;
    bool built = false, with_failed = false;
};

// State of fpl_emit_batch_device: the sizes of both output batches, built once per fpl_process_* call.
struct FplBatchEmit {
    DevBuf<int64_t> d_cnt;              // 4 x (n+1): reads / slot bytes per read, for out and for failed
    DevBuf<int64_t> d_off;              // their exclusive sum
    DevBuf<uint8_t> d_tmp;
    int64_t n_out = 0, out_bytes = 0, n_failed = 0, failed_bytes = 0;
    bool built = false;
};

// What the output is cut from: the per-read results, (--mask / --break) the list of output reads with its per-read ranges
// and the masked copy of the packed sequence buffer, the packed slots of the reads, and either the FASTQ chunk with its
// record table (fpl_emit_fastq_host) or the packed batch itself (fpl_emit_batch_device).
struct EmitSource {
    const fpl_read_result* res;
    int64_t n_reads;
    const fpl_segment* segs;        // null in the plain mode (the records' inline segments are the output reads)
    const int32_t* seg_off;         // segs of read r: [seg_off[2r], seg_off[2r+2])
    const uint8_t* mseq;            // masked bases in the packed layout (null: nothing was masked)
    const int64_t* offsets;         // packed-layout slot of read r
    const uint8_t* text;            // FASTQ text sink: the chunk and its record table
    const fpl_fastq_record* rec;
    const uint8_t* seq;             // batch sink: the packed batch
    const uint8_t* qual;
};

// One destination batch of fpl_emit_batch_device (device pointers; seq == null: not written)
struct EmitBatchOut {
    uint8_t* seq;
    uint8_t* qual;
    int64_t* offsets;
    int32_t* lens;
    fpl_segment* segs;              // may be null
};

// launched += the kernels it enqueued, also when it then fails; so do launch_emit_batch_*
int fpl_emit_build(FplEmit* e, const EmitSource& src, bool want_failed, cudaStream_t s, int& launched, char* err, size_t errlen);

// fpl_emit_batch_device: reserve -> launch_emit_batch_sizes -> scan (synchronous: the totals come to the host) -> copy
int fpl_emit_batch_reserve(FplBatchEmit* e, int64_t n_reads, char* err, size_t errlen);
void launch_emit_batch_sizes(const EmitSource& src, int64_t* cnt, cudaStream_t s, int& launched);
int fpl_emit_batch_scan(FplBatchEmit* e, int64_t n_reads, cudaStream_t s, char* err, size_t errlen);
void launch_emit_batch_copy(const EmitSource& src, const int64_t* off, const EmitBatchOut& out, const EmitBatchOut& failed,
                            cudaStream_t s, int& launched);
