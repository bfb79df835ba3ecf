#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fplgpu.h"
#include "fpl_buf.h"

#define FPL_SLOT_ALIGN 128
#define FPL_INGEST_FIRST_BYTES (1 << 20)   // first capacity of the ingest buffers (a FASTQ chunk is megabytes)

struct FplIngest {
    DevBuf<uint8_t> d_text;
    DevBuf<int64_t> d_nl;
    DevBuf<fpl_fastq_record> d_rec;
    DevBuf<int32_t> d_lens;
    DevBuf<int64_t> d_slots;
    DevBuf<int64_t> d_offsets;
    DevBuf<uint8_t> d_tmp;
    DevBuf<unsigned long long> d_misc;           // [0] newline count, [1] cub's count, [2] first bad record, [4] CR flag
    int64_t n_nl = 0, packed_bytes = 0;
};

// returns 0 ok, 1 = not the strict layout (caller falls back to the reference reader), -1 error (message in err)
int fpl_ingest_index(FplIngest* g, const uint8_t* h_text, int64_t n, int is_last, cudaStream_t s, int64_t* n_records,
                     int64_t* consumed, char* err, size_t errlen);
int fpl_ingest_pack(FplIngest* g, int64_t nrec, uint8_t* d_seq, uint8_t* d_qual, cudaStream_t s, char* err, size_t errlen);
