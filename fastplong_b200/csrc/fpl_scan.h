// The launchers of fpl_trim.cu, fpl_scan.cu and fpl_scan_fast.cu; each adds the kernels it enqueues to its last argument.
#pragma once
#include "fpl_device.cuh"
#include "fpl_scanplan.h"

void launch_trim(const DevParams&, const DevBatch&, ReadState*, fpl_read_result*, unsigned long long*, cudaStream_t, int&);
void launch_scan(const DevParams&, const DevBatch&, ReadState*, cudaStream_t, int&);
void launch_scan_fast(const DevParams&, const ScanPlan&, const DevBatch&, ReadState*, cudaStream_t, int&);
void launch_final(const DevParams&, const DevBatch&, const ReadState*, fpl_read_result*, StatSeg*, int32_t*, int*, cudaStream_t, int&);
void launch_count(const fpl_read_result*, int64_t, unsigned long long*, bool, const int32_t*, unsigned long long*, unsigned long long*,
                  int64_t, cudaStream_t, int&);
