#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
struct DevBatch;
struct ReadState;
#define QH_STRIPES 128      // stripes of k_scan_jit's histogram sums (CTA r: r % QH_STRIPES), defined in front of its source too
// qhist: the kernel also counts the quality histograms (version 2 built with doQhist; see fpl_scan_jit2_src.h)
struct FplJitKernel { void* fn = nullptr; bool qhist = false; };
int fpl_jit_build_scan(int device, const char* a0, const char* a1, bool doAdapters, bool doCounts, bool doCplx, bool doQhist,
                       int qq, FplJitKernel* out, char* err, size_t errlen);
// launched += the kernels it enqueued (none for an empty batch); -1 when the launch failed
int fpl_jit_launch_scan(const FplJitKernel* k, const DevBatch& b, ReadState* st, cudaStream_t stream, int& launched);
