// pb_filter_spec.h — plan-time specialised instantiations of pb_filter_kernel (pb_filter_spec.cu), reached through a small
// dispatch table so that pb_engine.cu does not have to compile them.  Not part of the public ABI.
#pragma once
#include <cuda_runtime.h>
struct DevQuery;
// PK: 0 = dictId range, 1 = IN / NOT IN membership LUT in shared memory.  RW: 0 = write the match list, 2 / 4 / 8 = the
// fused variant that aggregates the survivors of its candidate round from row groups of RW words (DevQuery::row_segs)
bool pb_filter_spec_available(int width, int pred_kind);
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) on the current device + resident CTAs per SM for `smem` bytes
cudaError_t pb_filter_spec_prepare(int width, int pred_kind, int rw, size_t smem, int* ctas_per_sm);
cudaError_t pb_filter_spec_launch(int width, int pred_kind, int rw, int grid, size_t smem, cudaStream_t st, const DevQuery* q);
