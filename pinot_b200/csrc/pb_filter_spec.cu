// pb_filter_spec.cu — the specialised instantiations of pb_filter_kernel<2, 4, W, PK, RW> (see the template's comment in
// pb_device.cuh): one small kernel per bit width 1..20 that is not a byte multiple and per predicate kind, each also as the
// fused variant for row groups of 2, 4 and 8 words.  The GPU analogue of FixedBitIntReader's one-class-per-width readers
// (SEGL/io/reader/impl/FixedBitIntReader.java:121-146), taken one step further: the predicate is compiled in as well.
#include "pb_device.cuh"
#include "pb_filter_spec.h"

#define PB_SPEC_WIDTHS(X) X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(17) X(18) X(19) X(20)

template <int W, int PK>
static const void* spec_kernel_of(int rw) {
  switch (rw) {
    case 0: return (const void*)pb_filter_kernel<2, 4, W, PK>;
    case 2: return (const void*)pb_filter_kernel<2, 4, W, PK, 2>;
    case 4: return (const void*)pb_filter_kernel<2, 4, W, PK, 4>;
    case 8: return (const void*)pb_filter_kernel<2, 4, W, PK, 8>;
    default: return nullptr;
  }
}

static const void* spec_kernel(int width, int pred_kind, int rw) {
  if (pred_kind != 0 && pred_kind != 1) return nullptr;
  switch (width) {
#define X(W) case W: return pred_kind == 0 ? spec_kernel_of<W, 0>(rw) : spec_kernel_of<W, 1>(rw);
    PB_SPEC_WIDTHS(X)
#undef X
    default: return nullptr;
  }
}

bool pb_filter_spec_available(int width, int pred_kind) { return spec_kernel(width, pred_kind, 0) != nullptr; }

cudaError_t pb_filter_spec_prepare(int width, int pred_kind, int rw, size_t smem, int* ctas_per_sm) {
  const void* k = spec_kernel(width, pred_kind, rw);
  if (!k) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) return e;
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, k, PB_NTHREADS, smem);
}

cudaError_t pb_filter_spec_launch(int width, int pred_kind, int rw, int grid, size_t smem, cudaStream_t st, const DevQuery* q) {
  const void* k = spec_kernel(width, pred_kind, rw);
  if (!k) return cudaErrorInvalidValue;
  void* args[] = {const_cast<DevQuery*>(q)};
  return cudaLaunchKernel(k, dim3(grid), dim3(PB_NTHREADS), args, smem, st);
}
