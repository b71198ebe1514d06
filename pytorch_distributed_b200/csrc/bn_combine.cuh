// The fixed summation order of the BatchNorm per-CTA partial rows, shared by combine_partials_kernel (bn_act.cu) and the
// synchronised exchange (sync_bn.cu), so that a rank's local sums are the same bits on both paths.
#pragma once
#include <cuda_runtime.h>

namespace ptd {

// Column i of part[nblocks][n], summed by a 1024-thread CTA that covers 32 columns: thread (ty, tx) adds rows ty, ty + 32,
// ... of column i (combine_slice, stored to sm[ty][tx]), then, after a __syncthreads(), thread (0, tx) adds the 32 slice
// sums in order (combine_fold).
__device__ __forceinline__ float combine_slice(const float* __restrict__ part, int nblocks, int n, int i, int ty) {
  float s = 0.f;
  if (i < n)
    for (int b = ty; b < nblocks; b += 32) s += part[(size_t)b * n + i];
  return s;
}
__device__ __forceinline__ float combine_fold(const float (&sm)[32][33], int tx) {
  float t = 0.f;
  for (int k = 0; k < 32; ++k) t += sm[k][tx];
  return t;
}

}  // namespace ptd
