// The fixed summation order of the BatchNorm per-CTA partial rows, shared by combine_partials_kernel (bn_act.cu) and the
// synchronised exchange (sync_bn.cu), so that a rank's local sums are the same bits on both paths; and the BatchNorm
// backward apply arithmetic, shared by bn_act.cu and the fused data-gradient GEMM (gemm_bnstats.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "comm_types.h"

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

// BatchNorm parameters and their gradients: fp32, bf16 or fp16 (dt: comm_types.h DType)
__device__ __forceinline__ float ld_w(const void* p, int dt, int i) {
  switch (dt) {
    case kF32: return reinterpret_cast<const float*>(p)[i];
    case kBF16: return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
    default: return __half2float(reinterpret_cast<const __half*>(p)[i]);
  }
}
__device__ __forceinline__ void st_w(void* p, int dt, int i, float v) {
  switch (dt) {
    case kF32: reinterpret_cast<float*>(p)[i] = v; break;
    case kBF16: reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v); break;
    default: reinterpret_cast<__half*>(p)[i] = __float2half_rn(v); break;
  }
}

// BatchNorm backward apply, dx = A*dz + B*x + D, shared by bn_bwd_apply_body (bn_act.cu) and the fused data-gradient GEMM
// (gemm_bnstats.cu), so that both write the same dx bits.  Every rounding is spelled out, because the two kernels must
// not be left to contract into FMAs on their own.  The roundings are the ones nvcc chose for bn_bwd_apply before they
// were spelled out, so its results did not change: D fuses its first product, except in the eighth (last unrolled) channel
// of a group of eight and in every channel of the synchronised variant, where it fuses B*mean (fuse_mean).
//   A = gamma*invstd,  B = -A*invstd*sum(dz*xhat)/m,  D = -A*sum(dz)/m - B*mean
struct BnBwdCoef { float a, b, d; };
__device__ __forceinline__ BnBwdCoef bn_bwd_coef(float gamma, float mean, float invstd, float sdz, float sdzx, float inv_m,
                                                 bool fuse_mean) {
  BnBwdCoef k;
  k.a = __fmul_rn(gamma, invstd);
  k.b = -__fmul_rn(__fmul_rn(__fmul_rn(k.a, invstd), sdzx), inv_m);
  k.d = fuse_mean ? __fmaf_rn(-k.b, mean, -__fmul_rn(__fmul_rn(k.a, sdz), inv_m))
                  : __fmaf_rn(-__fmul_rn(k.a, sdz), inv_m, -__fmul_rn(k.b, mean));
  return k;
}
__device__ __forceinline__ float bn_bwd_dx(float a, float b, float d, float dz, float x) {
  return __fadd_rn(__fmaf_rn(a, dz, __fmul_rn(b, x)), d);
}

}  // namespace ptd
