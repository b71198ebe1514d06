// Per-sample input augmentation of a uint8 batch, fused with the normalise / cast / layout pass of normalize_kernel
// (data_ops.cu): torchvision's transforms.v2.TrivialAugmentWide or AutoAugment(interpolation=BILINEAR) on the uint8 image,
// then the normalisation, then RandomErasing(value=0) on the normalised tensor.
//
//  augment_normalize : one CTA per sample.  An op that needs a per-image statistic first reduces it inside the CTA in
//                      integers (no float atomics, so the result does not depend on the order of the threads), then one
//                      streaming pass computes each output pixel's three uint8 values, rounds them as torchvision does,
//                      normalises them with the single FMA of normalize_nhwc / resample_normalize and zeroes the erase box
//                      in the same store.  Geometric ops gather their four taps from global memory (the sample, 150 KB
//                      at 224^2, stays in L2).
//                      A two-op table (AutoAugment's sub-policies) takes two launches: augment_stage_kernel writes op A's
//                      uint8 output into a scratch batch, then augment_chain_kernel runs op B on it as above (on the
//                      source for a row whose op A is Identity, i.e. not applied).  Measured on the H100, this beat one
//                      pass with op A's output in shared memory (3 H W bytes per CTA leave one CTA per SM).
//
// The host draws every sample's ops and magnitudes and encodes what the kernel needs into a row of prm float32
// (pytorch_distributed_b200/ops/augment.py), [n, kAugPrm] for one op per sample or [n, kAugChainPrm] for two:
//   prm[0]      op A's kernel code (AugOp below; anything else copies the image)
//   prm[1..6]   op A's parameters (below)
//   prm[7]      1: erase rows [prm[8], prm[8] + prm[10]) x columns [prm[9], prm[9] + prm[11])
//   prm[12..15] not read here (op A's index into op_names() + ("Invert",) and its signed magnitude, for the CPU reference)
//   prm[16]     two-op rows only: op B's kernel code, applied to op A's output
//   prm[17..22] op B's parameters
//   prm[23..31] not read here (op B's index and signed magnitude in prm[23], prm[24], for the CPU reference)
// kInvert exists in two-op rows only: in a one-op row it is an unknown code, and the one-op kernel is unchanged by it.
//
// Float order.  Every rounding torchvision's CPU kernels make is written out with __fmul_rn / __fadd_rn / __fmaf_rn /
// __fdiv_rn (the extension builds with --use_fast_math, which would contract products into FMAs and make `/` approximate):
//   grayscale   fma(b, 0.114, fma(g, 0.587, r * 0.2989)), floored     (r.mul(.2989).add_(g, alpha=.587).add_(b, alpha=.114))
//   _blend      fma(other, 1 - ratio, x * ratio), clamped to [0, 255] and truncated
//   Sharpness   the 3x3 blur (1 1 1 / 1 5 1 / 1 1 1) / 13 rounded half-to-even: it is computed exactly in integers, since
//               (8-neighbour sum + 5 centre) / 13 is never within 1/26 of a half, the rounding of any float order gives
//               the same integer; then fma(blur - x, 1 - factor, x); the one-pixel border is left as it is
//   affine grid (x * t0 + y * t1) + t2 of the pre-scaled inverse matrix, ix = (gx + 1) * W/2 - 0.5, bilinear weights
//               and the sum nw + ne + sw + se each rounded, then round half-to-even (_apply_grid_transform)
// Contrast's mean is sum(floor(gray)) / (H W).  The sum is an exact integer; torch sums the same floats in float32, which
// is exact in any order while 255 H W < 2^24, i.e. H W <= kAugMaxPixels: the launcher refuses larger images.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {
namespace {

enum AugOp : int {
  kIdentity = 0,
  kAffine = 1,       // prm[1..6]: t0..t5, the inverse matrix pre-divided by (W/2, H/2) as _affine_grid does
  kRot90 = 2,        // prm[1]: k = 1 or 3 (torch.rot90 over (H, W); square images only)
  kBrightness = 3,   // prm[1]: factor
  kColor = 4,        // prm[1]: ratio, prm[2]: fp32(1 - ratio)          (adjust_saturation)
  kContrast = 5,     // prm[1]: ratio, prm[2]: fp32(1 - ratio)
  kSharpness = 6,    // prm[1]: fp32(1 - factor)
  kPosterize = 7,    // prm[1]: bit mask
  kSolarize = 8,     // prm[1]: fp32 threshold
  kAutoContrast = 9,
  kEqualize = 10,
  kInvert = 11,      // 255 - v (two-op rows only)
};

constexpr int kColB = 16;   // first column of op B in a two-op row

constexpr int kThreads = 512;

__device__ __forceinline__ float gray_floor(float r, float g, float b) {
  return floorf(__fmaf_rn(b, 0.114f, __fmaf_rn(g, 0.587f, __fmul_rn(r, 0.2989f))));
}

// clamp to [0, 255], then the float -> uint8 conversion (truncation)
__device__ __forceinline__ int trunc_u8(float v) { return (int)fminf(255.f, fmaxf(0.f, v)); }

__device__ __forceinline__ int blend(float x, float other, float ratio, float alpha) {
  return trunc_u8(__fmaf_rn(other, alpha, __fmul_rn(x, ratio)));
}

// bilinear sample of plane p at (ix, iy) with zero padding (grid_sample, align_corners=False), rounded half-to-even
__device__ __forceinline__ int bilinear(const uint8_t* p, int H, int W, float ix, float iy) {
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float w = __fsub_rn(ix, x0), e = __fsub_rn(1.f, w);
  const float n = __fsub_rn(iy, y0), s = __fsub_rn(1.f, n);
  const int xi = (int)x0, yi = (int)y0;
  auto at = [&](int y, int x) -> float { return (x >= 0 && x < W && y >= 0 && y < H) ? (float)p[(size_t)y * W + x] : 0.f; };
  float v = __fmul_rn(at(yi, xi), __fmul_rn(s, e));
  v = __fadd_rn(v, __fmul_rn(at(yi, xi + 1), __fmul_rn(s, w)));
  v = __fadd_rn(v, __fmul_rn(at(yi + 1, xi), __fmul_rn(n, e)));
  v = __fadd_rn(v, __fmul_rn(at(yi + 1, xi + 1), __fmul_rn(n, w)));
  return (int)fminf(255.f, fmaxf(0.f, rintf(v)));
}

// One op over one sample: its per-image statistic (integer, order-free), then one streaming pass over the output pixels.
// src + k: the sample's three planes; q: the op's columns (q[0] kernel code, q[1..6] parameters);
// row: the sample's row (erase box).  kChain: the two-op kernel, which also knows kInvert.  kStage: write the op's uint8
// result to stage (the sample's three planes in the scratch batch) instead of erasing, normalising and storing it.
template <typename Out, bool NHWC_OUT, bool kChain, bool kStage>
__device__ __forceinline__ void apply_op(const uint8_t* src, int k, const float* q, const float* row, Out* dst, uint8_t* stage,
                                         int s, int H, int W, const float* na, const float* nb, int (*hist)[256], int (*lut)[256],
                                         int* red) {
  const int HW = H * W;
  const size_t plane = (size_t)HW;
  const uint8_t* img = src + (size_t)k * 3 * plane;
  const int op = (int)q[0];
  const float p1 = q[1], p2 = q[2];
  const float sa[3] = {na[0], na[1], na[2]}, sb[3] = {nb[0], nb[1], nb[2]};
  const bool erase = row[7] != 0.f;
  const int ei = (int)row[8], ej = (int)row[9], eh = (int)row[10], ew = (int)row[11];

  // ---- per-image statistics (integer, order-free)
  if (op == kContrast || op == kAutoContrast || op == kEqualize) {
    for (int t = threadIdx.x; t < 3 * 256; t += kThreads) (&hist[0][0])[t] = 0;
    const int init = op == kAutoContrast ? 255 : 0;       // Contrast: acc[0]; AutoContrast: min in acc[0..2], max in acc[3..5]
    if (threadIdx.x < 6) red[threadIdx.x] = threadIdx.x < 3 ? init : 0;
    __syncthreads();
    int acc[6] = {init, init, init, 0, 0, 0};
    for (int p = threadIdx.x; p < HW; p += kThreads) {
      const int r = img[p], g = img[plane + p], b = img[2 * plane + p];
      if (op == kContrast) {
        acc[0] += (int)gray_floor((float)r, (float)g, (float)b);
      } else if (op == kAutoContrast) {
        acc[0] = min(acc[0], r); acc[1] = min(acc[1], g); acc[2] = min(acc[2], b);
        acc[3] = max(acc[3], r); acc[4] = max(acc[4], g); acc[5] = max(acc[5], b);
      } else {
        atomicAdd(&hist[0][r], 1);
        atomicAdd(&hist[1][g], 1);
        atomicAdd(&hist[2][b], 1);
      }
    }
    if (op == kContrast) {
      atomicAdd(&red[0], acc[0]);
    } else if (op == kAutoContrast) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { atomicMin(&red[c], acc[c]); atomicMax(&red[3 + c], acc[3 + c]); }
    }
    __syncthreads();
    if (op == kEqualize && threadIdx.x < 3) {  // torchvision's (PIL's) LUT, one channel per thread
      const int c = threadIdx.x;
      int last = 255;
      while (last > 0 && hist[c][last] == 0) --last;       // the last non-empty bin: the first maximum of the cumulative sum
      const int step = (HW - hist[c][last]) / 255;
      int cum = 0;
      lut[c][0] = 0;
      for (int k = 1; k < 256; ++k) {                      // step == 0: the channel is returned as it is (identity LUT)
        cum += hist[c][k - 1];
        lut[c][k] = step == 0 ? k : min(255, (cum + step / 2) / step);
      }
    }
    __syncthreads();
  }
  // Contrast's mean: the float32 sum (exact, see the header) over the pixel count, correctly rounded
  const float mean = op == kContrast ? __fdiv_rn((float)red[0], (float)HW) : 0.f;
  float lo[3], inv[3];
  if (op == kAutoContrast) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const bool flat = red[c] == red[3 + c];
      lo[c] = flat ? 0.f : (float)red[c];
      inv[c] = flat ? 1.f : __fmul_rn((float)(red[3 + c] - red[c]), 1.0f / 255.0f);
    }
  }

  // ---- one streaming pass: 3 uint8 values per output pixel -> erase -> normalise -> store
  for (int p = threadIdx.x; p < HW; p += kThreads) {
    const int y = p / W, x = p - y * W;
    int v[3];
    const int r = img[p], g = img[plane + p], b = img[2 * plane + p];
    v[0] = r; v[1] = g; v[2] = b;
    switch (op) {
      case kAffine: {
        const float xs = (float)x - 0.5f * (float)(W - 1), ys = (float)y - 0.5f * (float)(H - 1);
        const float gx = __fadd_rn(__fmaf_rn(ys, q[2], __fmul_rn(xs, q[1])), q[3]);
        const float gy = __fadd_rn(__fmaf_rn(ys, q[5], __fmul_rn(xs, q[4])), q[6]);
        const float ix = __fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f * (float)W), 0.5f);
        const float iy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f * (float)H), 0.5f);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = bilinear(img + c * plane, H, W, ix, iy);
        break;
      }
      case kRot90: {   // k = 1: out[i][j] = in[j][W-1-i]; k = 3: out[i][j] = in[H-1-j][i]
        const int sp = (int)p1 == 1 ? x * W + (W - 1 - y) : (H - 1 - x) * W + y;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = img[c * plane + sp];
        break;
      }
      case kBrightness:
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = trunc_u8(__fmul_rn((float)v[c], p1));
        break;
      case kColor: {
        const float gr = gray_floor((float)r, (float)g, (float)b);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = blend((float)v[c], gr, p1, p2);
        break;
      }
      case kContrast:
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = blend((float)v[c], mean, p1, p2);
        break;
      case kSharpness:
        if (y > 0 && y < H - 1 && x > 0 && x < W - 1) {
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const uint8_t* pc = img + c * plane + p;
            const int s8 = pc[-W - 1] + pc[-W] + pc[-W + 1] + pc[-1] + pc[1] + pc[W - 1] + pc[W] + pc[W + 1];
            const int blur = (2 * (s8 + 5 * v[c]) + 13) / 26;       // nearest integer to (s8 + 5 x) / 13 (never a tie)
            v[c] = trunc_u8(__fmaf_rn((float)(blur - v[c]), p1, (float)v[c]));
          }
        }
        break;
      case kPosterize:
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] &= (int)p1;
        break;
      case kSolarize:
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = (float)v[c] >= p1 ? 255 - v[c] : v[c];
        break;
      case kAutoContrast:
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = trunc_u8(__fdiv_rn(__fsub_rn((float)v[c], lo[c]), inv[c]));
        break;
      case kEqualize:
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = lut[c][v[c]];
        break;
      default:
        if constexpr (kChain) {
          if (op == kInvert) {
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = 255 - v[c];
          }
        }
        break;
    }
    if constexpr (kStage) {
#pragma unroll
      for (int c = 0; c < 3; ++c) stage[c * plane + p] = (uint8_t)v[c];
      continue;
    }
    const bool zero = erase && y >= ei && y < ei + eh && x >= ej && x < ej + ew;
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = zero ? 0.f : __fmaf_rn((float)v[c], sa[c], sb[c]);
    if constexpr (NHWC_OUT) {
      Out* d = dst + ((size_t)s * plane + p) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c] = from_f32<Out>(o[c]);
    } else {
      Out* d = dst + (size_t)s * 3 * plane + p;
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c * plane] = from_f32<Out>(o[c]);
    }
  }
}

// one op per sample: prm [n, kAugPrm]
template <typename Out, bool NHWC_OUT>
__global__ void __launch_bounds__(kThreads) augment_normalize_kernel(const uint8_t* __restrict__ src, Out* __restrict__ dst,
                                                                    const float* __restrict__ prm, int prm_stride,
                                                                    const float* __restrict__ na, const float* __restrict__ nb,
                                                                    int H, int W) {
  __shared__ int hist[3][256];
  __shared__ int lut[3][256];
  __shared__ int red[6];                   // Contrast: [0] sum; AutoContrast: [0..2] min, [3..5] max
  const int s = blockIdx.x;
  const float* q = prm + (size_t)s * prm_stride;
  apply_op<Out, NHWC_OUT, false, false>(src, s, q, q, dst, nullptr, s, H, W, na, nb, hist, lut, red);
}

// two ops per sample, launch 1: op A of each sample that applies it, into the uint8 scratch batch
__global__ void __launch_bounds__(kThreads) augment_stage_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ scratch,
                                                                const float* __restrict__ prm, int H, int W) {
  __shared__ int hist[3][256];
  __shared__ int lut[3][256];
  __shared__ int red[6];
  const int s = blockIdx.x;
  const float* q = prm + (size_t)s * kAugChainPrm;
  if ((int)q[0] == kIdentity) return;      // op A not applied: launch 2 reads the source
  // the normalisation is not read by a stage; q stands in for its pointers
  apply_op<float, false, true, true>(src, s, q, q, nullptr, scratch + (size_t)s * 3 * H * W, s, H, W, q, q, hist, lut, red);
}

// two ops per sample, launch 2: op B on op A's output (the source where op A is not applied), erase, normalise, store
template <typename Out, bool NHWC_OUT>
__global__ void __launch_bounds__(kThreads) augment_chain_kernel(const uint8_t* __restrict__ src, const uint8_t* __restrict__ scratch,
                                                                Out* __restrict__ dst, const float* __restrict__ prm,
                                                                const float* __restrict__ na, const float* __restrict__ nb, int H,
                                                                int W) {
  __shared__ int hist[3][256];
  __shared__ int lut[3][256];
  __shared__ int red[6];
  const int s = blockIdx.x;
  const float* q = prm + (size_t)s * kAugChainPrm;
  const uint8_t* from = (int)q[0] == kIdentity ? src : scratch;
  apply_op<Out, NHWC_OUT, true, false>(from, s, q + kColB, q, dst, nullptr, s, H, W, na, nb, hist, lut, red);
}

template <typename Out>
void launch(const at::Tensor& src, at::Tensor& dst, const at::Tensor& prm, const at::Tensor& a, const at::Tensor& b, bool nhwc) {
  const int n = (int)src.size(0), H = (int)src.size(2), W = (int)src.size(3);
  const cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (prm.size(1) == kAugChainPrm) {
    at::Tensor scratch = at::empty_like(src);
    augment_stage_kernel<<<n, kThreads, 0, stream>>>(src.data_ptr<uint8_t>(), scratch.data_ptr<uint8_t>(), prm.data_ptr<float>(),
                                                     H, W);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    auto kernel = nhwc ? augment_chain_kernel<Out, true> : augment_chain_kernel<Out, false>;
    kernel<<<n, kThreads, 0, stream>>>(src.data_ptr<uint8_t>(), scratch.data_ptr<uint8_t>(), reinterpret_cast<Out*>(dst.data_ptr()),
                                       prm.data_ptr<float>(), a.data_ptr<float>(), b.data_ptr<float>(), H, W);
  } else {
    auto kernel = nhwc ? augment_normalize_kernel<Out, true> : augment_normalize_kernel<Out, false>;
    kernel<<<n, kThreads, 0, stream>>>(src.data_ptr<uint8_t>(), reinterpret_cast<Out*>(dst.data_ptr()), prm.data_ptr<float>(),
                                       (int)prm.size(1), a.data_ptr<float>(), b.data_ptr<float>(), H, W);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace

at::Tensor augment_normalize(const at::Tensor& src, const at::Tensor& prm, const at::Tensor& a, const at::Tensor& b, int64_t out_dtype,
                             bool channels_last) {
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kByte && src.dim() == 4 && src.size(1) == 3 && src.is_contiguous(),
              "augment_normalize expects a contiguous uint8 NCHW batch with 3 channels on the GPU");
  const int64_t n = src.size(0), H = src.size(2), W = src.size(3);
  TORCH_CHECK(n > 0 && n <= 65535 && H > 0 && W > 0, "augment_normalize: bad batch geometry");
  TORCH_CHECK(H * W <= kAugMaxPixels, "augment_normalize: images of more than 65793 pixels (kAugMaxPixels), beyond which "
              "Contrast's float32 mean is no longer exact in torchvision's order");
  TORCH_CHECK(prm.device() == src.device() && prm.scalar_type() == at::kFloat && prm.is_contiguous() && prm.dim() == 2 &&
                  prm.size(0) == n && (prm.size(1) == kAugPrm || prm.size(1) == kAugChainPrm),
              "augment_normalize: prm must be a contiguous float32 [n, kAugPrm] (one op per sample) or [n, kAugChainPrm] "
              "(two) tensor on the batch's device");
  TORCH_CHECK(a.scalar_type() == at::kFloat && b.scalar_type() == at::kFloat && a.numel() == 3 && b.numel() == 3 &&
                  a.device() == src.device() && b.device() == src.device(),
              "augment_normalize: a and b must be float32 [3] on the batch's device");
  c10::cuda::CUDAGuard guard(src.device());
  const at::ScalarType ot = out_dtype == kBF16 ? at::kBFloat16 : out_dtype == kF16 ? at::kHalf : at::kFloat;
  at::Tensor dst = at::empty(src.sizes(), src.options().dtype(ot).memory_format(channels_last ? at::MemoryFormat::ChannelsLast
                                                                                              : at::MemoryFormat::Contiguous));
  switch (ot) {
    case at::kBFloat16: launch<__nv_bfloat16>(src, dst, prm, a, b, channels_last); break;
    case at::kHalf: launch<__half>(src, dst, prm, a, b, channels_last); break;
    default: launch<float>(src, dst, prm, a, b, channels_last); break;
  }
  return dst;
}

}  // namespace ptd
