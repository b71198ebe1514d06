// Device half of the shard loader's staging mode (csrc/host/loader.cpp, "staging for the device resample"): the
// antialiased triangle-filter resample of the loader's resample(), done on the GPU from the staged source regions and
// taps, fused with the normalise / cast / layout pass of normalize_kernel (data_ops.cu).
//
// The result is bit-identical to resample() on the host followed by normalize_nhwc:
//   * both passes sum in resample()'s k order with one rounding per multiply and one per add (__fmul_rn / __fadd_rn,
//     never contracted), and the horizontally resampled rows stay fp32;
//   * rounding to uint8 is +0.5, clamp to [0, 255], truncate;
//   * the normalisation is the single FFMA normalize_kernel compiles to (x * a[c] + b[c] under --use_fast_math).
// No value in either pass can be subnormal (weights are 0 or >= ~1e-17, pixels are integers), so the ftz variants
// --use_fast_math selects round exactly like the host's instructions.
//
// One CTA per (sample, band of kBandRows output rows).  The CTA resamples horizontally the source rows its band reads
// into shared memory, then runs the vertical pass from there.  When a band reads more rows than shared memory holds
// (strong down-scaling), it is done in several runs of output rows.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {

namespace {

struct StageDesc {    // mirrors StageDesc in csrc/host/loader.cpp
  int64_t region;     // arena offset of the HWC uint8 region (rh x rw x 3)
  int64_t taps;       // arena offset of: x first, x count (int32 [out_w]), x weights (float [out_w][kx]), same for y
  int32_t rw, rh;
  int32_t kx, ky;
};
static_assert(sizeof(StageDesc) == 32, "StageDesc layout");

constexpr int kThreads = 256;
constexpr int kBandRows = 16;
constexpr int kSmemTarget = 64 << 10;      // 3 CTAs per SM; at out_w = 224 it holds 24 resampled rows

template <typename Out> __device__ __forceinline__ Out out_px(float v) { return from_f32<Out>(v); }
template <> __device__ __forceinline__ uint8_t out_px<uint8_t>(float v) { return (uint8_t)v; }

template <typename Out, bool NHWC_OUT>
__global__ void __launch_bounds__(kThreads) resample_normalize_kernel(const uint8_t* __restrict__ arena, Out* __restrict__ dst,
                                                                      const float* __restrict__ na, const float* __restrict__ nb,
                                                                      int out_h, int out_w, int cap_rows) {
  extern __shared__ float rows[];          // [cap_rows][out_w][3]
  const int s = blockIdx.y;
  const StageDesc d = reinterpret_cast<const StageDesc*>(arena)[s];
  const uint8_t* region = arena + d.region;
  const int32_t* fx = reinterpret_cast<const int32_t*>(arena + d.taps);
  const int32_t* cx = fx + out_w;
  const float* wx = reinterpret_cast<const float*>(cx + out_w);
  const int32_t* fy = reinterpret_cast<const int32_t*>(wx + (size_t)out_w * d.kx);
  const int32_t* cy = fy + out_h;
  const float* wy = reinterpret_cast<const float*>(cy + out_h);
  const float sa[3] = {na[0], na[1], na[2]}, sb[3] = {nb[0], nb[1], nb[2]};
  const size_t src_stride = (size_t)d.rw * 3;
  const size_t plane = (size_t)out_h * out_w;
  const int band_end = min(out_h, (int)(blockIdx.x + 1) * kBandRows);

  for (int o0 = blockIdx.x * kBandRows; o0 < band_end;) {
    // the longest run of output rows [o0, o1) whose source rows [lo, hi) fit in shared memory (one row always fits:
    // the launcher sizes cap_rows to the largest count of the loader's y taps)
    int lo = fy[o0], hi = fy[o0] + cy[o0], o1 = o0 + 1;
    for (; o1 < band_end; ++o1) {
      const int l = min(lo, fy[o1]), h = max(hi, fy[o1] + cy[o1]);
      if (h - l > cap_rows) break;
      lo = l;
      hi = h;
    }
    const int n_h = (hi - lo) * out_w;                   // horizontal pass -> rows[r][x][c]
    for (int t = threadIdx.x; t < n_h; t += kThreads) {
      const int r = t / out_w, x = t - r * out_w;
      const uint8_t* p = region + (size_t)(lo + r) * src_stride + (size_t)fx[x] * 3;
      const float* w = wx + (size_t)x * d.kx;
      const int n = cx[x];
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      for (int k = 0; k < n; ++k) {
        const float wk = w[k];
        a0 = __fadd_rn(a0, __fmul_rn(wk, (float)p[3 * k]));
        a1 = __fadd_rn(a1, __fmul_rn(wk, (float)p[3 * k + 1]));
        a2 = __fadd_rn(a2, __fmul_rn(wk, (float)p[3 * k + 2]));
      }
      float* q = rows + (size_t)t * 3;
      q[0] = a0;
      q[1] = a1;
      q[2] = a2;
    }
    __syncthreads();
    const int n_v = (o1 - o0) * out_w;                   // vertical pass, uint8 rounding, normalise, store
    for (int t = threadIdx.x; t < n_v; t += kThreads) {
      const int o = o0 + t / out_w, x = t % out_w;
      const float* w = wy + (size_t)o * d.ky;
      const float* base = rows + ((size_t)(fy[o] - lo) * out_w + x) * 3;
      const int n = cy[o];
      float acc[3] = {0.f, 0.f, 0.f};
      for (int k = 0; k < n; ++k) {
        const float wk = w[k];
        const float* p = base + (size_t)k * out_w * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(wk, p[c]));
      }
      float v[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float px = (float)__float2uint_rz(fminf(255.f, fmaxf(0.f, __fadd_rn(acc[c], 0.5f))));
        v[c] = std::is_same<Out, uint8_t>::value ? px : __fmaf_rn(px, sa[c], sb[c]);   // uint8: the pixel itself
      }
      const size_t pix = (size_t)o * out_w + x;
      if constexpr (NHWC_OUT) {
        Out* q = dst + ((size_t)s * plane + pix) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) q[c] = out_px<Out>(v[c]);
      } else {
        Out* q = dst + (size_t)s * 3 * plane + pix;
#pragma unroll
        for (int c = 0; c < 3; ++c) q[c * plane] = out_px<Out>(v[c]);
      }
    }
    __syncthreads();
    o0 = o1;
  }
}

template <typename Out>
void launch(const at::Tensor& arena, at::Tensor& dst, const at::Tensor& a, const at::Tensor& b, int n, int out_h, int out_w,
            int cap_rows, bool nhwc) {
  const size_t smem = (size_t)cap_rows * out_w * 3 * sizeof(float);
  auto kernel = nhwc ? resample_normalize_kernel<Out, true> : resample_normalize_kernel<Out, false>;
  C10_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((out_h + kBandRows - 1) / kBandRows, n);
  kernel<<<grid, kThreads, smem, at::cuda::getCurrentCUDAStream()>>>(arena.data_ptr<uint8_t>(), reinterpret_cast<Out*>(dst.data_ptr()),
                                                                     a.data_ptr<float>(), b.data_ptr<float>(), out_h, out_w, cap_rows);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace

// arena: a staged batch copied to the device (descriptors of samples 0..n-1 first).  max_rows: an upper bound of the
// y tap counts (ShardLoader.stage_max_rows()).  Returns the tensor normalize_nhwc returns for the host-resampled batch: [n, 3, out_h, out_w] of
// (pixel * a[c] + b[c]) in out_dtype, channels_last or contiguous.  out_dtype kU8Out returns the uint8 batch itself (contiguous
// NCHW, no normalisation): the input of augment_normalize, the same bytes as the host-resampled batch.
at::Tensor resample_normalize(const at::Tensor& arena, int64_t n, int64_t out_h, int64_t out_w, int64_t max_rows, const at::Tensor& a,
                              const at::Tensor& b, int64_t out_dtype, bool channels_last) {
  TORCH_CHECK(arena.is_cuda() && arena.scalar_type() == at::kByte && arena.dim() == 1 && arena.is_contiguous(),
              "resample_normalize expects a contiguous uint8 arena on the GPU");
  TORCH_CHECK(n > 0 && n <= 65535 && out_h > 0 && out_w > 0 && max_rows > 0, "resample_normalize: bad batch geometry");
  TORCH_CHECK(arena.numel() >= n * (int64_t)sizeof(StageDesc), "resample_normalize: arena smaller than its descriptor table");
  TORCH_CHECK(a.scalar_type() == at::kFloat && b.scalar_type() == at::kFloat && a.numel() == 3 && b.numel() == 3 && a.is_cuda() && b.is_cuda());
  c10::cuda::CUDAGuard guard(arena.device());
  const int row_bytes = (int)out_w * 3 * (int)sizeof(float);
  const int cap_rows = std::max<int>((int)max_rows, kSmemTarget / row_bytes);
  int smem_max = 0;
  C10_CUDA_CHECK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, arena.get_device()));
  TORCH_CHECK((int64_t)cap_rows * row_bytes <= smem_max, "resample_normalize: ", cap_rows, " source rows of width ", out_w,
              " do not fit in shared memory");
  const at::ScalarType ot = out_dtype == kU8Out ? at::kByte : out_dtype == kBF16 ? at::kBFloat16 : out_dtype == kF16 ? at::kHalf : at::kFloat;
  TORCH_CHECK(!(ot == at::kByte && channels_last), "resample_normalize: the uint8 output is NCHW");
  at::Tensor dst = at::empty({n, 3, out_h, out_w}, arena.options().dtype(ot).memory_format(channels_last ? at::MemoryFormat::ChannelsLast
                                                                                                        : at::MemoryFormat::Contiguous));
  switch (ot) {
    case at::kByte: launch<uint8_t>(arena, dst, a, b, (int)n, (int)out_h, (int)out_w, cap_rows, false); break;
    case at::kBFloat16: launch<__nv_bfloat16>(arena, dst, a, b, (int)n, (int)out_h, (int)out_w, cap_rows, channels_last); break;
    case at::kHalf: launch<__half>(arena, dst, a, b, (int)n, (int)out_h, (int)out_w, cap_rows, channels_last); break;
    default: launch<float>(arena, dst, a, b, (int)n, (int)out_h, (int)out_w, cap_rows, channels_last); break;
  }
  return dst;
}

}  // namespace ptd
