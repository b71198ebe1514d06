// Training-time target policy: MixUp / CutMix of a device batch and a cross-entropy against the mixed, label-smoothed
// probability targets (torchvision's transforms.v2.MixUp / CutMix and nn.CrossEntropyLoss(label_smoothing=eps)).
//
//  mix_batch   : out = mix(x, roll(x, 1, 0)) in ONE pass over the batch (bf16 / fp16 / fp32, NCHW or channels_last), plus
//                y_b = roll(y, 1) and the dominant label (the argmax of the mixed target, first index on a tie).
//  soft_ce_fwd : per row lse and loss_r = lse - (1-eps)(la z[y_a] + lb z[y_b]) - (eps/C) sum z, then the rows summed in a
//                fixed order into the mean (a second one-CTA kernel: no float atomics).
//  soft_ce_bwd : dz = g / B (softmax(z) - q), q = (1-eps)(la onehot(y_a) + lb onehot(y_b)) + eps/C, never materialised.
//
// Every per-step value lives in the float[8] parameter tensor `prm`, read on the device, so a captured CUDA graph follows the
// host's new draws: prm[0] mode (1 MixUp, 2 CutMix, anything else: copy), prm[1] la = fp32(lambda), prm[2] lb = fp32(1 - lambda)
// (CutMix: of the box-adjusted lambda), prm[3..6] the CutMix box x1, y1, x2, y2 (rows [y1, y2), columns [x1, x2)).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {
namespace {

// IEEE fp32 product / sum, each rounded, no FMA contraction and denormals kept (the extension builds with --use_fast_math):
// torch's roll(1, 0).mul_(1 - lam).add_(x.mul(lam)) on fp32 CPU tensors, bit for bit
__device__ __forceinline__ float mul_rn(float a, float b) {
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float add_rn(float a, float b) {
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// storage bits of one element <-> fp32
template <typename T> struct Bits;
template <> struct Bits<float> {
  using U = uint32_t;
  static __device__ __forceinline__ float f(U u) { return __uint_as_float(u); }
  static __device__ __forceinline__ U u(float f) { return __float_as_uint(f); }
};
template <> struct Bits<__nv_bfloat16> {
  using U = uint16_t;
  static __device__ __forceinline__ float f(U u) { return __uint_as_float((uint32_t)u << 16); }
  static __device__ __forceinline__ U u(float f) { return __bfloat16_as_ushort(__float2bfloat16_rn(f)); }
};
template <> struct Bits<__half> {
  using U = uint16_t;
  static __device__ __forceinline__ float f(U u) { return __half2float(__ushort_as_half(u)); }
  static __device__ __forceinline__ U u(float f) { return __half_as_ushort(__float2half_rn(f)); }
};

template <typename T> union Pack {
  static constexpr int N = 16 / sizeof(typename Bits<T>::U);
  V4 v;
  typename Bits<T>::U e[N];
};

struct MixGeom {
  int B, C, H, W;
  int64_t chw;    // elements per sample (the sample stride of both layouts)
};

// (h, w) of the element at offset o inside its sample
template <bool NHWC> __device__ __forceinline__ void pixel_of(const MixGeom& g, int64_t o, int& h, int& w) {
  const int64_t p = NHWC ? o / g.C : o % ((int64_t)g.H * g.W);
  h = (int)(p / g.W);
  w = (int)(p - (int64_t)h * g.W);
}

template <typename T, bool NHWC>
__global__ void __launch_bounds__(256) mix_batch_kernel(const T* __restrict__ x, T* __restrict__ out, const int64_t* __restrict__ y,
                                                        int64_t* __restrict__ yb, int64_t* __restrict__ dom, const float* __restrict__ prm,
                                                        MixGeom g, int64_t nvec, int64_t total, bool prev_vec) {
  using Bt = Bits<T>;
  using U = typename Bt::U;
  constexpr int N = Pack<T>::N;
  const int mode = (int)prm[0];
  const float la = prm[1], lb = prm[2];
  const int x1 = (int)prm[3], y1 = (int)prm[4], x2 = (int)prm[5], y2 = (int)prm[6];
  const int64_t gs = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t wrap = (int64_t)(g.B - 1) * g.chw;       // sample 0 pairs with sample B-1
  const U* xu = reinterpret_cast<const U*>(x);
  U* ou = reinterpret_cast<U*>(out);

  for (int64_t n = t0; n < g.B; n += gs) {
    const int64_t a = y[n], b = y[n == 0 ? g.B - 1 : n - 1];
    yb[n] = b;
    dom[n] = la > lb ? a : la < lb ? b : (a < b ? a : b);
  }

  // 16-byte vectors: element k of vector v is flat index v * N + k, in sample n (the vector may cross into sample n + 1
  // when the sample stride is not a multiple of N; then the paired elements are read one by one)
  for (int64_t v = t0; v < nvec; v += gs) {
    const int64_t i0 = v * N;
    const int64_t n0 = i0 / g.chw;
    const int64_t o0 = i0 - n0 * g.chw;
    Pack<T> xv, pv, r;
    xv.v = ld_stream(xu + i0);
    if (mode == 1) {
      if (prev_vec) {
        pv.v = ld_stream(xu + (n0 == 0 ? i0 + wrap : i0 - g.chw));
      } else {
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const int64_t i = i0 + k;
          const int64_t n = o0 + k < g.chw ? n0 : n0 + 1;
          pv.e[k] = xu[n == 0 ? i + wrap : i - g.chw];
        }
      }
#pragma unroll
      for (int k = 0; k < N; ++k) r.e[k] = Bt::u(add_rn(mul_rn(Bt::f(pv.e[k]), lb), mul_rn(Bt::f(xv.e[k]), la)));
    } else if (mode == 2) {
      uint32_t inb = 0;          // bit k: element k lies in the box
      int h, w;
      pixel_of<NHWC>(g, o0, h, w);
      int c = NHWC ? (int)(o0 % g.C) : 0;
      int64_t o = o0;
#pragma unroll
      for (int k = 0; k < N; ++k) {
        inb |= (uint32_t)(h >= y1 && h < y2 && w >= x1 && w < x2) << k;
        // advance to element k + 1
        if (++o == g.chw) { o = 0; h = 0; w = 0; c = 0; continue; }
        if (NHWC && ++c < g.C) continue;
        c = 0;
        if (++w == g.W) { w = 0; if (++h == g.H) h = 0; }
      }
      r = xv;
      if (inb) {
        if (prev_vec) pv.v = ld_stream(xu + (n0 == 0 ? i0 + wrap : i0 - g.chw));
#pragma unroll
        for (int k = 0; k < N; ++k) {
          if (!(inb >> k & 1)) continue;
          const int64_t i = i0 + k;
          const int64_t n = o0 + k < g.chw ? n0 : n0 + 1;
          r.e[k] = prev_vec ? pv.e[k] : xu[n == 0 ? i + wrap : i - g.chw];
        }
      }
    } else {
      r = xv;
    }
    st_v4(ou + i0, r.v);
  }

  // the elements after the last whole vector (all of them when the pointers are not 16-byte aligned)
  for (int64_t i = nvec * N + t0; i < total; i += gs) {
    const int64_t n = i / g.chw, o = i - n * g.chw;
    const int64_t ip = n == 0 ? i + wrap : i - g.chw;
    U rv = xu[i];
    if (mode == 1) {
      rv = Bt::u(add_rn(mul_rn(Bt::f(xu[ip]), lb), mul_rn(Bt::f(xu[i]), la)));
    } else if (mode == 2) {
      int h, w;
      pixel_of<NHWC>(g, o, h, w);
      if (h >= y1 && h < y2 && w >= x1 && w < x2) rv = xu[ip];
    }
    ou[i] = rv;
  }
}

template <typename T>
void launch_mix(const at::Tensor& x, at::Tensor& out, const at::Tensor& y, at::Tensor& yb, at::Tensor& dom, const at::Tensor& prm, bool nhwc) {
  MixGeom g{(int)x.size(0), (int)x.size(1), (int)x.size(2), (int)x.size(3), x.size(1) * x.size(2) * x.size(3)};
  constexpr int N = Pack<T>::N;
  const int64_t total = x.numel();
  const bool aligned = ((reinterpret_cast<uintptr_t>(x.data_ptr()) | reinterpret_cast<uintptr_t>(out.data_ptr())) & 15) == 0;
  const int64_t nvec = aligned ? total / N : 0;
  const bool prev_vec = g.chw % N == 0;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int64_t work = std::max<int64_t>(std::max<int64_t>(nvec, total - nvec * N), g.B);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((work + 255) / 256, (int64_t)sms * 8));
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const T* xp = reinterpret_cast<const T*>(x.data_ptr());
  T* op = reinterpret_cast<T*>(out.data_ptr());
  const int64_t *yp = y.data_ptr<int64_t>();
  int64_t *ybp = yb.data_ptr<int64_t>(), *dp = dom.data_ptr<int64_t>();
  if (nhwc) mix_batch_kernel<T, true><<<grid, 256, 0, st>>>(xp, op, yp, ybp, dp, prm.data_ptr<float>(), g, nvec, total, prev_vec);
  else      mix_batch_kernel<T, false><<<grid, 256, 0, st>>>(xp, op, yp, ybp, dp, prm.data_ptr<float>(), g, nvec, total, prev_vec);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ soft-target cross-entropy
constexpr int kCeWarps = 8;   // rows per CTA: one warp per row

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(kCeWarps * 32) soft_ce_fwd_kernel(const T* __restrict__ z, int64_t ld, const int64_t* __restrict__ ya,
                                                                    const int64_t* __restrict__ yb, const float* __restrict__ prm, int B, int C,
                                                                    float eps, float* __restrict__ row_loss, float* __restrict__ lse_out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kCeWarps + (threadIdx.x >> 5);
  if (row >= B) return;
  const T* zr = z + (int64_t)row * ld;
  float m = -INFINITY;
  for (int j = lane; j < C; j += 32) m = fmaxf(m, to_f32<T>(zr[j]));
  m = warp_max(m);
  float s = 0.f, sz = 0.f;
  for (int j = lane; j < C; j += 32) {
    const float v = to_f32<T>(zr[j]);
    s += __expf(v - m);
    sz += v;
  }
  s = warp_sum(s);
  sz = warp_sum(sz);
  if (lane == 0) {
    const float lse = m + __logf(s);
    const int64_t a = ya[row], b = yb[row];
    float loss = __int_as_float(0x7fffffff);                // a label outside [0, C): NaN, and nothing is read for it
    if (a >= 0 && a < C && b >= 0 && b < C)
      loss = lse - (1.f - eps) * (prm[1] * to_f32<T>(zr[a]) + prm[2] * to_f32<T>(zr[b])) - (eps / (float)C) * sz;
    row_loss[row] = loss;
    lse_out[row] = lse;
  }
}

// mean of the row losses, summed in a fixed order (one CTA: per-thread strided sums, then a fixed tree)
__global__ void __launch_bounds__(256) soft_ce_mean_kernel(const float* __restrict__ row_loss, int B, float* __restrict__ loss) {
  __shared__ float sh[256];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += 256) s += row_loss[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = sh[0] / (float)B;
}

template <typename T>
__global__ void __launch_bounds__(kCeWarps * 32) soft_ce_bwd_kernel(const T* __restrict__ z, int64_t ld, const int64_t* __restrict__ ya,
                                                                    const int64_t* __restrict__ yb, const float* __restrict__ prm,
                                                                    const float* __restrict__ lse, const float* __restrict__ gout, int B, int C,
                                                                    float eps, T* __restrict__ dz) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kCeWarps + (threadIdx.x >> 5);
  if (row >= B) return;
  const T* zr = z + (int64_t)row * ld;
  T* dr = dz + (int64_t)row * C;
  const float scale = gout[0] / (float)B;
  const float l = lse[row];
  const int64_t a = ya[row], b = yb[row];
  const bool bad = a < 0 || a >= C || b < 0 || b >= C;
  const float ta = (1.f - eps) * prm[1], tb = (1.f - eps) * prm[2], te = eps / (float)C;
  for (int j = lane; j < C; j += 32) {
    const float p = __expf(to_f32<T>(zr[j]) - l);
    const float q = ((j == a ? ta : 0.f) + (j == b ? tb : 0.f)) + te;
    dr[j] = from_f32<T>(bad ? __int_as_float(0x7fffffff) : (p - q) * scale);
  }
}

void check_ce(const at::Tensor& z, const at::Tensor& ya, const at::Tensor& yb, const at::Tensor& prm) {
  TORCH_CHECK(z.is_cuda() && z.dim() == 2 && z.stride(1) == 1 && z.stride(0) >= z.size(1), "soft_ce: logits must be a CUDA [B, C] matrix with unit inner stride");
  TORCH_CHECK(z.scalar_type() == at::kFloat || z.scalar_type() == at::kBFloat16 || z.scalar_type() == at::kHalf, "soft_ce: logits must be fp32, bf16 or fp16");
  TORCH_CHECK(z.size(0) > 0 && z.size(1) > 0 && z.size(0) < (1LL << 31) && z.size(1) < (1LL << 31), "soft_ce: empty or oversized logits");
  for (const at::Tensor* t : {&ya, &yb})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->is_contiguous() && t->numel() == z.size(0), "soft_ce: labels must be contiguous int64 [B]");
  TORCH_CHECK(prm.is_cuda() && prm.scalar_type() == at::kFloat && prm.is_contiguous() && prm.numel() >= 8, "soft_ce: parameters must be float[8]");
}

}  // namespace

void mix_batch(const at::Tensor& x, at::Tensor out, const at::Tensor& y, at::Tensor yb, at::Tensor dom, const at::Tensor& prm) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && x.size(0) > 0, "mix_batch: x must be a CUDA [B, C, H, W] batch");
  const bool nhwc = !x.is_contiguous() && x.is_contiguous(at::MemoryFormat::ChannelsLast);
  TORCH_CHECK(nhwc || x.is_contiguous(), "mix_batch: x must be contiguous NCHW or channels_last");
  TORCH_CHECK(out.sizes() == x.sizes() && out.strides() == x.strides() && out.scalar_type() == x.scalar_type() && out.device() == x.device(),
              "mix_batch: out must match x in shape, layout, dtype and device");
  TORCH_CHECK(x.size(0) < (1LL << 31) && x.size(2) * x.size(3) < (1LL << 31), "mix_batch: batch too large");
  for (const at::Tensor* t : std::initializer_list<const at::Tensor*>{&y, &yb, &dom})
    TORCH_CHECK(t->device() == x.device() && t->scalar_type() == at::kLong && t->is_contiguous() && t->numel() == x.size(0),
                "mix_batch: labels must be contiguous int64 [B] on the batch's device");
  TORCH_CHECK(prm.device() == x.device() && prm.scalar_type() == at::kFloat && prm.is_contiguous() && prm.numel() >= 8,
              "mix_batch: parameters must be float[8] on the batch's device");
  c10::cuda::CUDAGuard guard(x.device());
  switch (x.scalar_type()) {
    case at::kBFloat16: launch_mix<__nv_bfloat16>(x, out, y, yb, dom, prm, nhwc); break;
    case at::kHalf: launch_mix<__half>(x, out, y, yb, dom, prm, nhwc); break;
    case at::kFloat: launch_mix<float>(x, out, y, yb, dom, prm, nhwc); break;
    default: TORCH_CHECK(false, "mix_batch: x must be fp32, bf16 or fp16");
  }
}

std::vector<at::Tensor> soft_ce_fwd(const at::Tensor& z, const at::Tensor& ya, const at::Tensor& yb, const at::Tensor& prm, double eps) {
  check_ce(z, ya, yb, prm);
  c10::cuda::CUDAGuard guard(z.device());
  const int B = (int)z.size(0), C = (int)z.size(1);
  auto fo = z.options().dtype(at::kFloat);
  at::Tensor loss = at::empty({}, fo), row = at::empty({B}, fo), lse = at::empty({B}, fo);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int grid = (B + kCeWarps - 1) / kCeWarps;
#define CE_FWD(T) \
  soft_ce_fwd_kernel<T><<<grid, kCeWarps * 32, 0, st>>>(reinterpret_cast<const T*>(z.data_ptr()), z.stride(0), ya.data_ptr<int64_t>(), \
                                                        yb.data_ptr<int64_t>(), prm.data_ptr<float>(), B, C, (float)eps, \
                                                        row.data_ptr<float>(), lse.data_ptr<float>())
  switch (z.scalar_type()) {
    case at::kBFloat16: CE_FWD(__nv_bfloat16); break;
    case at::kHalf: CE_FWD(__half); break;
    default: CE_FWD(float); break;
  }
#undef CE_FWD
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  soft_ce_mean_kernel<<<1, 256, 0, st>>>(row.data_ptr<float>(), B, loss.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {loss, row, lse};
}

at::Tensor soft_ce_bwd(const at::Tensor& z, const at::Tensor& ya, const at::Tensor& yb, const at::Tensor& prm, const at::Tensor& lse,
                       const at::Tensor& gout, double eps) {
  check_ce(z, ya, yb, prm);
  TORCH_CHECK(lse.device() == z.device() && lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == z.size(0),
              "soft_ce_bwd: lse must be the forward's float [B]");
  TORCH_CHECK(gout.device() == z.device() && gout.scalar_type() == at::kFloat && gout.numel() == 1, "soft_ce_bwd: g must be one fp32 value");
  c10::cuda::CUDAGuard guard(z.device());
  const int B = (int)z.size(0), C = (int)z.size(1);
  at::Tensor dz = at::empty({B, C}, z.options());
  at::Tensor g = gout.contiguous();
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int grid = (B + kCeWarps - 1) / kCeWarps;
#define CE_BWD(T) \
  soft_ce_bwd_kernel<T><<<grid, kCeWarps * 32, 0, st>>>(reinterpret_cast<const T*>(z.data_ptr()), z.stride(0), ya.data_ptr<int64_t>(), \
                                                        yb.data_ptr<int64_t>(), prm.data_ptr<float>(), lse.data_ptr<float>(), \
                                                        g.data_ptr<float>(), B, C, (float)eps, reinterpret_cast<T*>(dz.data_ptr()))
  switch (z.scalar_type()) {
    case at::kBFloat16: CE_BWD(__nv_bfloat16); break;
    case at::kHalf: CE_BWD(__half); break;
    default: CE_BWD(float); break;
  }
#undef CE_BWD
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dz;
}

}  // namespace ptd
