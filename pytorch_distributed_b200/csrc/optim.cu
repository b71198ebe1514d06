// K6: fused unscale + overflow-skip + weight-decay + momentum + SGD update (+ low-precision model copy).
//
// Replaces, for /root/reference/apex_distributed.py:328-330, apex's amp_C.multi_tensor_scale (unscale + inf check),
// the patched optimizer.step() and (O2) the master->model half copy; and for every other entrypoint
// torch.optim.SGD.step() (/root/reference/distributed.py:153-156,269).
//
// Two front-ends:
//   fused_sgd_flat  : gradients are read straight out of the (already all-reduced) wire arena; master weights,
//                     momentum and the model copy are flat buffers with the SAME layout, so the whole optimizer
//                     is ONE perfectly coalesced streaming kernel with no pointer tables (20 B/element of HBM
//                     traffic with a bf16 arena: 2 R grad + 4 R/W master + 4 R/W momentum + 2 W model).
//   fused_sgd_multi : classic chunked multi-tensor-apply over arbitrary tensor lists.
//
// Hyper-parameters live in a device tensor `hyper` = {lr, momentum, weight_decay, dampening, grad_multiplier,
// momentum_pending} so a captured CUDA graph keeps working when the LR schedule or the loss scale changes.
// momentum_pending (slot 5) is read only under dynamic loss scaling (a found_inf flag is given): while it is non-zero the
// step initialises the momentum buffer (m = g), as on the first step.  amp_update_scale clears it after the first step
// that was applied, so a skipped (overflowed) first step does not turn the next one into m = (1 - dampening) g.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {

struct SgdHyper { float lr, momentum, wd, dampening, gmul; };

__device__ __forceinline__ SgdHyper load_hyper(const float* h) { return SgdHyper{h[0], h[1], h[2], h[3], h[4]}; }

__device__ __forceinline__ void sgd_update(float g, float& p, float& m, const SgdHyper& h, bool nesterov, bool first) {
  g = g * h.gmul + h.wd * p;
  if (h.momentum != 0.f) {
    m = first ? g : h.momentum * m + (1.f - h.dampening) * g;
    g = nesterov ? g + h.momentum * m : m;
  }
  p -= h.lr * g;
}

template <typename G, typename C, bool HAS_COPY>
__global__ void __launch_bounds__(256) fused_sgd_flat_kernel(const G* __restrict__ grad, float* __restrict__ master,
                                                             float* __restrict__ mom, C* __restrict__ copy, int64_t n,
                                                             const float* __restrict__ hyper, const int* __restrict__ found_inf,
                                                             bool nesterov, bool first) {
  if (found_inf && *found_inf) return;  // dynamic loss scaling: skip the step on overflow
  const SgdHyper h = load_hyper(hyper);
  first = first || (found_inf && hyper[5] != 0.f);
  const int64_t nvec = n >> 3;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * blockDim.x) {
    float g[8], p[8], m[8];
    load8<G>(grad + (v << 3), g, /*sys=*/true);  // arena was written by peers / the switch: bypass L1
    load8<float>(master + (v << 3), p);
    load8<float>(mom + (v << 3), m);
#pragma unroll
    for (int k = 0; k < 8; ++k) sgd_update(g[k], p[k], m[k], h, nesterov, first);
    store8<float>(master + (v << 3), p);
    store8<float>(mom + (v << 3), m);
    if constexpr (HAS_COPY) store8<C>(copy + (v << 3), p);
  }
  // n is padded to a multiple of 8 by the arena layout; no scalar tail.
}

void fused_sgd_flat(at::Tensor grad, at::Tensor master, at::Tensor momentum, c10::optional<at::Tensor> model_copy, at::Tensor hyper,
                    c10::optional<at::Tensor> found_inf, bool nesterov, bool first_step) {
  const int64_t n = master.numel();
  TORCH_CHECK(n % 8 == 0, "flat optimizer buffers must be padded to a multiple of 8 elements");
  TORCH_CHECK(grad.numel() >= n && momentum.numel() == n, "flat buffer size mismatch");
  TORCH_CHECK(master.scalar_type() == at::kFloat && momentum.scalar_type() == at::kFloat && hyper.scalar_type() == at::kFloat);
  TORCH_CHECK(master.is_contiguous() && momentum.is_contiguous() && grad.is_contiguous());
  TORCH_CHECK(!found_inf.has_value() || hyper.numel() >= 6, "hyper needs slot 5 (momentum_pending) when found_inf is given");
  c10::cuda::CUDAGuard guard(master.device());
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int grid = (int)std::min<int64_t>((n / 8 + 255) / 256, (int64_t)sms * 8);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  float* mp = master.data_ptr<float>();
  float* vp = momentum.data_ptr<float>();
  const float* hp = hyper.data_ptr<float>();
#define LAUNCH(G, C, HC, cptr) \
  fused_sgd_flat_kernel<G, C, HC><<<grid, 256, 0, st>>>(reinterpret_cast<const G*>(grad.data_ptr()), mp, vp, cptr, n, hp, fi, nesterov, first_step)
  const bool has_copy = model_copy.has_value();
  if (has_copy) TORCH_CHECK(model_copy->numel() == n && model_copy->is_contiguous());
  const auto gt = grad.scalar_type();
  const auto ct = has_copy ? model_copy->scalar_type() : at::kFloat;
  if (gt == at::kBFloat16) {
    if (!has_copy) LAUNCH(__nv_bfloat16, float, false, nullptr);
    else if (ct == at::kBFloat16) LAUNCH(__nv_bfloat16, __nv_bfloat16, true, reinterpret_cast<__nv_bfloat16*>(model_copy->data_ptr()));
    else if (ct == at::kHalf) LAUNCH(__nv_bfloat16, __half, true, reinterpret_cast<__half*>(model_copy->data_ptr()));
    else TORCH_CHECK(false, "unsupported model copy dtype");
  } else if (gt == at::kHalf) {
    if (!has_copy) LAUNCH(__half, float, false, nullptr);
    else if (ct == at::kHalf) LAUNCH(__half, __half, true, reinterpret_cast<__half*>(model_copy->data_ptr()));
    else if (ct == at::kBFloat16) LAUNCH(__half, __nv_bfloat16, true, reinterpret_cast<__nv_bfloat16*>(model_copy->data_ptr()));
    else TORCH_CHECK(false, "unsupported model copy dtype");
  } else if (gt == at::kFloat) {
    if (!has_copy) LAUNCH(float, float, false, nullptr);
    else if (ct == at::kBFloat16) LAUNCH(float, __nv_bfloat16, true, reinterpret_cast<__nv_bfloat16*>(model_copy->data_ptr()));
    else if (ct == at::kHalf) LAUNCH(float, __half, true, reinterpret_cast<__half*>(model_copy->data_ptr()));
    else TORCH_CHECK(false, "unsupported model copy dtype");
  } else {
    TORCH_CHECK(false, "unsupported gradient dtype");
  }
#undef LAUNCH
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// ---------------------------------------------------------------- chunked multi-tensor apply
constexpr int kMtaTensors = 30;
constexpr int kMtaBlocks = 320;
constexpr int kMtaChunk = 8192;  // elements per CTA

template <int DEPTH>
struct MtaArgs {
  void* ptr[DEPTH][kMtaTensors];
  int64_t numel[kMtaTensors];
  uint8_t dtype[DEPTH][kMtaTensors];
  uint8_t block_tensor[kMtaBlocks];
  int32_t block_chunk[kMtaBlocks];
};

__device__ __forceinline__ float ld_any(const void* p, int dt, int64_t i) {
  switch (dt) {
    case kF32: return reinterpret_cast<const float*>(p)[i];
    case kBF16: return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
    default: return __half2float(reinterpret_cast<const __half*>(p)[i]);
  }
}
__device__ __forceinline__ void st_any(void* p, int dt, int64_t i, float v) {
  switch (dt) {
    case kF32: reinterpret_cast<float*>(p)[i] = v; break;
    case kBF16: reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v); break;
    default: reinterpret_cast<__half*>(p)[i] = __float2half_rn(v); break;
  }
}

// lists: 0 grad, 1 param (fp32 master), 2 momentum (fp32), 3 model copy (optional: ptr may be null)
__global__ void __launch_bounds__(256) fused_sgd_multi_kernel(const __grid_constant__ MtaArgs<4> a, const float* __restrict__ hyper,
                                                              const int* __restrict__ found_inf, bool nesterov, bool first) {
  if (found_inf && *found_inf) return;
  const SgdHyper h = load_hyper(hyper);
  first = first || (found_inf && hyper[5] != 0.f);
  const int t = a.block_tensor[blockIdx.x];
  const int64_t begin = (int64_t)a.block_chunk[blockIdx.x] * kMtaChunk;
  const int64_t end = min(begin + (int64_t)kMtaChunk, a.numel[t]);
  float* p = reinterpret_cast<float*>(a.ptr[1][t]);
  float* m = reinterpret_cast<float*>(a.ptr[2][t]);
  const int gdt = a.dtype[0][t], cdt = a.dtype[3][t];
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    float g = ld_any(a.ptr[0][t], gdt, i), pv = p[i], mv = m[i];
    sgd_update(g, pv, mv, h, nesterov, first);
    p[i] = pv;
    m[i] = mv;
    if (a.ptr[3][t]) st_any(a.ptr[3][t], cdt, i, pv);
  }
}

// dst = src * scale, found_inf |= any non-finite(src)
__global__ void __launch_bounds__(256) multi_tensor_scale_kernel(const __grid_constant__ MtaArgs<2> a, float scale, int* found_inf) {
  const int t = a.block_tensor[blockIdx.x];
  const int64_t begin = (int64_t)a.block_chunk[blockIdx.x] * kMtaChunk;
  const int64_t end = min(begin + (int64_t)kMtaChunk, a.numel[t]);
  bool bad = false;
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    float v = ld_any(a.ptr[0][t], a.dtype[0][t], i);
    bad |= !isfinite(v);
    st_any(a.ptr[1][t], a.dtype[1][t], i, v * scale);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1;
}

// out = a * x + b * y, found_inf |= any non-finite(x or y)   (apex amp_C.multi_tensor_axpby: master-gradient accumulation)
__global__ void __launch_bounds__(256) multi_tensor_axpby_kernel(const __grid_constant__ MtaArgs<3> a, float ca, float cb, int* found_inf) {
  const int t = a.block_tensor[blockIdx.x];
  const int64_t begin = (int64_t)a.block_chunk[blockIdx.x] * kMtaChunk;
  const int64_t end = min(begin + (int64_t)kMtaChunk, a.numel[t]);
  bool bad = false;
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    const float x = ld_any(a.ptr[0][t], a.dtype[0][t], i), y = ld_any(a.ptr[1][t], a.dtype[1][t], i);
    bad |= !isfinite(x) || !isfinite(y);
    st_any(a.ptr[2][t], a.dtype[2][t], i, ca * x + cb * y);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1;
}

static uint8_t dtype_code(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return kF32;
    case at::kBFloat16: return kBF16;
    case at::kHalf: return kF16;
    default: TORCH_CHECK(false, "unsupported dtype ", t.scalar_type()); return 0;
  }
}

template <int DEPTH, typename LaunchFn>
static void mta_for_each(const std::vector<std::vector<at::Tensor>>& lists, LaunchFn&& launch) {
  const size_t n = lists[0].size();
  MtaArgs<DEPTH> a;
  int nt = 0, nb = 0;
  auto flush = [&]() {
    if (nb > 0) launch(a, nb);
    nt = 0;
    nb = 0;
  };
  for (size_t i = 0; i < n; ++i) {
    const int64_t numel = lists[0][i].numel();
    if (numel == 0) continue;
    const int64_t chunks = (numel + kMtaChunk - 1) / kMtaChunk;
    int64_t c = 0;
    while (c < chunks) {
      if (nt == kMtaTensors || nb == kMtaBlocks) flush();
      // (re)register tensor i in this launch
      for (int d = 0; d < DEPTH; ++d) {
        if (lists[d].empty() || !lists[d][i].defined()) { a.ptr[d][nt] = nullptr; a.dtype[d][nt] = 0; continue; }
        TORCH_CHECK(lists[d][i].numel() == numel && lists[d][i].is_non_overlapping_and_dense(), "multi-tensor lists must match and be dense");
        a.ptr[d][nt] = lists[d][i].data_ptr();
        a.dtype[d][nt] = dtype_code(lists[d][i]);
      }
      a.numel[nt] = numel;
      while (c < chunks && nb < kMtaBlocks) {
        a.block_tensor[nb] = (uint8_t)nt;
        a.block_chunk[nb] = (int32_t)c;
        ++nb;
        ++c;
      }
      ++nt;
    }
  }
  flush();
}

void fused_sgd_multi(std::vector<at::Tensor> grads, std::vector<at::Tensor> params, std::vector<at::Tensor> momenta,
                     std::vector<at::Tensor> model_copies, at::Tensor hyper, c10::optional<at::Tensor> found_inf, bool nesterov,
                     bool first_step) {
  if (params.empty()) return;
  TORCH_CHECK(grads.size() == params.size() && momenta.size() == params.size());
  TORCH_CHECK(model_copies.empty() || model_copies.size() == params.size());
  for (auto& p : params) TORCH_CHECK(p.scalar_type() == at::kFloat, "params (masters) must be fp32");
  for (auto& m : momenta) TORCH_CHECK(m.scalar_type() == at::kFloat, "momentum must be fp32");
  TORCH_CHECK(!found_inf.has_value() || hyper.numel() >= 6, "hyper needs slot 5 (momentum_pending) when found_inf is given");
  c10::cuda::CUDAGuard guard(params[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const float* hp = hyper.data_ptr<float>();
  mta_for_each<4>({grads, params, momenta, model_copies}, [&](const MtaArgs<4>& a, int nb) {
    fused_sgd_multi_kernel<<<nb, 256, 0, st>>>(a, hp, fi, nesterov, first_step);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

void multi_tensor_scale(std::vector<at::Tensor> src, std::vector<at::Tensor> dst, double scale, at::Tensor found_inf) {
  if (src.empty()) return;
  TORCH_CHECK(src.size() == dst.size());
  TORCH_CHECK(found_inf.scalar_type() == at::kInt && found_inf.numel() >= 1);
  c10::cuda::CUDAGuard guard(src[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  mta_for_each<2>({src, dst}, [&](const MtaArgs<2>& a, int nb) {
    multi_tensor_scale_kernel<<<nb, 256, 0, st>>>(a, (float)scale, found_inf.data_ptr<int>());
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

void multi_tensor_axpby(std::vector<at::Tensor> x, std::vector<at::Tensor> y, std::vector<at::Tensor> out, double a, double b,
                        at::Tensor found_inf) {
  if (x.empty()) return;
  TORCH_CHECK(x.size() == y.size() && x.size() == out.size());
  TORCH_CHECK(found_inf.scalar_type() == at::kInt && found_inf.numel() >= 1);
  c10::cuda::CUDAGuard guard(x[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  mta_for_each<3>({x, y, out}, [&](const MtaArgs<3>& args, int nb) {
    multi_tensor_axpby_kernel<<<nb, 256, 0, st>>>(args, (float)a, (float)b, found_inf.data_ptr<int>());
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

// Dynamic loss-scale state machine on the device (apex semantics: x2 after `interval` clean steps, /2 and skip on
// overflow).  Also refreshes hyper[4] = grad multiplier = 1/scale, clears hyper[5] (momentum_pending) after an applied
// step and clears found_inf for the next step.
__global__ void amp_update_scale_kernel(float* scale, int* tracker, int* found_inf, float growth, float backoff, int interval, float* hyper,
                                        bool has_pending, float extra_mul) {
  const bool bad = *found_inf != 0;
  if (bad) {
    *scale = fmaxf(*scale * backoff, 1.0f);
    *tracker = 0;
  } else {
    int t = *tracker + 1;
    if (t >= interval) {
      float s = *scale * growth;
      if (isfinite(s)) *scale = s;
      t = 0;
    }
    *tracker = t;
  }
  *found_inf = 0;
  if (hyper) hyper[4] = extra_mul / *scale;
  if (has_pending && !bad) hyper[5] = 0.f;
}

void amp_update_scale(at::Tensor scale, at::Tensor growth_tracker, at::Tensor found_inf, double growth, double backoff, int64_t interval,
                      at::Tensor hyper) {
  TORCH_CHECK(scale.scalar_type() == at::kFloat && growth_tracker.scalar_type() == at::kInt && found_inf.scalar_type() == at::kInt);
  c10::cuda::CUDAGuard guard(scale.device());
  float* hp = hyper.defined() && hyper.numel() >= 5 ? hyper.data_ptr<float>() : nullptr;
  const bool has_pending = hp && hyper.numel() >= 6;
  amp_update_scale_kernel<<<1, 1, 0, at::cuda::getCurrentCUDAStream()>>>(scale.data_ptr<float>(), growth_tracker.data_ptr<int>(),
                                                                         found_inf.data_ptr<int>(), (float)growth, (float)backoff,
                                                                         (int)interval, hp, has_pending, 1.0f);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace ptd
