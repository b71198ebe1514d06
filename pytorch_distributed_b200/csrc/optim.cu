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
//
// Exponential moving average (ModelEma): every update kernel has an HAS_EMA instantiation that also streams an fp32 average
// e of the masters, updated from the new master p as e = fmaf(d, e, w p) with d = hyper[6] and w = hyper[7] = fp32(1 - d)
// (+8 B/element).  d = 0 gives e = p and d = 1 leaves e unchanged, bit for bit.  The found_inf early return skips it with
// the step.  ema_multi applies the same formula to any tensor lists (BatchNorm buffers, optimizers other than these).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {

struct SgdHyper { float lr, momentum, wd, dampening, gmul; };
struct EmaHyper { float d, w; };

__device__ __forceinline__ float ema_update(float e, float p, const EmaHyper& h) { return __fmaf_rn(h.d, e, __fmul_rn(h.w, p)); }

__device__ __forceinline__ SgdHyper load_hyper(const float* h) { return SgdHyper{h[0], h[1], h[2], h[3], h[4]}; }

__device__ __forceinline__ void sgd_update(float g, float& p, float& m, const SgdHyper& h, bool nesterov, bool first) {
  g = g * h.gmul + h.wd * p;
  if (h.momentum != 0.f) {
    m = first ? g : h.momentum * m + (1.f - h.dampening) * g;
    g = nesterov ? g + h.momentum * m : m;
  }
  p -= h.lr * g;
}

// `ema` is the last parameter so that the HAS_EMA = false instantiations keep their parameter offsets (and SASS)
template <typename G, typename C, bool HAS_COPY, bool HAS_EMA>
__global__ void __launch_bounds__(256) fused_sgd_flat_kernel(const G* __restrict__ grad, float* __restrict__ master,
                                                             float* __restrict__ mom, C* __restrict__ copy, int64_t n,
                                                             const float* __restrict__ hyper, const int* __restrict__ found_inf,
                                                             bool nesterov, bool first, float* __restrict__ ema) {
  if (found_inf && *found_inf) return;  // dynamic loss scaling: skip the step on overflow
  const SgdHyper h = load_hyper(hyper);
  EmaHyper eh{};
  if constexpr (HAS_EMA) eh = EmaHyper{hyper[6], hyper[7]};
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
    if constexpr (HAS_EMA) {
      float e[8];
      load8<float>(ema + (v << 3), e);
#pragma unroll
      for (int k = 0; k < 8; ++k) e[k] = ema_update(e[k], p[k], eh);
      store8<float>(ema + (v << 3), e);
    }
  }
  // n is padded to a multiple of 8 by the arena layout; no scalar tail.
}

static void check_ema_flat(const c10::optional<at::Tensor>& ema, int64_t n, const at::Tensor& hyper) {
  if (!ema.has_value()) return;
  TORCH_CHECK(ema->scalar_type() == at::kFloat && ema->numel() == n && ema->is_contiguous() && ema->device() == hyper.device(),
              "the EMA buffer must be a contiguous fp32 tensor with the masters' layout");
  TORCH_CHECK(hyper.numel() >= 8, "hyper needs slots 6, 7 (EMA decay) when an EMA buffer is given");
}

void fused_sgd_flat(at::Tensor grad, at::Tensor master, at::Tensor momentum, c10::optional<at::Tensor> model_copy, at::Tensor hyper,
                    c10::optional<at::Tensor> found_inf, bool nesterov, bool first_step, c10::optional<at::Tensor> ema) {
  const int64_t n = master.numel();
  TORCH_CHECK(n % 8 == 0, "flat optimizer buffers must be padded to a multiple of 8 elements");
  TORCH_CHECK(grad.numel() >= n && momentum.numel() == n, "flat buffer size mismatch");
  TORCH_CHECK(master.scalar_type() == at::kFloat && momentum.scalar_type() == at::kFloat && hyper.scalar_type() == at::kFloat);
  TORCH_CHECK(master.is_contiguous() && momentum.is_contiguous() && grad.is_contiguous());
  TORCH_CHECK(!found_inf.has_value() || hyper.numel() >= 6, "hyper needs slot 5 (momentum_pending) when found_inf is given");
  check_ema_flat(ema, n, hyper);
  c10::cuda::CUDAGuard guard(master.device());
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int grid = (int)std::min<int64_t>((n / 8 + 255) / 256, (int64_t)sms * 8);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  float* mp = master.data_ptr<float>();
  float* vp = momentum.data_ptr<float>();
  const float* hp = hyper.data_ptr<float>();
  float* ep = ema.has_value() ? ema->data_ptr<float>() : nullptr;
#define LAUNCH(G, C, HC, cptr)                                                                                                   \
  do {                                                                                                                          \
    if (ep) fused_sgd_flat_kernel<G, C, HC, true><<<grid, 256, 0, st>>>(reinterpret_cast<const G*>(grad.data_ptr()), mp, vp, cptr, \
                                                                        n, hp, fi, nesterov, first_step, ep);                  \
    else fused_sgd_flat_kernel<G, C, HC, false><<<grid, 256, 0, st>>>(reinterpret_cast<const G*>(grad.data_ptr()), mp, vp, cptr, \
                                                                       n, hp, fi, nesterov, first_step, nullptr);              \
  } while (0)
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

// lists: 0 grad, 1 param (fp32 master), 2 momentum (fp32), 3 model copy (optional: ptr may be null), 4 fp32 EMA (HAS_EMA)
template <bool HAS_EMA>
__global__ void __launch_bounds__(256) fused_sgd_multi_kernel(const __grid_constant__ MtaArgs<HAS_EMA ? 5 : 4> a, const float* __restrict__ hyper,
                                                              const int* __restrict__ found_inf, bool nesterov, bool first) {
  if (found_inf && *found_inf) return;
  const SgdHyper h = load_hyper(hyper);
  EmaHyper eh{};
  if constexpr (HAS_EMA) eh = EmaHyper{hyper[6], hyper[7]};
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
    if constexpr (HAS_EMA) {
      float* e = reinterpret_cast<float*>(a.ptr[4][t]);
      e[i] = ema_update(e[i], pv, eh);
    }
  }
}

// dst = fmaf(d, dst, w * src) with {d, w} = dw[0..1] (fp32 dst, any float src); nothing on found_inf.  lists: 0 src, 1 dst
__global__ void __launch_bounds__(256) ema_multi_kernel(const __grid_constant__ MtaArgs<2> a, const float* __restrict__ dw,
                                                        const int* __restrict__ found_inf) {
  if (found_inf && *found_inf) return;
  const EmaHyper eh{dw[0], dw[1]};
  const int t = a.block_tensor[blockIdx.x];
  const int64_t begin = (int64_t)a.block_chunk[blockIdx.x] * kMtaChunk;
  const int64_t end = min(begin + (int64_t)kMtaChunk, a.numel[t]);
  float* e = reinterpret_cast<float*>(a.ptr[1][t]);
  const int sdt = a.dtype[0][t];
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) e[i] = ema_update(e[i], ld_any(a.ptr[0][t], sdt, i), eh);
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

// launch(a, nb, src): src[slot] is the index in `lists` of the tensor registered in that slot of `a`
template <int DEPTH, typename LaunchFn>
static void mta_for_each(const std::vector<std::vector<at::Tensor>>& lists, LaunchFn&& launch) {
  const size_t n = lists[0].size();
  MtaArgs<DEPTH> a;
  int src[kMtaTensors];
  int nt = 0, nb = 0;
  auto flush = [&]() {
    if (nb > 0) launch(a, nb, static_cast<const int*>(src));
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
      src[nt] = (int)i;
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

// EMA list of a multi-tensor update: empty (no EMA) or one fp32 tensor per master, with the master's strides
static void check_ema_multi(const std::vector<at::Tensor>& ema, const std::vector<at::Tensor>& params, const at::Tensor& hyper) {
  if (ema.empty()) return;
  TORCH_CHECK(ema.size() == params.size(), "the EMA list needs one tensor per parameter");
  TORCH_CHECK(hyper.numel() >= 8, "hyper needs slots 6, 7 (EMA decay) when an EMA list is given");
  for (size_t i = 0; i < ema.size(); ++i)
    TORCH_CHECK(ema[i].scalar_type() == at::kFloat && ema[i].strides() == params[i].strides() && ema[i].numel() == params[i].numel(),
                "EMA tensors must be fp32 with their master's shape and strides");
}

void fused_sgd_multi(std::vector<at::Tensor> grads, std::vector<at::Tensor> params, std::vector<at::Tensor> momenta,
                     std::vector<at::Tensor> model_copies, at::Tensor hyper, c10::optional<at::Tensor> found_inf, bool nesterov,
                     bool first_step, std::vector<at::Tensor> ema) {
  if (params.empty()) return;
  TORCH_CHECK(grads.size() == params.size() && momenta.size() == params.size());
  TORCH_CHECK(model_copies.empty() || model_copies.size() == params.size());
  for (auto& p : params) TORCH_CHECK(p.scalar_type() == at::kFloat, "params (masters) must be fp32");
  for (auto& m : momenta) TORCH_CHECK(m.scalar_type() == at::kFloat, "momentum must be fp32");
  TORCH_CHECK(!found_inf.has_value() || hyper.numel() >= 6, "hyper needs slot 5 (momentum_pending) when found_inf is given");
  check_ema_multi(ema, params, hyper);
  c10::cuda::CUDAGuard guard(params[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const float* hp = hyper.data_ptr<float>();
  if (!ema.empty()) {
    mta_for_each<5>({grads, params, momenta, model_copies, ema}, [&](const MtaArgs<5>& a, int nb, const int*) {
      fused_sgd_multi_kernel<true><<<nb, 256, 0, st>>>(a, hp, fi, nesterov, first_step);
      C10_CUDA_KERNEL_LAUNCH_CHECK();
    });
    return;
  }
  mta_for_each<4>({grads, params, momenta, model_copies}, [&](const MtaArgs<4>& a, int nb, const int*) {
    fused_sgd_multi_kernel<false><<<nb, 256, 0, st>>>(a, hp, fi, nesterov, first_step);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

void ema_multi(std::vector<at::Tensor> src, std::vector<at::Tensor> dst, at::Tensor dw, c10::optional<at::Tensor> found_inf) {
  if (dst.empty()) return;
  TORCH_CHECK(src.size() == dst.size(), "ema_multi: one source per average");
  TORCH_CHECK(dw.scalar_type() == at::kFloat && dw.numel() >= 2 && dw.is_cuda(), "ema_multi: dw = fp32 {d, 1 - d} on the device");
  for (size_t i = 0; i < dst.size(); ++i)
    TORCH_CHECK(dst[i].scalar_type() == at::kFloat && dst[i].strides() == src[i].strides(),
                "ema_multi: averages must be fp32 with their source's strides");
  c10::cuda::CUDAGuard guard(dst[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const float* dp = dw.data_ptr<float>();
  mta_for_each<2>({src, dst}, [&](const MtaArgs<2>& a, int nb, const int*) {
    ema_multi_kernel<<<nb, 256, 0, st>>>(a, dp, fi);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

void multi_tensor_scale(std::vector<at::Tensor> src, std::vector<at::Tensor> dst, double scale, at::Tensor found_inf) {
  if (src.empty()) return;
  TORCH_CHECK(src.size() == dst.size());
  TORCH_CHECK(found_inf.scalar_type() == at::kInt && found_inf.numel() >= 1);
  c10::cuda::CUDAGuard guard(src[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  mta_for_each<2>({src, dst}, [&](const MtaArgs<2>& a, int nb, const int*) {
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
  mta_for_each<3>({x, y, out}, [&](const MtaArgs<3>& args, int nb, const int*) {
    multi_tensor_axpby_kernel<<<nb, 256, 0, st>>>(args, (float)a, (float)b, found_inf.data_ptr<int>());
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

// ---------------------------------------------------------------- LARC layer-wise adaptive rates (apex.parallel.LARC)
// Per parameter tensor p with unscaled gradient g = grad * gmul, wd = hyper[2], lr = hyper[0]:
//   pn = ||p||, gn = ||g||;  if pn != 0 and gn != 0:  f = trust * pn / (gn + pn * wd + eps), clip: f = min(f / lr, 1),
//   g = (g + wd * p) * f;  otherwise g is left as is and gets no weight decay (apex);  then sgd_update with wd = 0.
// Two passes, one CTA per kLarcChunk-element chunk of one tensor (chunks counted from the tensor's first element):
//   larc_norm_*  writes the chunk's fp32 partial sums {sum p^2, sum g^2} to partials[cbase + chunk];
//   larc_sgd_*   adds its tensor's partials in ascending chunk order, forms pn, gn, f and applies the update; chunk 0 of
//                each tensor writes {pn, gn, f} to stats[row] (f = 1 where a norm is zero).
// Within a chunk thread i adds elements 8 (i + 256 k) + j, j = 0..7 then k ascending, and the CTA combines the 256
// thread sums in a fixed tree.  No float atomics: the flat, per-bucket and multi-tensor front ends give the same bits.
// HBM traffic per element (bf16 gradient, bf16 copy): 6 B norm pass + the 20 B of the SGD update.
constexpr int kLarcChunk = kMtaChunk;  // the multi-tensor front end's chunk: its block_chunk is the LARC chunk
constexpr int kLarcThreads = 256;
static_assert(kLarcChunk == kLarcChunkElems, "host.h publishes the LARC chunk size");
static_assert(kLarcChunk % (8 * kLarcThreads) == 0, "a chunk is a whole number of 8-element groups per thread");

struct LarcFactor { float pn, gn, f; bool adapt; };

// per-tensor data of a multi-tensor launch, by slot: first partial, statistics row, first-step flag
struct LarcSlots {
  int32_t cbase[kMtaTensors];
  int32_t row[kMtaTensors];
  uint8_t first[kMtaTensors];
};

__device__ __forceinline__ float ldcg_f(const float* p) { return __ldcg(p); }
__device__ __forceinline__ float ldcg_f(const __nv_bfloat16* p) { return __bfloat162float(__ldcg(p)); }
__device__ __forceinline__ float ldcg_f(const __half* p) { return __half2float(__ldcg(p)); }

// the one summation order of every front end: elements j < cnt of one 8-element group
__device__ __forceinline__ void larc_acc8(const float (&p)[8], const float (&g)[8], float gmul, int cnt, float& sp, float& sg) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < cnt) {
      sp = __fmaf_rn(p[j], p[j], sp);
      const float u = __fmul_rn(g[j], gmul);
      sg = __fmaf_rn(u, u, sg);
    }
  }
}

// CTA sum of (a, b) in a fixed order: butterfly within each warp, then warp 0 over the warp totals.  Valid in thread 0.
__device__ __forceinline__ float2 larc_cta_sum(float a, float b) {
  __shared__ float2 red[kLarcThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = __fadd_rn(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = make_float2(a, b);
  __syncthreads();
  if (w == 0) {
    const float2 v = l < kLarcThreads / 32 ? red[l] : make_float2(0.f, 0.f);
    a = v.x;
    b = v.y;
#pragma unroll
    for (int o = kLarcThreads / 64; o > 0; o >>= 1) {
      a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, o));
      b = __fadd_rn(b, __shfl_xor_sync(0xffffffffu, b, o));
    }
  }
  return make_float2(a, b);
}

__device__ __forceinline__ LarcFactor larc_factor(const float2* part, int64_t nchunks, const SgdHyper& h, float trust, float eps, bool clip) {
  float sp = 0.f, sg = 0.f;
  for (int64_t c = 0; c < nchunks; ++c) {
    const float2 v = part[c];
    sp = __fadd_rn(sp, v.x);
    sg = __fadd_rn(sg, v.y);
  }
  LarcFactor r;
  r.pn = __fsqrt_rn(sp);
  r.gn = __fsqrt_rn(sg);
  r.adapt = r.pn != 0.f && r.gn != 0.f;
  r.f = 1.f;
  if (r.adapt) {
    r.f = __fdiv_rn(__fmul_rn(trust, r.pn), __fadd_rn(__fmaf_rn(r.pn, h.wd, r.gn), eps));
    if (clip) r.f = fminf(__fdiv_rn(r.f, h.lr), 1.f);
  }
  return r;
}

// Not inlined: the compiler may contract sgd_update's products into FMAs differently in different callers, and the flat
// and multi-tensor kernels must give the same bits.  One compiled body serves both; scalar arguments and a float2 result
// {p, m} keep the call in registers (no addressable arguments, so nothing goes through local memory).
__device__ __noinline__ float2 larc_update(float g, float p, float m, float f, bool adapt, float lr, float mom, float wd, float damp,
                                           float gmul, bool nesterov, bool first) {
  g = __fmul_rn(g, gmul);
  if (adapt) g = __fmul_rn(__fmaf_rn(wd, p, g), f);
  sgd_update(g, p, m, SgdHyper{lr, mom, 0.f, damp, 1.f}, nesterov, first);
  return make_float2(p, m);
}

__device__ __forceinline__ void larc_apply(float g, float& p, float& m, const LarcFactor& r, const SgdHyper& h, bool nesterov, bool first) {
  const float2 pm = larc_update(g, p, m, r.f, r.adapt, h.lr, h.momentum, h.wd, h.dampening, h.gmul, nesterov, first);
  p = pm.x;
  m = pm.y;
}

__device__ __forceinline__ void larc_write_stats(float* stats, int64_t row, const LarcFactor& r) {
  stats[3 * row] = r.pn;
  stats[3 * row + 1] = r.gn;
  stats[3 * row + 2] = r.f;
}

// Flat front end.  info[t] = {element offset in the flat buffers, numel, first chunk, statistics row}, tensors in
// ascending offset order; chunk_tensor[q] = tensor of global chunk q.  CTA b runs chunk chunk_lo + b.
struct LarcChunk { int64_t off, begin, len, cbase, nchunks, row, c; };

__device__ __forceinline__ LarcChunk larc_chunk(const int32_t* chunk_tensor, const int64_t* info, int64_t q) {
  const int64_t* e = info + 4 * chunk_tensor[q];
  LarcChunk k;
  k.off = e[0];
  k.cbase = e[2];
  k.row = e[3];
  k.c = q - k.cbase;
  k.begin = k.c * kLarcChunk;
  k.len = min((int64_t)kLarcChunk, e[1] - k.begin);
  k.nchunks = (e[1] + kLarcChunk - 1) / kLarcChunk;
  return k;
}

template <typename G>
__global__ void __launch_bounds__(kLarcThreads) larc_norm_flat_kernel(const G* __restrict__ grad, const float* __restrict__ master,
                                                                      const int32_t* __restrict__ chunk_tensor, const int64_t* __restrict__ info,
                                                                      int64_t chunk_lo, float2* __restrict__ partials,
                                                                      const float* __restrict__ hyper, const int* __restrict__ found_inf) {
  if (found_inf && *found_inf) return;
  const int64_t q = chunk_lo + blockIdx.x;
  const LarcChunk k = larc_chunk(chunk_tensor, info, q);
  const G* gp = grad + k.off + k.begin;
  const float* pp = master + k.off + k.begin;
  const float gmul = hyper[4];
  float sp = 0.f, sg = 0.f;
  for (int64_t i = 8 * threadIdx.x; i < k.len; i += 8 * kLarcThreads) {
    float p[8], g[8];
    const int cnt = (int)min((int64_t)8, k.len - i);
    if (cnt == 8) {
      load8<G>(gp + i, g, /*sys=*/true);  // arena: bypass L1, as fused_sgd_flat
      load8<float>(pp + i, p);
    } else {
      for (int j = 0; j < cnt; ++j) {
        g[j] = ldcg_f(gp + i + j);
        p[j] = pp[i + j];
      }
    }
    larc_acc8(p, g, gmul, cnt, sp, sg);
  }
  const float2 s = larc_cta_sum(sp, sg);
  if (threadIdx.x == 0) partials[q] = s;
}

template <typename G, typename C, bool HAS_COPY, bool HAS_EMA>
__global__ void __launch_bounds__(kLarcThreads) larc_sgd_flat_kernel(const G* __restrict__ grad, float* __restrict__ master, float* __restrict__ mom,
                                                                     C* __restrict__ copy, const int32_t* __restrict__ chunk_tensor,
                                                                     const int64_t* __restrict__ info, int64_t chunk_lo,
                                                                     const float2* __restrict__ partials, float* __restrict__ stats,
                                                                     const float* __restrict__ hyper, const int* __restrict__ found_inf,
                                                                     bool nesterov, bool first, float trust, float eps, bool clip,
                                                                     float* __restrict__ ema) {
  if (found_inf && *found_inf) return;  // dynamic loss scaling: skip the step on overflow
  const SgdHyper h = load_hyper(hyper);
  EmaHyper eh{};
  if constexpr (HAS_EMA) eh = EmaHyper{hyper[6], hyper[7]};
  first = first || (found_inf && hyper[5] != 0.f);
  const LarcChunk k = larc_chunk(chunk_tensor, info, chunk_lo + blockIdx.x);
  const LarcFactor r = larc_factor(partials + k.cbase, k.nchunks, h, trust, eps, clip);
  if (k.c == 0 && threadIdx.x == 0) larc_write_stats(stats, k.row, r);
  const int64_t base = k.off + k.begin;
  for (int64_t i = 8 * threadIdx.x; i < k.len; i += 8 * kLarcThreads) {
    const int64_t e = base + i;
    if (k.len - i >= 8) {
      float g[8], p[8], m[8];
      load8<G>(grad + e, g, /*sys=*/true);
      load8<float>(master + e, p);
      load8<float>(mom + e, m);
#pragma unroll
      for (int j = 0; j < 8; ++j) larc_apply(g[j], p[j], m[j], r, h, nesterov, first);
      store8<float>(master + e, p);
      store8<float>(mom + e, m);
      if constexpr (HAS_COPY) store8<C>(copy + e, p);
      if constexpr (HAS_EMA) {
        float a[8];
        load8<float>(ema + e, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = ema_update(a[j], p[j], eh);
        store8<float>(ema + e, a);
      }
    } else {
      for (int64_t x = e; x < base + k.len; ++x) {
        float p = master[x], m = mom[x];
        larc_apply(ldcg_f(grad + x), p, m, r, h, nesterov, first);
        master[x] = p;
        mom[x] = m;
        if constexpr (HAS_COPY) {
          if constexpr (std::is_same<C, __nv_bfloat16>::value) copy[x] = __float2bfloat16_rn(p);
          else copy[x] = __float2half_rn(p);
        }
        if constexpr (HAS_EMA) ema[x] = ema_update(ema[x], p, eh);
      }
    }
  }
}

// Multi-tensor front end: lists 0 grad, 1 fp32 master (norm pass: lists 0 grad, 1 master).
__global__ void __launch_bounds__(kLarcThreads) larc_norm_multi_kernel(const __grid_constant__ MtaArgs<2> a, const __grid_constant__ LarcSlots s,
                                                                       float2* __restrict__ partials, const float* __restrict__ hyper,
                                                                       const int* __restrict__ found_inf) {
  if (found_inf && *found_inf) return;
  const int t = a.block_tensor[blockIdx.x];
  const int c = a.block_chunk[blockIdx.x];
  const int64_t begin = (int64_t)c * kLarcChunk;
  const int64_t len = min((int64_t)kLarcChunk, a.numel[t] - begin);
  const float* pp = reinterpret_cast<const float*>(a.ptr[1][t]) + begin;
  const int gdt = a.dtype[0][t];
  const float gmul = hyper[4];
  float sp = 0.f, sg = 0.f;
  for (int64_t i = 8 * threadIdx.x; i < len; i += 8 * kLarcThreads) {
    float p[8], g[8];
    const int cnt = (int)min((int64_t)8, len - i);
    for (int j = 0; j < cnt; ++j) {
      g[j] = ld_any(a.ptr[0][t], gdt, begin + i + j);
      p[j] = pp[i + j];
    }
    larc_acc8(p, g, gmul, cnt, sp, sg);
  }
  const float2 r = larc_cta_sum(sp, sg);
  if (threadIdx.x == 0) partials[s.cbase[t] + c] = r;
}

// lists: 0 grad, 1 fp32 master, 2 momentum (fp32), 3 model copy (optional: ptr may be null), 4 fp32 EMA (HAS_EMA)
template <bool HAS_EMA>
__global__ void __launch_bounds__(kLarcThreads) larc_sgd_multi_kernel(const __grid_constant__ MtaArgs<HAS_EMA ? 5 : 4> a, const __grid_constant__ LarcSlots s,
                                                                      const float2* __restrict__ partials, float* __restrict__ stats,
                                                                      const float* __restrict__ hyper, const int* __restrict__ found_inf,
                                                                      bool nesterov, float trust, float eps, bool clip) {
  if (found_inf && *found_inf) return;
  const SgdHyper h = load_hyper(hyper);
  EmaHyper eh{};
  if constexpr (HAS_EMA) eh = EmaHyper{hyper[6], hyper[7]};
  const int t = a.block_tensor[blockIdx.x];
  const bool first = s.first[t] || (found_inf && hyper[5] != 0.f);
  const int c = a.block_chunk[blockIdx.x];
  const LarcFactor r = larc_factor(partials + s.cbase[t], (a.numel[t] + kLarcChunk - 1) / kLarcChunk, h, trust, eps, clip);
  if (c == 0 && threadIdx.x == 0) larc_write_stats(stats, s.row[t], r);
  const int64_t begin = (int64_t)c * kLarcChunk;
  const int64_t end = min(begin + (int64_t)kLarcChunk, a.numel[t]);
  float* p = reinterpret_cast<float*>(a.ptr[1][t]);
  float* m = reinterpret_cast<float*>(a.ptr[2][t]);
  const int gdt = a.dtype[0][t], cdt = a.dtype[3][t];
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    float pv = p[i], mv = m[i];
    larc_apply(ld_any(a.ptr[0][t], gdt, i), pv, mv, r, h, nesterov, first);
    p[i] = pv;
    m[i] = mv;
    if (a.ptr[3][t]) st_any(a.ptr[3][t], cdt, i, pv);
    if constexpr (HAS_EMA) {
      float* e = reinterpret_cast<float*>(a.ptr[4][t]);
      e[i] = ema_update(e[i], pv, eh);
    }
  }
}

static void check_larc_common(const at::Tensor& hyper, const c10::optional<at::Tensor>& found_inf, const at::Tensor& stats, double trust,
                              double eps) {
  TORCH_CHECK(hyper.scalar_type() == at::kFloat && hyper.numel() >= 5, "hyper must be fp32 with slots 0..4");
  TORCH_CHECK(!found_inf.has_value() || hyper.numel() >= 6, "hyper needs slot 5 (momentum_pending) when found_inf is given");
  TORCH_CHECK(stats.scalar_type() == at::kFloat && stats.is_contiguous(), "LARC statistics must be a contiguous fp32 tensor");
  TORCH_CHECK(std::isfinite(trust) && trust > 0 && std::isfinite(eps) && eps >= 0, "LARC needs trust_coefficient > 0 and eps >= 0");
}

// calls fn(G{}, C{}, has_copy) with the gradient / model-copy types of fused_sgd_flat's instantiations
template <typename Fn>
static void larc_flat_types(at::ScalarType gt, c10::optional<at::ScalarType> ct, Fn&& fn) {
  auto with_copy = [&](auto g) {
    if (!ct.has_value()) fn(g, float{}, std::false_type{});
    else if (*ct == at::kBFloat16) fn(g, __nv_bfloat16{}, std::true_type{});
    else if (*ct == at::kHalf) fn(g, __half{}, std::true_type{});
    else TORCH_CHECK(false, "unsupported model copy dtype");
  };
  if (gt == at::kBFloat16) with_copy(__nv_bfloat16{});
  else if (gt == at::kHalf) with_copy(__half{});
  else if (gt == at::kFloat) with_copy(float{});
  else TORCH_CHECK(false, "unsupported gradient dtype");
}

void larc_sgd_flat(at::Tensor grad, at::Tensor master, at::Tensor momentum, c10::optional<at::Tensor> model_copy, at::Tensor hyper,
                   c10::optional<at::Tensor> found_inf, bool nesterov, bool first_step, at::Tensor chunk_tensor, at::Tensor info,
                   int64_t chunk_lo, int64_t chunk_hi, at::Tensor partials, at::Tensor stats, double trust, double eps, bool clip,
                   c10::optional<at::Tensor> ema) {
  const int64_t n = master.numel();
  TORCH_CHECK(grad.numel() >= n && momentum.numel() == n, "flat buffer size mismatch");
  TORCH_CHECK(master.scalar_type() == at::kFloat && momentum.scalar_type() == at::kFloat);
  TORCH_CHECK(master.is_contiguous() && momentum.is_contiguous() && grad.is_contiguous());
  check_larc_common(hyper, found_inf, stats, trust, eps);
  TORCH_CHECK(chunk_tensor.scalar_type() == at::kInt && info.scalar_type() == at::kLong && info.dim() == 2 && info.size(1) == 4 &&
                  chunk_tensor.is_contiguous() && info.is_contiguous(), "LARC chunk table: int32 [chunks] and int64 [tensors, 4]");
  TORCH_CHECK(0 <= chunk_lo && chunk_lo <= chunk_hi && chunk_hi <= chunk_tensor.numel(), "LARC chunk range outside the table");
  TORCH_CHECK(partials.scalar_type() == at::kFloat && partials.is_contiguous() && partials.numel() >= 2 * chunk_tensor.numel(),
              "LARC partials: fp32 [2 * chunks]");
  if (model_copy.has_value()) TORCH_CHECK(model_copy->numel() == n && model_copy->is_contiguous());
  check_ema_flat(ema, n, hyper);
  if (chunk_hi == chunk_lo) return;
  c10::cuda::CUDAGuard guard(master.device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const int grid = (int)(chunk_hi - chunk_lo);
  const int32_t* ct = chunk_tensor.data_ptr<int32_t>();
  const int64_t* inf = info.data_ptr<int64_t>();
  float2* part = reinterpret_cast<float2*>(partials.data_ptr<float>());
  const float* hp = hyper.data_ptr<float>();
  larc_flat_types(grad.scalar_type(), model_copy.has_value() ? c10::optional<at::ScalarType>(model_copy->scalar_type()) : c10::nullopt,
                  [&](auto g, auto c, auto has_copy) {
                    using G = decltype(g);
                    using C = decltype(c);
                    const G* gp = reinterpret_cast<const G*>(grad.data_ptr());
                    larc_norm_flat_kernel<G><<<grid, kLarcThreads, 0, st>>>(gp, master.data_ptr<float>(), ct, inf, chunk_lo, part, hp, fi);
                    C10_CUDA_KERNEL_LAUNCH_CHECK();
                    C* cp = has_copy ? reinterpret_cast<C*>(model_copy->data_ptr()) : nullptr;
                    if (ema.has_value())
                      larc_sgd_flat_kernel<G, C, decltype(has_copy)::value, true><<<grid, kLarcThreads, 0, st>>>(
                          gp, master.data_ptr<float>(), momentum.data_ptr<float>(), cp, ct, inf, chunk_lo, part, stats.data_ptr<float>(), hp,
                          fi, nesterov, first_step, (float)trust, (float)eps, clip, ema->data_ptr<float>());
                    else
                      larc_sgd_flat_kernel<G, C, decltype(has_copy)::value, false><<<grid, kLarcThreads, 0, st>>>(
                          gp, master.data_ptr<float>(), momentum.data_ptr<float>(), cp, ct, inf, chunk_lo, part, stats.data_ptr<float>(), hp,
                          fi, nesterov, first_step, (float)trust, (float)eps, clip, nullptr);
                    C10_CUDA_KERNEL_LAUNCH_CHECK();
                  });
}

void larc_sgd_multi(std::vector<at::Tensor> grads, std::vector<at::Tensor> params, std::vector<at::Tensor> momenta,
                    std::vector<c10::optional<at::Tensor>> model_copies, at::Tensor hyper, c10::optional<at::Tensor> found_inf, bool nesterov,
                    std::vector<bool> first, std::vector<int64_t> rows, at::Tensor stats, double trust, double eps, bool clip,
                    std::vector<at::Tensor> ema) {
  const size_t n = params.size();
  if (n == 0) return;
  TORCH_CHECK(grads.size() == n && momenta.size() == n && first.size() == n && rows.size() == n, "LARC lists must have one entry per tensor");
  TORCH_CHECK(model_copies.empty() || model_copies.size() == n);
  for (auto& p : params) TORCH_CHECK(p.scalar_type() == at::kFloat, "params (masters) must be fp32");
  for (auto& m : momenta) TORCH_CHECK(m.scalar_type() == at::kFloat, "momentum must be fp32");
  check_larc_common(hyper, found_inf, stats, trust, eps);
  check_ema_multi(ema, params, hyper);
  std::vector<at::Tensor> copies;
  for (auto& c : model_copies) copies.push_back(c.has_value() ? *c : at::Tensor());
  std::vector<int32_t> cbase(n);
  int64_t chunks = 0;
  for (size_t i = 0; i < n; ++i) {
    TORCH_CHECK(rows[i] >= 0 && 3 * (rows[i] + 1) <= stats.numel(), "LARC statistics row outside the buffer");
    cbase[i] = (int32_t)chunks;
    chunks += (params[i].numel() + kLarcChunk - 1) / kLarcChunk;
  }
  TORCH_CHECK(chunks < INT32_MAX, "too many LARC chunks");
  c10::cuda::CUDAGuard guard(params[0].device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const float* hp = hyper.data_ptr<float>();
  at::Tensor partials = at::empty({std::max<int64_t>(2 * chunks, 2)}, params[0].options());
  float2* part = reinterpret_cast<float2*>(partials.data_ptr<float>());
  auto slots = [&](const int* src, int count) {
    LarcSlots s{};
    for (int k = 0; k < count; ++k) {
      s.cbase[k] = cbase[src[k]];
      s.row[k] = (int32_t)rows[src[k]];
      s.first[k] = first[src[k]] ? 1 : 0;
    }
    return s;
  };
  // every norm of the list is formed before any update launch
  mta_for_each<2>({grads, params}, [&](const MtaArgs<2>& a, int nb, const int* src) {
    larc_norm_multi_kernel<<<nb, kLarcThreads, 0, st>>>(a, slots(src, a.block_tensor[nb - 1] + 1), part, hp, fi);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
  if (!ema.empty()) {
    mta_for_each<5>({grads, params, momenta, copies, ema}, [&](const MtaArgs<5>& a, int nb, const int* src) {
      larc_sgd_multi_kernel<true><<<nb, kLarcThreads, 0, st>>>(a, slots(src, a.block_tensor[nb - 1] + 1), part, stats.data_ptr<float>(), hp, fi,
                                                               nesterov, (float)trust, (float)eps, clip);
      C10_CUDA_KERNEL_LAUNCH_CHECK();
    });
    return;
  }
  mta_for_each<4>({grads, params, momenta, copies}, [&](const MtaArgs<4>& a, int nb, const int* src) {
    larc_sgd_multi_kernel<false><<<nb, kLarcThreads, 0, st>>>(a, slots(src, a.block_tensor[nb - 1] + 1), part, stats.data_ptr<float>(), hp, fi,
                                                              nesterov, (float)trust, (float)eps, clip);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
}

// ---------------------------------------------------------------- global-norm gradient clipping (torch.nn.utils.clip_grad_norm_)
// total = ||g * hyper[4]||_2 over every parameter of the step; coef = clamp(max_norm / (total + 1e-6), max = 1) with
// max_norm = hyper[8] (a NaN total gives a NaN coef, an infinite one 0).  The update kernels above then run unchanged with a
// clipped copy of each group's hyper in which slot 4 is hyper[4] * coef, so weight decay, momentum and LARC see g * coef.
//   grad_sumsq_*   one fp32 partial sum of (g * hyper[4])^2 per chunk, over the LARC chunks (flat: its chunk table; multi:
//                  chunks counted from each tensor's first element) and in LARC's per-chunk order;
//   clip_finalize  one CTA: adds the partials in a fixed order, writes total, the clipped hyper copies and counts coef < 1.
// All three return at once on found_inf, so a skipped step leaves total, the copies and the count as they were.
// HBM traffic: the gradient once (2 B/element with a bf16 arena); the finalize reads 4 B per chunk.
constexpr int kClipGroups = 16;
constexpr int kClipHyperSlots = 9;  // lr, momentum, wd, dampening, gmul, momentum_pending, EMA d, EMA 1 - d, max_norm

struct ClipHypers {
  const float* src[kClipGroups];
  float* dst[kClipGroups];
  int32_t len[kClipGroups];
  int32_t n;
};

// elements j < cnt of one 8-element group, in larc_acc8's order
__device__ __forceinline__ void sumsq_acc8(const float (&g)[8], float gmul, int cnt, float& s) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < cnt) {
      const float u = __fmul_rn(g[j], gmul);
      s = __fmaf_rn(u, u, s);
    }
  }
}

template <typename G>
__global__ void __launch_bounds__(kLarcThreads) grad_sumsq_flat_kernel(const G* __restrict__ grad, const int32_t* __restrict__ chunk_tensor,
                                                                       const int64_t* __restrict__ info, float* __restrict__ partials,
                                                                       const float* __restrict__ hyper, const int* __restrict__ found_inf) {
  if (found_inf && *found_inf) return;
  const int64_t q = blockIdx.x;
  const LarcChunk k = larc_chunk(chunk_tensor, info, q);
  const G* gp = grad + k.off + k.begin;
  const float gmul = hyper[4];
  float s = 0.f;
  for (int64_t i = 8 * threadIdx.x; i < k.len; i += 8 * kLarcThreads) {
    float g[8];
    const int cnt = (int)min((int64_t)8, k.len - i);
    if (cnt == 8) {
      load8<G>(gp + i, g, /*sys=*/true);  // arena: bypass L1, as fused_sgd_flat
    } else {
      for (int j = 0; j < cnt; ++j) g[j] = ldcg_f(gp + i + j);
    }
    sumsq_acc8(g, gmul, cnt, s);
  }
  const float2 r = larc_cta_sum(s, 0.f);
  if (threadIdx.x == 0) partials[q] = r.x;
}

// list 0: gradients (any float dtype); the partial of chunk c of slot t goes to partials[s.cbase[t] + c]
__global__ void __launch_bounds__(kLarcThreads) grad_sumsq_multi_kernel(const __grid_constant__ MtaArgs<1> a, const __grid_constant__ LarcSlots s,
                                                                        float* __restrict__ partials, const float* __restrict__ hyper,
                                                                        const int* __restrict__ found_inf) {
  if (found_inf && *found_inf) return;
  const int t = a.block_tensor[blockIdx.x];
  const int c = a.block_chunk[blockIdx.x];
  const int64_t begin = (int64_t)c * kLarcChunk;
  const int64_t len = min((int64_t)kLarcChunk, a.numel[t] - begin);
  const int gdt = a.dtype[0][t];
  const float gmul = hyper[4];
  float acc = 0.f;
  for (int64_t i = 8 * threadIdx.x; i < len; i += 8 * kLarcThreads) {
    float g[8];
    const int cnt = (int)min((int64_t)8, len - i);
    for (int j = 0; j < cnt; ++j) g[j] = ld_any(a.ptr[0][t], gdt, begin + i + j);
    sumsq_acc8(g, gmul, cnt, acc);
  }
  const float2 r = larc_cta_sum(acc, 0.f);
  if (threadIdx.x == 0) partials[s.cbase[t] + c] = r.x;
}

// Thread i adds partials i, i + 256, ... in ascending order, then the CTA combines the thread sums in larc_cta_sum's tree.
__global__ void __launch_bounds__(kLarcThreads) clip_finalize_kernel(const float* __restrict__ partials, int64_t nparts,
                                                                     const __grid_constant__ ClipHypers h, const int* __restrict__ found_inf,
                                                                     float* __restrict__ total, int* __restrict__ count) {
  if (found_inf && *found_inf) return;
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < nparts; i += kLarcThreads) s = __fadd_rn(s, partials[i]);
  const float2 r = larc_cta_sum(s, 0.f);
  __shared__ float coef_s;
  if (threadIdx.x == 0) {
    const float tn = __fsqrt_rn(r.x);
    const float max_norm = h.src[0][8];
    float coef = __fdiv_rn(max_norm, __fadd_rn(tn, 1e-6f));
    coef = coef > 1.f ? 1.f : coef;  // torch.clamp(max=1): NaN stays NaN (fminf would return 1)
    *total = tn;
    if (coef < 1.f) *count += 1;
    coef_s = coef;
  }
  __syncthreads();
  const float coef = coef_s;
  for (int g = 0; g < h.n; ++g)
    for (int k = threadIdx.x; k < h.len[g]; k += kLarcThreads) h.dst[g][k] = k == 4 ? __fmul_rn(h.src[g][4], coef) : h.src[g][k];
}

void grad_sumsq_flat(at::Tensor grad, at::Tensor chunk_tensor, at::Tensor info, at::Tensor partials, at::Tensor hyper,
                     c10::optional<at::Tensor> found_inf) {
  TORCH_CHECK(grad.is_contiguous() && hyper.scalar_type() == at::kFloat && hyper.numel() >= 5, "grad_sumsq_flat: contiguous arena, fp32 hyper");
  TORCH_CHECK(chunk_tensor.scalar_type() == at::kInt && info.scalar_type() == at::kLong && info.dim() == 2 && info.size(1) == 4 &&
                  chunk_tensor.is_contiguous() && info.is_contiguous(), "chunk table: int32 [chunks] and int64 [tensors, 4]");
  TORCH_CHECK(partials.scalar_type() == at::kFloat && partials.is_contiguous() && partials.numel() >= chunk_tensor.numel(),
              "grad_sumsq_flat: fp32 partials, one per chunk");
  const int64_t chunks = chunk_tensor.numel();
  if (chunks == 0) return;
  TORCH_CHECK(chunks < INT32_MAX, "too many chunks");
  c10::cuda::CUDAGuard guard(grad.device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  const int32_t* ct = chunk_tensor.data_ptr<int32_t>();
  const int64_t* inf = info.data_ptr<int64_t>();
  const auto gt = grad.scalar_type();
  auto launch = [&](auto g) {
    using G = decltype(g);
    grad_sumsq_flat_kernel<G><<<(int)chunks, kLarcThreads, 0, st>>>(reinterpret_cast<const G*>(grad.data_ptr()), ct, inf,
                                                                    partials.data_ptr<float>(), hyper.data_ptr<float>(), fi);
  };
  if (gt == at::kBFloat16) launch(__nv_bfloat16{});
  else if (gt == at::kHalf) launch(__half{});
  else if (gt == at::kFloat) launch(float{});
  else TORCH_CHECK(false, "unsupported gradient dtype");
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

int64_t grad_sumsq_multi(std::vector<at::Tensor> grads, at::Tensor hyper, c10::optional<at::Tensor> found_inf, at::Tensor partials,
                         int64_t partial_off) {
  const size_t n = grads.size();
  std::vector<int32_t> cbase(n);
  int64_t chunks = partial_off;
  for (size_t i = 0; i < n; ++i) {
    cbase[i] = (int32_t)chunks;
    chunks += (grads[i].numel() + kLarcChunk - 1) / kLarcChunk;
  }
  TORCH_CHECK(partial_off >= 0 && chunks < INT32_MAX, "grad_sumsq_multi: partial offset out of range");
  TORCH_CHECK(partials.scalar_type() == at::kFloat && partials.is_contiguous() && partials.numel() >= chunks,
              "grad_sumsq_multi: fp32 partials with room for every chunk");
  TORCH_CHECK(hyper.scalar_type() == at::kFloat && hyper.numel() >= 5, "hyper must be fp32 with slots 0..4");
  if (n == 0) return chunks;
  c10::cuda::CUDAGuard guard(partials.device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  mta_for_each<1>({grads}, [&](const MtaArgs<1>& a, int nb, const int* src) {
    LarcSlots s{};
    for (int k = 0; k <= a.block_tensor[nb - 1]; ++k) s.cbase[k] = cbase[src[k]];
    grad_sumsq_multi_kernel<<<nb, kLarcThreads, 0, st>>>(a, s, partials.data_ptr<float>(), hyper.data_ptr<float>(), fi);
    C10_CUDA_KERNEL_LAUNCH_CHECK();
  });
  return chunks;
}

void clip_finalize(at::Tensor partials, int64_t nparts, std::vector<at::Tensor> hypers, std::vector<at::Tensor> clipped,
                   c10::optional<at::Tensor> found_inf, at::Tensor total, at::Tensor count) {
  TORCH_CHECK(!hypers.empty() && hypers.size() <= (size_t)kClipGroups && clipped.size() == hypers.size(),
              "clip_finalize: 1 to ", kClipGroups, " hyper tensors, each with its clipped copy");
  TORCH_CHECK(partials.scalar_type() == at::kFloat && partials.is_contiguous() && 0 <= nparts && nparts <= partials.numel(),
              "clip_finalize: fp32 partials");
  TORCH_CHECK(total.scalar_type() == at::kFloat && total.numel() >= 1 && count.scalar_type() == at::kInt && count.numel() >= 1,
              "clip_finalize: fp32 total and int32 count");
  ClipHypers h{};
  for (size_t g = 0; g < hypers.size(); ++g) {
    TORCH_CHECK(hypers[g].scalar_type() == at::kFloat && hypers[g].is_contiguous() && hypers[g].numel() >= kClipHyperSlots,
                "clip_finalize: hyper needs slot 8 (max_norm)");
    TORCH_CHECK(clipped[g].scalar_type() == at::kFloat && clipped[g].is_contiguous() && clipped[g].numel() == hypers[g].numel(),
                "clip_finalize: the clipped copy must match its hyper");
    h.src[g] = hypers[g].data_ptr<float>();
    h.dst[g] = clipped[g].data_ptr<float>();
    h.len[g] = (int32_t)hypers[g].numel();
  }
  h.n = (int32_t)hypers.size();
  c10::cuda::CUDAGuard guard(partials.device());
  const int* fi = found_inf.has_value() ? reinterpret_cast<const int*>(found_inf->data_ptr()) : nullptr;
  clip_finalize_kernel<<<1, kLarcThreads, 0, at::cuda::getCurrentCUDAStream()>>>(partials.data_ptr<float>(), nparts, h, fi,
                                                                                  total.data_ptr<float>(), count.data_ptr<int>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
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
