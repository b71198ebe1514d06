// Fused multi-tensor collectives over NVLink / NVSwitch peer memory (sm_90a).
//
//   K1  fused_allreduce   : (cast+scale+pack) -> barrier -> reduce-scatter+all-gather -> barrier -> (unpack)
//                           one kernel per gradient bucket, launched from the backward hooks.
//                           Variants: two-shot / one-shot, NVLS multimem / plain P2P.
//   K2  fused_broadcast   : root packs its tensors and multicasts them; peers unpack. One barrier.
//   K3  barrier           : signal-pad barrier, no payload.
//   K4  metrics_allreduce : top-1/top-5 counting + low-latency (flag-in-payload) all-reduce of
//                           {loss, acc1, acc5}; one single-CTA kernel, no separate barrier.
//
// These replace, for the reference call sites:
//   loss.backward() under DDP  -> NCCL bucket all-reduce      (/root/reference/distributed.py:147,268)
//   DDP ctor / forward         -> rank-0 param/buffer bcast    (/root/reference/distributed.py:147,250)
//   dist.barrier()             -> (/root/reference/distributed.py:256,303)
//   accuracy() + 3x reduce_mean-> (/root/reference/distributed.py:254-260,381-395)
//
// Work decomposition (K1/K2): the bucket owns a contiguous range of the symmetric arena. CTA b owns the
// sub-range [b*block_elems, (b+1)*block_elems) on EVERY rank, so all cross-GPU dependencies are between CTAs with
// the same blockIdx.x and a per-CTA flag barrier is enough (no grid-wide sync, no host involvement).
// A static segment table maps each CTA's range back onto the (scattered) gradient tensors; the tensor base
// pointers of this step travel in the kernel parameters.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {

struct PtrPack {
  void* ptr[kMaxPtrs];
  uint8_t dtype[kMaxPtrs];
};

struct PlanArgs {
  const int32_t* seg_begin;  // [grid + 1]
  const Seg* segs;
  int64_t data_off_bytes;    // arena offset (bytes) of this plan's element 0
  int64_t block_elems;       // elements per CTA range (multiple of world * 8)
  uint32_t* plan_calls;      // local per-CTA call counter (double buffering for broadcast)
  uint32_t* found_inf;       // symmetric-pad relative: nullptr => no non-finite check
  float scale;
  int writeback;             // 1 => unpack the reduced values into the tensors
  int root;                  // broadcast root
  int flags;                 // kPrepacked: the gradients already live in the arena (bucket views): no pack pass, the scale
                             //             is applied to the REDUCED values instead
  int64_t result_off_bytes;  // one-shot: arena offset (bytes) of the range that receives the reduced values (-1: third
                             //           region of the plan's own allocation)
};
constexpr int kPrepacked = 1;

constexpr int kThreads = 512;

// ---------------------------------------------------------------- segment <-> arena movers
template <typename W, typename S>
__device__ __forceinline__ void pack_seg(const S* __restrict__ src, W* __restrict__ dst, int len, float scale) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  const int nvec = aligned ? (len >> 3) : 0;
  int v = threadIdx.x;
  // 4 independent 16/32-byte loads in flight per thread: a 32-CTA kernel has to pull its weight on HBM
  for (; v + 3 * (int)blockDim.x < nvec; v += 4 * blockDim.x) {
    float f[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u) load8<S>(src + ((v + u * (int)blockDim.x) << 3), f[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
#pragma unroll
      for (int k = 0; k < 8; ++k) f[u][k] *= scale;
      store8<W>(dst + ((v + u * (int)blockDim.x) << 3), f[u]);
    }
  }
  for (; v < nvec; v += blockDim.x) {
    float f[8];
    load8<S>(src + (v << 3), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] *= scale;
    store8<W>(dst + (v << 3), f);
  }
  for (int i = (nvec << 3) + threadIdx.x; i < len; i += blockDim.x) dst[i] = from_f32<W>(to_f32<S>(src[i]) * scale);
}

template <typename W, typename D>
__device__ __forceinline__ bool unpack_seg(const W* __restrict__ src, D* __restrict__ dst, int len, bool check) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
  const int nvec = aligned ? (len >> 3) : 0;
  bool bad = false;
  int v = threadIdx.x;
  for (; v + 3 * (int)blockDim.x < nvec; v += 4 * blockDim.x) {
    float f[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u) load8<W>(src + ((v + u * (int)blockDim.x) << 3), f[u], /*sys=*/true);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (check) {
#pragma unroll
        for (int k = 0; k < 8; ++k) bad |= !isfinite(f[u][k]);
      }
      store8<D>(dst + ((v + u * (int)blockDim.x) << 3), f[u]);
    }
  }
  for (; v < nvec; v += blockDim.x) {
    float f[8];
    load8<W>(src + (v << 3), f, /*sys=*/true);
    if (check) {
#pragma unroll
      for (int k = 0; k < 8; ++k) bad |= !isfinite(f[k]);
    }
    store8<D>(dst + (v << 3), f);
  }
  for (int i = (nvec << 3) + threadIdx.x; i < len; i += blockDim.x) {
    float x = to_f32<W>(*reinterpret_cast<const volatile W*>(src + i));
    if (check) bad |= !isfinite(x);
    dst[i] = from_f32<D>(x);
  }
  return bad;
}

template <typename W>
__device__ __forceinline__ void pack_block(const PtrPack& pk, const PlanArgs& a, W* arena_local) {
  for (int s = a.seg_begin[blockIdx.x]; s < a.seg_begin[blockIdx.x + 1]; ++s) {
    const Seg sg = a.segs[s];
    W* dst = arena_local + sg.arena_off;
    switch (pk.dtype[sg.tensor]) {
      case kF32:  pack_seg<W, float>(reinterpret_cast<const float*>(pk.ptr[sg.tensor]) + sg.src_off, dst, sg.len, a.scale); break;
      case kBF16: pack_seg<W, __nv_bfloat16>(reinterpret_cast<const __nv_bfloat16*>(pk.ptr[sg.tensor]) + sg.src_off, dst, sg.len, a.scale); break;
      default:    pack_seg<W, __half>(reinterpret_cast<const __half*>(pk.ptr[sg.tensor]) + sg.src_off, dst, sg.len, a.scale); break;
    }
  }
}

template <typename W>
__device__ __forceinline__ bool unpack_block(const PtrPack& pk, const PlanArgs& a, const W* arena_local, bool check) {
  bool bad = false;
  for (int s = a.seg_begin[blockIdx.x]; s < a.seg_begin[blockIdx.x + 1]; ++s) {
    const Seg sg = a.segs[s];
    const W* src = arena_local + sg.arena_off;
    switch (pk.dtype[sg.tensor]) {
      case kF32:  bad |= unpack_seg<W, float>(src, reinterpret_cast<float*>(pk.ptr[sg.tensor]) + sg.src_off, sg.len, check); break;
      case kBF16: bad |= unpack_seg<W, __nv_bfloat16>(src, reinterpret_cast<__nv_bfloat16*>(pk.ptr[sg.tensor]) + sg.src_off, sg.len, check); break;
      default:    bad |= unpack_seg<W, __half>(src, reinterpret_cast<__half*>(pk.ptr[sg.tensor]) + sg.src_off, sg.len, check); break;
    }
  }
  return bad;
}

// Sum the 16-byte unit at byte offset `off` over all ranks with plain peer loads (fp32 accumulation).
// The adds run in rank order 0..world-1 on EVERY rank, so the result is a fixed function of the inputs: the one-shot
// kernel's ranks (each reduces the whole range itself) hold the same bits and take the same non-finite decision, and
// the two-shot / reduce-to-caller results do not depend on which rank owns a slice or calls.
template <typename W>
__device__ __forceinline__ void p2p_reduce_unit(const CommCtx& c, int64_t off, float (&acc)[sizeof(W) == 4 ? 4 : 8]) {
  constexpr int N = sizeof(W) == 4 ? 4 : 8;
#pragma unroll
  for (int k = 0; k < N; ++k) acc[k] = 0.f;
  for (int p = 0; p < c.world; ++p) {
    V4 v = ld_sys(c.base[p] + off);
    if constexpr (sizeof(W) == 4) {
      acc[0] += __uint_as_float(v.x); acc[1] += __uint_as_float(v.y); acc[2] += __uint_as_float(v.z); acc[3] += __uint_as_float(v.w);
    } else {
      float2 t;
      t = Wire<W>::unpack2(v.x); acc[0] += t.x; acc[1] += t.y;
      t = Wire<W>::unpack2(v.y); acc[2] += t.x; acc[3] += t.y;
      t = Wire<W>::unpack2(v.z); acc[4] += t.x; acc[5] += t.y;
      t = Wire<W>::unpack2(v.w); acc[6] += t.x; acc[7] += t.y;
    }
  }
}
template <typename W>
__device__ __forceinline__ V4 to_unit(const float (&acc)[sizeof(W) == 4 ? 4 : 8]) {
  if constexpr (sizeof(W) == 4) {
    return V4{__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]), __float_as_uint(acc[3])};
  } else {
    return V4{Wire<W>::pack2(acc[0], acc[1]), Wire<W>::pack2(acc[2], acc[3]), Wire<W>::pack2(acc[4], acc[5]), Wire<W>::pack2(acc[6], acc[7])};
  }
}
template <typename W>
__device__ __forceinline__ V4 scale_unit(const V4& v, float s) {
  if constexpr (sizeof(W) == 4) {
    return V4{__float_as_uint(__uint_as_float(v.x) * s), __float_as_uint(__uint_as_float(v.y) * s),
              __float_as_uint(__uint_as_float(v.z) * s), __float_as_uint(__uint_as_float(v.w) * s)};
  } else {
    float2 a = Wire<W>::unpack2(v.x), b = Wire<W>::unpack2(v.y), c = Wire<W>::unpack2(v.z), d = Wire<W>::unpack2(v.w);
    return V4{Wire<W>::pack2(a.x * s, a.y * s), Wire<W>::pack2(b.x * s, b.y * s), Wire<W>::pack2(c.x * s, c.y * s),
              Wire<W>::pack2(d.x * s, d.y * s)};
  }
}
template <typename W>
__device__ __forceinline__ bool unit_nonfinite(const V4& v) {
  if constexpr (sizeof(W) == 4) {
    return !isfinite(__uint_as_float(v.x)) || !isfinite(__uint_as_float(v.y)) || !isfinite(__uint_as_float(v.z)) || !isfinite(__uint_as_float(v.w));
  } else {
    float2 a = Wire<W>::unpack2(v.x), b = Wire<W>::unpack2(v.y), c = Wire<W>::unpack2(v.z), d = Wire<W>::unpack2(v.w);
    return !isfinite(a.x) || !isfinite(a.y) || !isfinite(b.x) || !isfinite(b.y) || !isfinite(c.x) || !isfinite(c.y) || !isfinite(d.x) || !isfinite(d.y);
  }
}

// ================================================================= K1: fused bucket all-reduce (two-shot)
// phase 0  pack   : this rank's gradients -> local arena, cast to the wire dtype, pre-scaled by 1/world
// barrier         : peers' packs visible
// phase 1  reduce : rank r owns slice r of every CTA range: in-switch reduce (multimem.ld_reduce) or peer loads,
//                   result multicast (multimem.st) or stored to every peer  == reduce-scatter + all-gather
// barrier         : every slice of this CTA's range has landed in the local arena
// phase 2  unpack : (optional) local arena -> gradient tensors; otherwise the optimizer reads the arena directly
template <typename W, bool NVLS>
__global__ void __launch_bounds__(kThreads) fused_allreduce_kernel(const __grid_constant__ CommCtx c,
                                                                   const __grid_constant__ PtrPack pk,
                                                                   const __grid_constant__ PlanArgs a) {
  uint32_t seq = load_seq(c);
  W* local = reinterpret_cast<W*>(c.base[c.rank] + a.data_off_bytes);
  const bool prepacked = (a.flags & kPrepacked) != 0;      // gradients are bucket views: autograd wrote them into the arena
  const bool rescale = prepacked && a.scale != 1.0f;
  if (!prepacked) pack_block<W>(pk, a, local);
  if (c.world == 1 && !a.found_inf && !rescale) {
    // single rank: the "reduction" is the packed arena itself - no flags, no second pass over the data
    if (a.writeback) {
      __syncthreads();
      unpack_block<W>(pk, a, local, false);
    }
    return;
  }
  block_barrier(c, seq);

  constexpr int kUnitElems = 16 / sizeof(W);
  const int64_t slice_elems = a.block_elems / c.world;
  const int64_t slice_off = a.data_off_bytes + ((int64_t)blockIdx.x * a.block_elems + (int64_t)c.rank * slice_elems) * sizeof(W);
  const int units = (int)(slice_elems / kUnitElems);
  bool bad = false;
  if constexpr (NVLS) {
    char* mc = c.mc_base + slice_off;
    constexpr int U = 4;
    int u = threadIdx.x;
    for (; u + (U - 1) * kThreads < units; u += U * kThreads) {
      V4 v[U];
#pragma unroll
      for (int k = 0; k < U; ++k) v[k] = Multimem<W>::ld_reduce(mc + (int64_t)(u + k * kThreads) * 16);
#pragma unroll
      for (int k = 0; k < U; ++k) {
        if (rescale) v[k] = scale_unit<W>(v[k], a.scale);
        if (a.found_inf) bad |= unit_nonfinite<W>(v[k]);
        multimem_st(mc + (int64_t)(u + k * kThreads) * 16, v[k]);
      }
    }
    for (; u < units; u += kThreads) {
      V4 v = Multimem<W>::ld_reduce(mc + (int64_t)u * 16);
      if (rescale) v = scale_unit<W>(v, a.scale);
      if (a.found_inf) bad |= unit_nonfinite<W>(v);
      multimem_st(mc + (int64_t)u * 16, v);
    }
  } else {
    for (int u = threadIdx.x; u < units; u += kThreads) {
      float acc[sizeof(W) == 4 ? 4 : 8];
      const int64_t off = slice_off + (int64_t)u * 16;
      p2p_reduce_unit<W>(c, off, acc);
      if (rescale) {
#pragma unroll
        for (int k = 0; k < (sizeof(W) == 4 ? 4 : 8); ++k) acc[k] *= a.scale;
      }
      V4 v = to_unit<W>(acc);
      if (a.found_inf) bad |= unit_nonfinite<W>(v);
      for (int i = 0; i < c.world; ++i) st_sys(c.base[(c.rank + i) % c.world] + off, v);
    }
  }
  if (a.found_inf && __syncthreads_or(bad) && threadIdx.x < c.world) {
    // tell every rank (including myself) that this step's reduced gradients are non-finite
    const int64_t word_off = reinterpret_cast<char*>(a.found_inf) - c.base[c.rank];
    *reinterpret_cast<volatile uint32_t*>(c.base[threadIdx.x] + word_off) = 1u;
  }
  block_barrier(c, seq);
  if (a.writeback) unpack_block<W>(pk, a, local, false);
  store_seq(c, seq);
}

// ================================================================= K1b: one-shot all-reduce (small payloads)
// Every rank reduces the WHOLE CTA range itself: one network traversal and ONE barrier instead of two; W x the link
// traffic, so only for latency-bound sizes (the crossover is measured by tools/comm_bench.py).
//   pack   : gradients -> staging[call & 1]   (double buffered: a peer may still be reading the previous call's pack)
//   barrier: peers' packs visible
//   reduce : in-switch sum (multimem.ld_reduce) or peer loads of the whole CTA range -> the RESULT range of the local arena
//            (the bucket's slot of the gradient arena when an engine owns one: the flat optimizer reads it in place)
//   unpack : (optional) result range -> gradient tensors
template <typename W, bool NVLS>
__global__ void __launch_bounds__(kThreads) oneshot_allreduce_kernel(const __grid_constant__ CommCtx c,
                                                                     const __grid_constant__ PtrPack pk,
                                                                     const __grid_constant__ PlanArgs a) {
  uint32_t seq = load_seq(c);
  const uint32_t call = a.plan_calls[blockIdx.x];
  const int64_t half_bytes = (int64_t)gridDim.x * a.block_elems * sizeof(W);
  const int64_t stage_off = a.data_off_bytes + (call & 1) * half_bytes;
  const int64_t result_off = a.result_off_bytes >= 0 ? a.result_off_bytes : a.data_off_bytes + 2 * half_bytes;
  pack_block<W>(pk, a, reinterpret_cast<W*>(c.base[c.rank] + stage_off));
  block_barrier(c, seq);
  constexpr int kUnitElems = 16 / sizeof(W);
  const int64_t blk_bytes = (int64_t)blockIdx.x * a.block_elems * sizeof(W);
  const int units = (int)(a.block_elems / kUnitElems);
  bool bad = false;
  {
    // latency-bound by design (one traversal of the switch per unit): keep 8 requests in flight per thread
    constexpr int U = 8;
    const int64_t src0 = stage_off + blk_bytes, dst0 = result_off + blk_bytes;
    int u = threadIdx.x;
    for (; u + (U - 1) * kThreads < units; u += U * kThreads) {
      V4 v[U];
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const int64_t off = src0 + (int64_t)(u + k * kThreads) * 16;
        if constexpr (NVLS) {
          v[k] = Multimem<W>::ld_reduce(c.mc_base + off);
        } else {
          float acc[sizeof(W) == 4 ? 4 : 8];
          p2p_reduce_unit<W>(c, off, acc);
          v[k] = to_unit<W>(acc);
        }
      }
#pragma unroll
      for (int k = 0; k < U; ++k) {
        if (a.found_inf) bad |= unit_nonfinite<W>(v[k]);
        st_v4(c.base[c.rank] + dst0 + (int64_t)(u + k * kThreads) * 16, v[k]);
      }
    }
    for (; u < units; u += kThreads) {
      const int64_t off = src0 + (int64_t)u * 16;
      V4 v;
      if constexpr (NVLS) {
        v = Multimem<W>::ld_reduce(c.mc_base + off);
      } else {
        float acc[sizeof(W) == 4 ? 4 : 8];
        p2p_reduce_unit<W>(c, off, acc);
        v = to_unit<W>(acc);
      }
      if (a.found_inf) bad |= unit_nonfinite<W>(v);
      st_v4(c.base[c.rank] + dst0 + (int64_t)u * 16, v);
    }
  }
  if (a.found_inf && __syncthreads_or(bad) && threadIdx.x == 0) {
    // every rank reduced the same values in the same order (rank order on P2P; on NVLS the switch's sum, which
    // tests/mp_gpu_checks.py requires to be identical across ranks), so every rank takes the same decision: a local store
    // is enough
    *reinterpret_cast<volatile uint32_t*>(a.found_inf) = 1u;
  }
  __syncthreads();
  if (a.writeback) unpack_block<W>(pk, a, reinterpret_cast<const W*>(c.base[c.rank] + result_off), false);
  if (threadIdx.x == 0) a.plan_calls[blockIdx.x] = call + 1;
  store_seq(c, seq);
}

// Replicate `units` 16-byte units starting at arena byte offset `off0` from the local arena into every peer's
// (one multimem.st per unit through the switch, or W-1 peer stores): 4 loads in flight per thread.
template <bool NVLS>
__device__ __forceinline__ void push_range(const CommCtx& c, int64_t off0, int units) {
  constexpr int U = 4;
  int u = threadIdx.x;
  for (; u + (U - 1) * kThreads < units; u += U * kThreads) {
    V4 v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) v[k] = ld_sys(c.base[c.rank] + off0 + (int64_t)(u + k * kThreads) * 16);
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t off = off0 + (int64_t)(u + k * kThreads) * 16;
      if constexpr (NVLS) {
        multimem_st(c.mc_base + off, v[k]);
      } else {
        for (int i = 1; i < c.world; ++i) st_sys(c.base[(c.rank + i) % c.world] + off, v[k]);
      }
    }
  }
  for (; u < units; u += kThreads) {
    const int64_t off = off0 + (int64_t)u * 16;
    V4 v = ld_sys(c.base[c.rank] + off);
    if constexpr (NVLS) {
      multimem_st(c.mc_base + off, v);
    } else {
      for (int i = 1; i < c.world; ++i) st_sys(c.base[(c.rank + i) % c.world] + off, v);
    }
  }
}

// ================================================================= K2: fused multi-tensor broadcast
// root: tensors -> (multicast | every peer's) arena; barrier; non-root: arena -> tensors.
template <typename W, bool NVLS>
__global__ void __launch_bounds__(kThreads) fused_broadcast_kernel(const __grid_constant__ CommCtx c,
                                                                   const __grid_constant__ PtrPack pk,
                                                                   const __grid_constant__ PlanArgs a) {
  uint32_t seq = load_seq(c);
  const uint32_t call = a.plan_calls[blockIdx.x];
  const int64_t half_bytes = (int64_t)gridDim.x * a.block_elems * sizeof(W);
  const int64_t data_off = a.data_off_bytes + (call & 1) * half_bytes;
  W* local = reinterpret_cast<W*>(c.base[c.rank] + data_off);
  constexpr int kUnitElems = 16 / sizeof(W);
  if (c.rank == a.root) {
    pack_block<W>(pk, a, local);
    __syncthreads();
    // push my CTA range to everyone else
    const int64_t off0 = data_off + (int64_t)blockIdx.x * a.block_elems * sizeof(W);
    const int units = (int)(a.block_elems / kUnitElems);
    push_range<NVLS>(c, off0, units);
  }
  block_barrier(c, seq);
  if (c.rank != a.root) unpack_block<W>(pk, a, local, false);
  __syncthreads();
  if (threadIdx.x == 0) a.plan_calls[blockIdx.x] = call + 1;
  store_seq(c, seq);
}

// ================================================================= host-synchronised variants (single-process engine)
// nn.DataParallel runs all GPUs from one process, so ordering between devices is done with CUDA events on the host
// side and these kernels carry no flags.  (/root/reference/dataparallel.py:138: replicate = K2', backward
// reduce-add onto GPU0 = K5.)
//   kind 3  pack      : tensors -> local arena (cast + scale)
//   kind 4  reduce    : K5 - the calling device pulls the sum of EVERY device's arena range (in-switch reduce or
//                       peer loads), leaves it in its own arena and optionally unpacks it into its tensors
//   kind 5  push      : K2' - pack + multicast (or peer stores) of the range into every device's arena
//   kind 6  unpack    : local arena -> tensors
template <typename W>
__global__ void __launch_bounds__(kThreads) pack_only_kernel(const __grid_constant__ CommCtx c, const __grid_constant__ PtrPack pk,
                                                             const __grid_constant__ PlanArgs a) {
  pack_block<W>(pk, a, reinterpret_cast<W*>(c.base[c.rank] + a.data_off_bytes));
}
template <typename W>
__global__ void __launch_bounds__(kThreads) unpack_only_kernel(const __grid_constant__ CommCtx c, const __grid_constant__ PtrPack pk,
                                                               const __grid_constant__ PlanArgs a) {
  unpack_block<W>(pk, a, reinterpret_cast<const W*>(c.base[c.rank] + a.data_off_bytes), false);
}
template <typename W, bool NVLS>
__global__ void __launch_bounds__(kThreads) reduce_to_caller_kernel(const __grid_constant__ CommCtx c, const __grid_constant__ PtrPack pk,
                                                                    const __grid_constant__ PlanArgs a) {
  constexpr int kUnitElems = 16 / sizeof(W);
  const int64_t off0 = a.data_off_bytes + (int64_t)blockIdx.x * a.block_elems * sizeof(W);
  const int units = (int)(a.block_elems / kUnitElems);
  {
    constexpr int U = 8;       // the root pulls every unit through the switch: 8 in-switch reductions in flight per thread
    int u = threadIdx.x;
    for (; u + (U - 1) * kThreads < units; u += U * kThreads) {
      V4 v[U];
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const int64_t off = off0 + (int64_t)(u + k * kThreads) * 16;
        if constexpr (NVLS) {
          v[k] = Multimem<W>::ld_reduce(c.mc_base + off);
        } else {
          float acc[sizeof(W) == 4 ? 4 : 8];
          p2p_reduce_unit<W>(c, off, acc);
          v[k] = to_unit<W>(acc);
        }
      }
#pragma unroll
      for (int k = 0; k < U; ++k) st_v4(c.base[c.rank] + off0 + (int64_t)(u + k * kThreads) * 16, v[k]);
    }
    for (; u < units; u += kThreads) {
      const int64_t off = off0 + (int64_t)u * 16;
      V4 v;
      if constexpr (NVLS) {
        v = Multimem<W>::ld_reduce(c.mc_base + off);
      } else {
        float acc[sizeof(W) == 4 ? 4 : 8];
        p2p_reduce_unit<W>(c, off, acc);
        v = to_unit<W>(acc);
      }
      st_v4(c.base[c.rank] + off, v);
    }
  }
  if (a.writeback) {
    __syncthreads();
    unpack_block<W>(pk, a, reinterpret_cast<const W*>(c.base[c.rank] + a.data_off_bytes), false);
  }
}
template <typename W, bool NVLS>
__global__ void __launch_bounds__(kThreads) push_kernel(const __grid_constant__ CommCtx c, const __grid_constant__ PtrPack pk,
                                                        const __grid_constant__ PlanArgs a) {
  constexpr int kUnitElems = 16 / sizeof(W);
  W* local = reinterpret_cast<W*>(c.base[c.rank] + a.data_off_bytes);
  pack_block<W>(pk, a, local);
  __syncthreads();
  const int64_t off0 = a.data_off_bytes + (int64_t)blockIdx.x * a.block_elems * sizeof(W);
  const int units = (int)(a.block_elems / kUnitElems);
  push_range<NVLS>(c, off0, units);
}

// ================================================================= K3: barrier
__global__ void barrier_kernel(const __grid_constant__ CommCtx c) {
  uint32_t seq = load_seq(c);
  block_barrier(c, seq);
  store_seq(c, seq);
}

// ================================================================= K4: accuracy + metric all-reduce (LL protocol)
// Single CTA. Rows of `logits` are scanned by warps: a sample is top-k correct iff fewer than k logits are
// strictly greater than the target logit.  The three local means are then pushed into every peer's inbox as
// 8-byte {value, sequence} words (atomic on NVLink), and each rank sums its own inbox - no barrier.
template <typename T>
__device__ __forceinline__ float ldf(const T* p) { return to_f32<T>(*p); }

template <typename T>
__global__ void __launch_bounds__(1024) metrics_kernel(const __grid_constant__ CommCtx c, const T* __restrict__ logits,
                                                       const int64_t* __restrict__ target, const float* __restrict__ loss,
                                                       int batch, int classes, int64_t row_stride, uint32_t* ll_seq,
                                                       float* __restrict__ out /*[4]: loss, acc1, acc5, seq*/) {
  __shared__ int s_top1, s_top5;
  if (threadIdx.x == 0) { s_top1 = 0; s_top5 = 0; }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  int top1 = 0, top5 = 0;
  for (int r = warp; r < batch; r += nwarps) {
    const T* row = logits + (int64_t)r * row_stride;
    const int64_t t = target[r];
    const bool valid = t >= 0 && t < classes;      // a target outside [0, classes) is never correct
    const float tv = valid ? ldf(row + t) : INFINITY;
    int cnt = 0;
    for (int j = lane; j < classes; j += 32) cnt += (ldf(row + j) > tv) ? 1 : 0;
#pragma unroll
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    top1 += valid && cnt < 1;
    top5 += valid && cnt < 5;
  }
  if (lane == 0) { atomicAdd(&s_top1, top1); atomicAdd(&s_top5, top5); }
  __syncthreads();
  if (threadIdx.x >= 32) return;
  // ---- warp 0: exchange
  float vals[3];
  vals[0] = loss ? *loss : 0.f;
  vals[1] = 100.f * (float)s_top1 / (float)batch;
  vals[2] = 100.f * (float)s_top5 / (float)batch;
  uint32_t seq = 0;
  if (c.world > 1) {
    seq = *ll_seq + 1;
    const int par = seq & 1;
    // lane l < world*3 : send value (l % 3) to peer (l / 3)
    for (int l = lane; l < c.world * 3; l += 32) {
      const int peer = l / 3, slot = l % 3;
      uint2 w{__float_as_uint(vals[slot]), seq};
      uint2* dst = &pad_of(c, peer)->inbox[par][c.rank][slot];
      asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1,%2};" ::"l"(dst), "r"(w.x), "r"(w.y) : "memory");
    }
    float sum[3] = {0.f, 0.f, 0.f};
    const uint64_t t0 = globaltimer_ns();
    for (int l = lane; l < c.world * 3; l += 32) {
      const int src = l / 3, slot = l % 3;
      const uint2* p = &pad_of(c, c.rank)->inbox[par][src][slot];
      uint2 w;
      while (true) {
        asm volatile("ld.relaxed.sys.global.v2.u32 {%0,%1}, [%2];" : "=r"(w.x), "=r"(w.y) : "l"(p) : "memory");
        if (w.y == seq) break;
        if (c.timeout_ms && globaltimer_ns() - t0 > (uint64_t)c.timeout_ms * 1000000ull) {
          if (c.status) { *reinterpret_cast<volatile uint32_t*>(c.status) = 0xDEAD1000u | (uint32_t)c.rank; __threadfence_system(); }
          __trap();
        }
      }
      sum[slot] += __uint_as_float(w.x);
    }
#pragma unroll
    for (int s = 0; s < 3; ++s) {
#pragma unroll
      for (int o = 16; o; o >>= 1) sum[s] += __shfl_xor_sync(0xffffffffu, sum[s], o);
      vals[s] = sum[s] / (float)c.world;
    }
  }
  if (lane == 0) {
    out[0] = vals[0]; out[1] = vals[1]; out[2] = vals[2]; out[3] = (float)seq;
    if (c.world > 1) *ll_seq = seq;
  }
}

// Plain 3-float (or n<=8 float) LL all-reduce mean, for reduce_mean()/hvd.allreduce on scalars.
__global__ void ll_allreduce_kernel(const __grid_constant__ CommCtx c, const float* __restrict__ in, float* __restrict__ out,
                                    int n, float scale, uint32_t* ll_seq) {
  const int lane = threadIdx.x;
  const uint32_t seq = *ll_seq + 1;
  const int par = seq & 1;
  for (int l = lane; l < c.world * n; l += 32) {
    const int peer = l / n, slot = l % n;
    uint2 w{__float_as_uint(in[slot]), seq};
    uint2* dst = &pad_of(c, peer)->inbox[par][c.rank][slot];
    asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1,%2};" ::"l"(dst), "r"(w.x), "r"(w.y) : "memory");
  }
  const uint64_t t0 = globaltimer_ns();
  // lane s < n sums slot s over the sources in rank order (deterministic)
  if (lane < n) {
    float sum = 0.f;
    for (int src = 0; src < c.world; ++src) {
      const uint2* p = &pad_of(c, c.rank)->inbox[par][src][lane];
      uint2 w;
      while (true) {
        asm volatile("ld.relaxed.sys.global.v2.u32 {%0,%1}, [%2];" : "=r"(w.x), "=r"(w.y) : "l"(p) : "memory");
        if (w.y == seq) break;
        if (c.timeout_ms && globaltimer_ns() - t0 > (uint64_t)c.timeout_ms * 1000000ull) {
          if (c.status) { *reinterpret_cast<volatile uint32_t*>(c.status) = 0xDEAD2000u | (uint32_t)c.rank; __threadfence_system(); }
          __trap();
        }
      }
      sum += __uint_as_float(w.x);
    }
    out[lane] = sum * scale;
  }
  __syncwarp();
  if (lane == 0) *ll_seq = seq;
}

// ================================================================= rank-local fp32 gradient accumulation (no peers)
// Driven by a bucket's plan (segment table + pointer pack), one launch per bucket and pass, nothing crosses GPUs.  `acc`
// is the bucket's slice of an fp32 buffer with the gradient arena's element layout (element acc[seg.arena_off + i]).
//   grad_accumulate : acc += float(g)                                   (every pass of a no_sync group but the last)
//   grad_fold       : g = round_to_dtype(acc + float(g)); acc = 0       (the last pass, right before K1)
// Each element is one IEEE fp32 add in pass order (add.rn.f32: no contraction, denormals kept), so the sum is the one
// torch's acc.add_(g.float()) / (acc + g.float()).to(g.dtype) give.  Only the segments' elements are touched: the padding
// between tensors is never written.  blockIdx.y splits every plan CTA's segments over gridDim.y CTAs.
__device__ __forceinline__ float add_rn(float a, float b) {
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

template <bool kFold, typename S>
__device__ __forceinline__ void accum_seg(S* __restrict__ g, float* __restrict__ acc, int len) {
  const int stride = blockDim.x * gridDim.y;
  const int t0 = threadIdx.x + blockIdx.y * blockDim.x;
  // acc is 32-byte aligned at every segment start (arena offsets are multiples of 8 elements); the gradient may not be
  const bool aligned = ((reinterpret_cast<uintptr_t>(g) & 15) == 0);
  const int nvec = aligned ? (len >> 3) : 0;
  int v = t0;
  for (; v + stride < nvec; v += 2 * stride) {       // two independent 8-element units in flight per thread
    float f[2][8], a[2][8];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      load8<S>(g + ((v + u * stride) << 3), f[u]);
      load8<float>(acc + ((v + u * stride) << 3), a[u]);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
#pragma unroll
      for (int k = 0; k < 8; ++k) a[u][k] = add_rn(a[u][k], f[u][k]);
      if constexpr (kFold) {
        store8<S>(g + ((v + u * stride) << 3), a[u]);
        const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        store8<float>(acc + ((v + u * stride) << 3), z);
      } else {
        store8<float>(acc + ((v + u * stride) << 3), a[u]);
      }
    }
  }
  for (; v < nvec; v += stride) {
    float f[8], a[8];
    load8<S>(g + (v << 3), f);
    load8<float>(acc + (v << 3), a);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = add_rn(a[k], f[k]);
    if constexpr (kFold) {
      store8<S>(g + (v << 3), a);
      const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      store8<float>(acc + (v << 3), z);
    } else {
      store8<float>(acc + (v << 3), a);
    }
  }
  for (int i = (nvec << 3) + t0; i < len; i += stride) {
    const float s = add_rn(acc[i], to_f32<S>(g[i]));
    if constexpr (kFold) {
      g[i] = from_f32<S>(s);
      acc[i] = 0.f;
    } else {
      acc[i] = s;
    }
  }
}

template <bool kFold>
__device__ __forceinline__ void accum_block(const PtrPack& pk, const int32_t* __restrict__ seg_begin, const Seg* __restrict__ segs,
                                            float* __restrict__ acc) {
  for (int s = seg_begin[blockIdx.x]; s < seg_begin[blockIdx.x + 1]; ++s) {
    const Seg sg = segs[s];
    float* a = acc + sg.arena_off;
    switch (pk.dtype[sg.tensor]) {
      case kF32:  accum_seg<kFold, float>(reinterpret_cast<float*>(pk.ptr[sg.tensor]) + sg.src_off, a, sg.len); break;
      case kBF16: accum_seg<kFold, __nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(pk.ptr[sg.tensor]) + sg.src_off, a, sg.len); break;
      default:    accum_seg<kFold, __half>(reinterpret_cast<__half*>(pk.ptr[sg.tensor]) + sg.src_off, a, sg.len); break;
    }
  }
}

__global__ void __launch_bounds__(kThreads) grad_accumulate_kernel(const __grid_constant__ PtrPack pk, const int32_t* __restrict__ seg_begin,
                                                                   const Seg* __restrict__ segs, float* __restrict__ acc) {
  accum_block<false>(pk, seg_begin, segs, acc);
}

__global__ void __launch_bounds__(kThreads) grad_fold_kernel(const __grid_constant__ PtrPack pk, const int32_t* __restrict__ seg_begin,
                                                             const Seg* __restrict__ segs, float* __restrict__ acc) {
  accum_block<true>(pk, seg_begin, segs, acc);
}

// ================================================================= host launchers
static void fill_ptrs(PtrPack& pk, const std::vector<at::Tensor>& ts) {
  TORCH_CHECK((int)ts.size() <= kMaxPtrs, "too many tensors in one plan launch: ", ts.size(), " > ", kMaxPtrs);
  for (size_t i = 0; i < ts.size(); ++i) {
    const auto& t = ts[i];
    TORCH_CHECK(t.is_cuda(), "collective tensors must be CUDA tensors");
    TORCH_CHECK(t.is_non_overlapping_and_dense(), "collective tensors must be dense");
    pk.ptr[i] = t.data_ptr();
    switch (t.scalar_type()) {
      case at::kFloat: pk.dtype[i] = kF32; break;
      case at::kBFloat16: pk.dtype[i] = kBF16; break;
      case at::kHalf: pk.dtype[i] = kF16; break;
      default: TORCH_CHECK(false, "unsupported dtype in fused collective: ", t.scalar_type());
    }
  }
}

// The pointer pack of a tensor list as an opaque CPU byte tensor: build it once for lists whose storage never moves
// (parameters of persistent replicas, static gradient buffers of captured graphs) and pass [pack] instead of the list.
at::Tensor pack_pointers(const std::vector<at::Tensor>& tensors) {
  at::Tensor out = at::zeros({(int64_t)sizeof(PtrPack)}, at::TensorOptions().dtype(at::kByte));
  PtrPack pk;
  memset(&pk, 0, sizeof(pk));
  fill_ptrs(pk, tensors);
  memcpy(out.data_ptr(), &pk, sizeof(PtrPack));
  return out;
}

template <typename W, bool NVLS>
static void launch_kind(int kind, int grid, cudaStream_t st, const CommCtx& c, const PtrPack& pk, const PlanArgs& a) {
  switch (kind) {
    case 0: fused_allreduce_kernel<W, NVLS><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    case 1: oneshot_allreduce_kernel<W, NVLS><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    case 2: fused_broadcast_kernel<W, NVLS><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    case 3: pack_only_kernel<W><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    case 4: reduce_to_caller_kernel<W, NVLS><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    case 5: push_kernel<W, NVLS><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    case 6: unpack_only_kernel<W><<<grid, kThreads, 0, st>>>(c, pk, a); break;
    default: TORCH_CHECK(false, "unknown plan kind ", kind);
  }
}

// kind: 0 two-shot all-reduce, 1 one-shot all-reduce, 2 broadcast, 3 pack, 4 reduce-to-caller, 5 push, 6 unpack
void launch_plan(const CommCtx& ctx, int kind, int wire_dtype, bool nvls, int grid, const std::vector<at::Tensor>& tensors,
                 int64_t seg_begin_ptr, int64_t segs_ptr, int64_t data_off_bytes, int64_t block_elems, int64_t plan_calls_ptr,
                 int64_t found_inf_ptr, double scale, bool writeback, int root, int flags, int64_t result_off_bytes) {
  // kinds 0-2 synchronise through the per-CTA flag table (kMaxBlocks rows); the host-synchronised kinds 3-6 carry no flags
  TORCH_CHECK(grid >= 1 && (grid <= kMaxBlocks || kind >= 3), "grid out of range");
  TORCH_CHECK(!nvls || ctx.mc_base != nullptr, "NVLS variant requested but no multicast mapping");
  PtrPack pk;
  if (tensors.size() == 1 && tensors[0].is_cpu() && tensors[0].scalar_type() == at::kByte && tensors[0].numel() == (int64_t)sizeof(PtrPack)) {
    // pre-built pointer pack (pack_pointers()): persistent tensor lists skip the per-launch list conversion and checks
    memcpy(&pk, tensors[0].data_ptr(), sizeof(PtrPack));
  } else {
    fill_ptrs(pk, tensors);
  }
  PlanArgs a;
  a.seg_begin = reinterpret_cast<const int32_t*>(seg_begin_ptr);
  a.segs = reinterpret_cast<const Seg*>(segs_ptr);
  a.data_off_bytes = data_off_bytes;
  a.block_elems = block_elems;
  a.plan_calls = reinterpret_cast<uint32_t*>(plan_calls_ptr);
  a.found_inf = reinterpret_cast<uint32_t*>(found_inf_ptr);
  a.scale = (float)scale;
  a.writeback = writeback ? 1 : 0;
  a.root = root;
  a.flags = flags;
  a.result_off_bytes = result_off_bytes;
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  switch (wire_dtype) {
    case kBF16: nvls ? launch_kind<__nv_bfloat16, true>(kind, grid, st, ctx, pk, a) : launch_kind<__nv_bfloat16, false>(kind, grid, st, ctx, pk, a); break;
    case kF16:  nvls ? launch_kind<__half, true>(kind, grid, st, ctx, pk, a) : launch_kind<__half, false>(kind, grid, st, ctx, pk, a); break;
    default:    nvls ? launch_kind<float, true>(kind, grid, st, ctx, pk, a) : launch_kind<float, false>(kind, grid, st, ctx, pk, a); break;
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void grad_accum(const std::vector<at::Tensor>& grads, const at::Tensor& seg_begin, const at::Tensor& segs, int64_t grid, int64_t split,
                at::Tensor acc, int64_t acc_off, int64_t region_elems, bool fold) {
  TORCH_CHECK(grid >= 1 && split >= 1 && split <= 65535, "grad_accum: grid out of range");
  TORCH_CHECK(seg_begin.is_cuda() && seg_begin.scalar_type() == at::kInt && seg_begin.numel() == grid + 1, "grad_accum: seg_begin must be int32[grid + 1]");
  TORCH_CHECK(segs.is_cuda() && segs.scalar_type() == at::kByte && segs.numel() % (int64_t)sizeof(Seg) == 0, "grad_accum: segs must be a byte segment table");
  TORCH_CHECK(acc.is_cuda() && acc.scalar_type() == at::kFloat && acc.is_contiguous() && acc.dim() == 1, "grad_accum: acc must be a flat fp32 CUDA tensor");
  TORCH_CHECK(acc_off >= 0 && region_elems >= 0 && acc_off + region_elems <= acc.numel(), "grad_accum: bucket range outside the accumulator");
  float* a = acc.data_ptr<float>() + acc_off;
  TORCH_CHECK((reinterpret_cast<uintptr_t>(a) & 31) == 0, "grad_accum: the bucket's accumulator slice must be 32-byte aligned");
  PtrPack pk;
  fill_ptrs(pk, grads);
  for (const auto& g : grads) TORCH_CHECK(g.device() == acc.device(), "grad_accum: gradients and accumulator on different devices");
  const c10::cuda::CUDAGuard guard(acc.device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const dim3 g((unsigned)grid, (unsigned)split);
  const auto* sb = seg_begin.data_ptr<int32_t>();
  const auto* sg = reinterpret_cast<const Seg*>(segs.data_ptr());
  if (fold) grad_fold_kernel<<<g, kThreads, 0, st>>>(pk, sb, sg, a);
  else grad_accumulate_kernel<<<g, kThreads, 0, st>>>(pk, sb, sg, a);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void launch_barrier(const CommCtx& ctx) {
  barrier_kernel<<<1, 32, 0, at::cuda::getCurrentCUDAStream()>>>(ctx);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void launch_metrics(const CommCtx& ctx, const at::Tensor& logits, const at::Tensor& target, const c10::optional<at::Tensor>& loss,
                    int64_t ll_seq_ptr, at::Tensor out) {
  TORCH_CHECK(logits.dim() == 2 && logits.stride(1) == 1, "logits must be [B, C] with unit inner stride");
  TORCH_CHECK(target.scalar_type() == at::kLong && target.is_contiguous(), "target must be contiguous int64");
  TORCH_CHECK(out.scalar_type() == at::kFloat && out.numel() >= 4 && out.is_contiguous(), "out must be float[4]");
  const float* lp = nullptr;
  if (loss.has_value()) {
    TORCH_CHECK(loss->scalar_type() == at::kFloat && loss->numel() == 1, "loss must be a float32 scalar");
    lp = loss->data_ptr<float>();
  }
  const int B = (int)logits.size(0), C = (int)logits.size(1);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  uint32_t* seq = reinterpret_cast<uint32_t*>(ll_seq_ptr);
  switch (logits.scalar_type()) {
    case at::kFloat:
      metrics_kernel<float><<<1, 1024, 0, st>>>(ctx, logits.data_ptr<float>(), target.data_ptr<int64_t>(), lp, B, C, logits.stride(0), seq, out.data_ptr<float>());
      break;
    case at::kBFloat16:
      metrics_kernel<__nv_bfloat16><<<1, 1024, 0, st>>>(ctx, reinterpret_cast<const __nv_bfloat16*>(logits.data_ptr()), target.data_ptr<int64_t>(), lp, B, C, logits.stride(0), seq, out.data_ptr<float>());
      break;
    case at::kHalf:
      metrics_kernel<__half><<<1, 1024, 0, st>>>(ctx, reinterpret_cast<const __half*>(logits.data_ptr()), target.data_ptr<int64_t>(), lp, B, C, logits.stride(0), seq, out.data_ptr<float>());
      break;
    default: TORCH_CHECK(false, "unsupported logits dtype");
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void launch_ll_allreduce(const CommCtx& ctx, const at::Tensor& in, at::Tensor out, double scale, int64_t ll_seq_ptr) {
  TORCH_CHECK(in.scalar_type() == at::kFloat && out.scalar_type() == at::kFloat && in.is_contiguous() && out.is_contiguous());
  TORCH_CHECK(in.numel() <= 8 && out.numel() >= in.numel(), "LL all-reduce handles at most 8 floats");
  ll_allreduce_kernel<<<1, 32, 0, at::cuda::getCurrentCUDAStream()>>>(ctx, in.data_ptr<float>(), out.data_ptr<float>(), (int)in.numel(),
                                                                     (float)scale, reinterpret_cast<uint32_t*>(ll_seq_ptr));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace ptd
