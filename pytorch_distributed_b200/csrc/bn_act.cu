// Fused NHWC BatchNorm (+ residual add) (+ ReLU), forward and backward, for sm_90a.
//
// The reference reaches cuDNN BN + ATen add + ATen ReLU through torchvision's ResNet
// (reference distributed.py:136-139,250).  A bf16 ResNet-50 step is bound by exactly those memory passes, so they
// are fused here:
//   forward : stats pass (1 read)  + apply pass  (x [+res] -> y, 1-bit ReLU mask)             eager: 3-5 R, 2-3 W
//   backward: reduce pass (dy,x,mask) + apply pass (dy,x,mask -> dx [,dres])                   eager: 6 R, 2-3 W
// The ReLU decision is kept as ONE BIT per element (a byte per thread-vector of 8 channels), so the backward never
// re-reads the 16-bit output tensor: 4.125 B/element per backward pass instead of 6.
// Layout: activations are channels_last, i.e. a row-major [M = N*H*W, C] matrix.  A thread owns 8 consecutive
// channels (one 16-byte vector for 16-bit dtypes) and walks down the rows, so every warp access is a fully
// coalesced 128..512-byte line and the per-channel reductions stay in registers until the end of the CTA.
// CTA-level combine (cta_combine): warp shuffles (lanes sharing a channel group) -> one shared-memory row per warp/row-group
// (plain stores, no shared atomics) -> one row of partial sums per CTA; finish_sums() adds the rows in a fixed order.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <map>

#include "bn_combine.cuh"
#include "common.cuh"
#include "host.h"

namespace ptd {

constexpr int kBnThreads = 256;
constexpr int kBnWarps = kBnThreads / 32;

struct RowMap {
  int cgs;     // channel groups (C / 8)
  int tpr;     // threads per row (power of two <= 256, or cgs when cgs < 256 and not a power of two)
  int rpp;     // rows per pass of one CTA
  int rlocal;  // this thread's row inside a pass
  int cg0;     // this thread's first channel group
  bool active;
  bool pow2;
};
__device__ __forceinline__ RowMap row_map(int C) {
  RowMap m;
  m.cgs = C >> 3;
  m.tpr = min(m.cgs, (int)blockDim.x);
  m.rpp = blockDim.x / m.tpr;
  m.rlocal = threadIdx.x / m.tpr;
  m.cg0 = threadIdx.x % m.tpr;
  m.active = m.rlocal < m.rpp;
  m.pow2 = (m.tpr & (m.tpr - 1)) == 0;
  return m;
}

// Combine the per-thread partial sums (a[8], b[8] for channel group `cg`) of a CTA into this CTA's row of the partials,
// part[blockIdx.x][0:C] / [C:2C]; combine_partials() then adds the rows in a fixed order.
// Caller loops over channel-group chunks; `sm` holds [slots][2 * tpr * 8] floats.
__device__ __forceinline__ void cta_combine(const RowMap& m, int cg_base, float (&a)[8], float (&b)[8], float* sm, float* part, int C) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int width = m.tpr * 8;        // channels covered per pass
  int slots, slot;
  bool writer = m.active;
  if (m.pow2 && m.tpr < 32) {         // several rows share a warp: fold them with shuffles first
    for (int o = m.tpr; o < 32; o <<= 1) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
        b[k] += __shfl_xor_sync(0xffffffffu, b[k], o);
      }
    }
    slots = kBnWarps;
    slot = warp;
    writer = lane < m.tpr;
  } else {
    slots = m.rpp;
    slot = m.rlocal;
  }
  __syncthreads();                    // previous chunk's readers are done with sm
  if (writer) {
    float* row = sm + (size_t)slot * 2 * width + m.cg0 * 8;
#pragma unroll
    for (int k = 0; k < 8; ++k) { row[k] = a[k]; row[width + k] = b[k]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * width; i += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < slots; ++r) s += sm[(size_t)r * 2 * width + i];
    const int half = i >= width, c = cg_base * 8 + (i - half * width);
    if (c < C) part[(size_t)blockIdx.x * 2 * C + half * C + c] = s;
  }
}

// gsum[i] += sum over b of part[b * n + i], always in the same order (b ascending within each of 32 slices, then the 32
// slice sums in order).  Float atomics across CTAs would make every BatchNorm statistic - and everything trained from
// it - depend on CTA scheduling; this way a step computes the same bits on every run.
__global__ void __launch_bounds__(1024) combine_partials_kernel(const float* __restrict__ part, int nblocks, int n,
                                                                float* __restrict__ gsum) {
  __shared__ float sm[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + tx;
  sm[ty][tx] = combine_slice(part, nblocks, n, i, ty);
  __syncthreads();
  if (ty == 0 && i < n) gsum[i] += combine_fold(sm, tx);
}

void combine_partials(const float* part, int nblocks, int n, float* gsum, cudaStream_t st) {
  combine_partials_kernel<<<(n + 31) / 32, 1024, 0, st>>>(part, nblocks, n, gsum);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// per-CTA partial sums [grid][2C] of one reduction pass
static at::Tensor partials(const at::Tensor& x, int grid, int C) {
  return at::empty({grid, 2 * C}, x.options().dtype(at::kFloat).memory_format(at::MemoryFormat::Contiguous));
}

// ------------------------------------------------------------------ forward: statistics
template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_stats_kernel(const T* __restrict__ x, float* __restrict__ part, int64_t M, int C,
                                                              int rows_per_block) {
  extern __shared__ float sm[];
  const RowMap m = row_map(C);
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block, r1 = min(M, r0 + (int64_t)rows_per_block);
  for (int cgb = 0; cgb < m.cgs; cgb += m.tpr) {
    const int cg = cgb + m.cg0;
    float s[8], q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] = 0.f; q[k] = 0.f; }
    if (m.active && cg < m.cgs) {
      const T* p = x + cg * 8;
      int64_t r = r0 + m.rlocal;
      for (; r + 7 * (int64_t)m.rpp < r1; r += 8 * (int64_t)m.rpp) {
        float f[8][8];
#pragma unroll
        for (int u = 0; u < 8; ++u) load8<T>(p + (r + (int64_t)u * m.rpp) * C, f[u]);
#pragma unroll
        for (int u = 0; u < 8; ++u)
#pragma unroll
          for (int k = 0; k < 8; ++k) { s[k] += f[u][k]; q[k] += f[u][k] * f[u][k]; }
      }
      for (; r < r1; r += m.rpp) {
        float f[8];
        load8<T>(p + r * C, f);
#pragma unroll
        for (int k = 0; k < 8; ++k) { s[k] += f[k]; q[k] += f[k] * f[k]; }
      }
    }
    cta_combine(m, cgb, s, q, sm, part, C);
  }
}

// Rows the statistics in gsum cover: this rank's M, or, synchronised (gsum = the global sums of a sync_bn_exchange work
// slice), the global count stored right after them.
template <bool SYNC>
__device__ __forceinline__ int64_t stat_rows(const float* gsum, int C, int64_t M) {
  if constexpr (SYNC) return *reinterpret_cast<const int64_t*>(gsum + 2 * C);
  else return M;
}

// ------------------------------------------------------------------ forward: normalise (+res) (+relu)
#define BN_APPLY_PARAMS                                                                                                    \
  const T *__restrict__ x, const T *__restrict__ res, T *__restrict__ y, uint8_t *__restrict__ mask,                      \
      const float *__restrict__ gsum, const void *__restrict__ w, const void *__restrict__ b, int wdt,                    \
      float *__restrict__ running_mean, float *__restrict__ running_var, int64_t *__restrict__ num_batches_tracked,       \
      float *__restrict__ saved, int64_t M, int C, float eps, float momentum, int training
#define BN_APPLY_ARGS x, res, y, mask, gsum, w, b, wdt, running_mean, running_var, num_batches_tracked, saved, M, C, eps, momentum, training
template <typename T, bool RELU, bool RES, bool SYNC>
__device__ __forceinline__ void bn_apply_body(BN_APPLY_PARAMS) {
  const RowMap m = row_map(C);
  const int64_t N = stat_rows<SYNC>(gsum, C, M);
  const float inv_m = 1.f / (float)N;
  if (training && num_batches_tracked && blockIdx.x == 0 && threadIdx.x == 0) *num_batches_tracked += 1;
  if (!m.active) return;
  for (int cg = m.cg0; cg < m.cgs; cg += m.tpr) {
    float sc[8], sh[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = cg * 8 + k;
      float mean, var;
      if (training) {
        mean = gsum[c] * inv_m;
        var = fmaxf(gsum[C + c] * inv_m - mean * mean, 0.f);
      } else {
        mean = running_mean[c];
        var = running_var[c];
      }
      const float invstd = rsqrtf(var + eps);
      sc[k] = ld_w(w, wdt, c) * invstd;
      sh[k] = ld_w(b, wdt, c) - mean * sc[k];
      if (training && blockIdx.x == 0 && m.rlocal == 0) {
        saved[c] = mean;
        saved[C + c] = invstd;
        if (running_mean) {
          const float unbiased = N > 1 ? var * ((float)N / (float)(N - 1)) : var;
          running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
          running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
        }
      }
    }
    const int64_t stride = (int64_t)gridDim.x * m.rpp;
    const int64_t coff = cg * 8;
    int64_t r = (int64_t)blockIdx.x * m.rpp + m.rlocal;
    for (; r + 3 * stride < M; r += 4 * stride) {
      float f[4][8], g[4][8];
#pragma unroll
      for (int u = 0; u < 4; ++u) load8<T>(x + (r + u * stride) * C + coff, f[u]);
      if constexpr (RES) {
#pragma unroll
        for (int u = 0; u < 4; ++u) load8<T>(res + (r + u * stride) * C + coff, g[u]);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        unsigned bits = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float v = f[u][k] * sc[k] + sh[k];
          if constexpr (RES) v += g[u][k];
          if constexpr (RELU) { bits |= (v > 0.f ? 1u : 0u) << k; v = fmaxf(v, 0.f); }
          f[u][k] = v;
        }
        store8<T>(y + (r + u * stride) * C + coff, f[u]);
        if constexpr (RELU) { if (mask) mask[(r + u * stride) * m.cgs + cg] = (uint8_t)bits; }
      }
    }
    for (; r < M; r += stride) {
      float f[8], g[8];
      load8<T>(x + r * C + coff, f);
      if constexpr (RES) load8<T>(res + r * C + coff, g);
      unsigned bits = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float v = f[k] * sc[k] + sh[k];
        if constexpr (RES) v += g[k];
        if constexpr (RELU) { bits |= (v > 0.f ? 1u : 0u) << k; v = fmaxf(v, 0.f); }
        f[k] = v;
      }
      store8<T>(y + r * C + coff, f);
      if constexpr (RELU) { if (mask) mask[r * m.cgs + cg] = (uint8_t)bits; }
    }
  }
}
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kBnThreads) bn_apply_kernel(BN_APPLY_PARAMS) { bn_apply_body<T, RELU, RES, false>(BN_APPLY_ARGS); }
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kBnThreads) bn_apply_sync_kernel(BN_APPLY_PARAMS) { bn_apply_body<T, RELU, RES, true>(BN_APPLY_ARGS); }
#undef BN_APPLY_PARAMS
#undef BN_APPLY_ARGS

// ------------------------------------------------------------------ backward: reductions
// gsum[0:C] = sum dz ; gsum[C:2C] = sum dz * xhat   with dz = dy * relu_mask
template <typename T, bool RELU>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_reduce_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ mask,
                                                                   const T* __restrict__ x, const float* __restrict__ saved,
                                                                   float* __restrict__ part, int64_t M, int C, int rows_per_block) {
  extern __shared__ float sm[];
  const RowMap m = row_map(C);
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block, r1 = min(M, r0 + (int64_t)rows_per_block);
  for (int cgb = 0; cgb < m.cgs; cgb += m.tpr) {
    const int cg = cgb + m.cg0;
    float s[8], q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] = 0.f; q[k] = 0.f; }
    if (m.active && cg < m.cgs) {
      float mean[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) mean[k] = saved[cg * 8 + k];
      const int64_t coff = cg * 8;
      int64_t r = r0 + m.rlocal;
      for (; r + 3 * (int64_t)m.rpp < r1; r += 4 * (int64_t)m.rpp) {
        float d[4][8], v[4][8];
        unsigned bits[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int64_t row = r + (int64_t)u * m.rpp;
          load8<T>(dy + row * C + coff, d[u]);
          load8<T>(x + row * C + coff, v[u]);
          if constexpr (RELU) bits[u] = mask[row * m.cgs + cg];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            float dz = d[u][k];
            if constexpr (RELU) dz = (bits[u] >> k) & 1u ? dz : 0.f;
            s[k] += dz;
            q[k] += dz * (v[u][k] - mean[k]);
          }
      }
      for (; r < r1; r += m.rpp) {
        float d[8], v[8];
        load8<T>(dy + r * C + coff, d);
        load8<T>(x + r * C + coff, v);
        unsigned bits = 0;
        if constexpr (RELU) bits = mask[r * m.cgs + cg];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float dz = d[k];
          if constexpr (RELU) dz = (bits >> k) & 1u ? dz : 0.f;
          s[k] += dz;
          q[k] += dz * (v[k] - mean[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) q[k] *= saved[C + cg * 8 + k];   // x invstd once per CTA, not per element
    }
    cta_combine(m, cgb, s, q, sm, part, C);
  }
}

// ------------------------------------------------------------------ backward: apply
// dx = gamma*invstd * (dz - mean(dz) - xhat * mean(dz*xhat)) ; dres = dz ; dgamma = sum dz*xhat ; dbeta = sum dz
// Synchronised: the means are over the global batch (global sums / global count), dgamma and dbeta stay this rank's sums
// (gsum - 2C in the sync_bn_exchange work slice), so that averaging the gradients over the ranks gives what
// torch.nn.SyncBatchNorm under DDP gives.
#define BN_BWD_APPLY_PARAMS                                                                                                \
  const T *__restrict__ dy, const uint8_t *__restrict__ mask, const T *__restrict__ x, const float *__restrict__ saved,    \
      const float *__restrict__ gsum, const void *__restrict__ w, int wdt, T *__restrict__ dx, T *__restrict__ dres,      \
      void *__restrict__ dw, void *__restrict__ db, int64_t M, int C
#define BN_BWD_APPLY_ARGS dy, mask, x, saved, gsum, w, wdt, dx, dres, dw, db, M, C
template <typename T, bool RELU, bool RES, bool SYNC>
__device__ __forceinline__ void bn_bwd_apply_body(BN_BWD_APPLY_PARAMS) {
  const RowMap m = row_map(C);
  if (!m.active) return;
  const float inv_m = 1.f / (float)stat_rows<SYNC>(gsum, C, M);
  for (int cg = m.cg0; cg < m.cgs; cg += m.tpr) {
    // dx = A*dz + B*x + D  with A = gamma*invstd, B = -A*invstd*mean(dz*xhat), D = -A*mean(dz) - B*mean
    float ka[8], kb[8], kd[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = cg * 8 + k;
      const float sdz = gsum[c], sdzx = gsum[C + c];
      const BnBwdCoef q = bn_bwd_coef(ld_w(w, wdt, c), saved[c], saved[C + c], sdz, sdzx, inv_m, SYNC || k == 7);
      ka[k] = q.a; kb[k] = q.b; kd[k] = q.d;
      if (blockIdx.x == 0 && m.rlocal == 0) {
        if constexpr (SYNC) {
          st_w(dw, wdt, c, gsum[c - C]);          // local sum dz * xhat
          st_w(db, wdt, c, gsum[c - 2 * C]);      // local sum dz
        } else {
          st_w(dw, wdt, c, sdzx);
          st_w(db, wdt, c, sdz);
        }
      }
    }
    const int64_t stride = (int64_t)gridDim.x * m.rpp;
    const int64_t coff = cg * 8;
    int64_t r = (int64_t)blockIdx.x * m.rpp + m.rlocal;
    for (; r + 3 * stride < M; r += 4 * stride) {
      float d[4][8], v[4][8];
      unsigned bits[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t row = r + u * stride;
        load8<T>(dy + row * C + coff, d[u]);
        load8<T>(x + row * C + coff, v[u]);
        if constexpr (RELU) bits[u] = mask[row * m.cgs + cg];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t off = (r + u * stride) * C + coff;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float dz = d[u][k];
          if constexpr (RELU) dz = (bits[u] >> k) & 1u ? dz : 0.f;
          d[u][k] = dz;
          v[u][k] = bn_bwd_dx(ka[k], kb[k], kd[k], dz, v[u][k]);
        }
        store8<T>(dx + off, v[u]);
        if constexpr (RES) store8<T>(dres + off, d[u]);
      }
    }
    for (; r < M; r += stride) {
      float d[8], v[8];
      const int64_t off = r * C + coff;
      load8<T>(dy + off, d);
      load8<T>(x + off, v);
      unsigned bits = 0;
      if constexpr (RELU) bits = mask[r * m.cgs + cg];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float dz = d[k];
        if constexpr (RELU) dz = (bits >> k) & 1u ? dz : 0.f;
        d[k] = dz;
        v[k] = bn_bwd_dx(ka[k], kb[k], kd[k], dz, v[k]);
      }
      store8<T>(dx + off, v);
      if constexpr (RES) store8<T>(dres + off, d);
    }
  }
}
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_apply_kernel(BN_BWD_APPLY_PARAMS) {
  bn_bwd_apply_body<T, RELU, RES, false>(BN_BWD_APPLY_ARGS);
}
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_apply_sync_kernel(BN_BWD_APPLY_PARAMS) {
  bn_bwd_apply_body<T, RELU, RES, true>(BN_BWD_APPLY_ARGS);
}
#undef BN_BWD_APPLY_PARAMS
#undef BN_BWD_APPLY_ARGS

// ------------------------------------------------------------------ host side
static int wdtype(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return kF32;
    case at::kBFloat16: return kBF16;
    case at::kHalf: return kF16;
    default: TORCH_CHECK(false, "unsupported BN parameter dtype"); return 0;
  }
}

static void check_nhwc(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.dim() == 4, name, " must be a 4-d CUDA tensor");
  TORCH_CHECK(t.is_contiguous(at::MemoryFormat::ChannelsLast), name, " must be channels_last contiguous");
}

struct Geometry { int64_t M; int C; int tpr; int rpp; int sms; size_t smem; };
static Geometry geometry(const at::Tensor& x) {
  Geometry g;
  g.C = (int)x.size(1);
  g.M = x.numel() / g.C;
  TORCH_CHECK(g.C % 8 == 0 && g.C <= 16384, "fused BN needs C % 8 == 0 and C <= 16384 (got ", g.C, ")");
  g.tpr = std::min(g.C / 8, kBnThreads);
  g.rpp = kBnThreads / g.tpr;
  g.sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const bool pow2 = (g.tpr & (g.tpr - 1)) == 0;
  const int slots = (pow2 && g.tpr < 32) ? kBnWarps : g.rpp;
  g.smem = (size_t)slots * 2 * g.tpr * 8 * sizeof(float);
  return g;
}
// Resident CTAs per SM of a kernel (occupancy API, cached per kernel/smem).
template <typename K>
static int resident_ctas(K kernel, size_t smem) {
  static std::map<std::pair<const void*, size_t>, int> cache;
  const auto key = std::make_pair(reinterpret_cast<const void*>(kernel), smem);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  int n = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kBnThreads, smem) != cudaSuccess || n < 1) n = 1;
  cache[key] = n;
  return n;
}
// Reduction passes give every CTA ONE contiguous row range.  The grid is a whole number of waves: exactly
// sms * resident CTAs when the tensor is large (no partial last wave: 2.66 waves cost 12 % in the first profile),
// fewer CTAs with >= 8 row-passes each when it is small.
static int reduce_grid(const Geometry& g, int* rows_per_block, int resident = 4) {
  int64_t blocks = (g.M + (int64_t)g.rpp * 8 - 1) / ((int64_t)g.rpp * 8);
  const int64_t wave = (int64_t)g.sms * resident;
  if (blocks > wave) blocks = blocks >= 2 * wave && g.M / (2 * wave) >= (int64_t)g.rpp * 64 ? 2 * wave : wave;
  blocks = std::max<int64_t>(blocks, 1);
  int64_t rpb = (g.M + blocks - 1) / blocks;
  rpb = (rpb + g.rpp - 1) / g.rpp * g.rpp;
  *rows_per_block = (int)rpb;
  return (int)((g.M + rpb - 1) / rpb);
}
static int apply_grid(const Geometry& g) {
  int64_t blocks = (g.M + (int64_t)g.rpp * 4 - 1) / ((int64_t)g.rpp * 4);
  return (int)std::max<int64_t>(std::min<int64_t>(blocks, (int64_t)g.sms * 8), 1);
}

template <typename T> struct Tag { using type = T; };
// f(Tag<T>{}) with T the element type of the activations x
template <typename F>
static void for_act_dtype(const at::Tensor& x, F&& f) {
  switch (x.scalar_type()) {
    case at::kBFloat16: f(Tag<__nv_bfloat16>{}); break;
    case at::kHalf: f(Tag<__half>{}); break;
    case at::kFloat: f(Tag<float>{}); break;
    default: TORCH_CHECK(false, "unsupported activation dtype");
  }
}

template <typename U>
static U* ptr_or_null(const at::Tensor& t) { return t.defined() ? t.data_ptr<U>() : nullptr; }

// The per-channel sum / sum of squares a forward apply kernel reads from `work`.  reduce: one statistics pass over x adds
// them there first; otherwise they are in place already (eval mode reads none; stats_ready: the producing GEMM reduced
// them, gemm_bnstats.cu).
template <typename T>
static const float* forward_sums(const at::Tensor& x, const Geometry& g, const at::Tensor& work, bool reduce, const SyncBN* sync,
                                 cudaStream_t st) {
  float* wk = ptr_or_null<float>(work);
  if (!reduce) return work_sums(wk, g.C, sync);
  int rpb;
  const int grid = reduce_grid(g, &rpb, resident_ctas(bn_stats_kernel<T>, g.smem));
  at::Tensor part = partials(x, grid, g.C);
  bn_stats_kernel<T><<<grid, kBnThreads, g.smem, st>>>(reinterpret_cast<const T*>(x.data_ptr()), part.data_ptr<float>(), g.M, g.C, rpb);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return finish_sums(part.data_ptr<float>(), grid, g.C, g.M, wk, sync, st);
}

template <typename T>
static void fwd_impl(const at::Tensor& x, const at::Tensor* res, at::Tensor& y, at::Tensor& mask, at::Tensor& work, at::Tensor& saved,
                     const at::Tensor& w, const at::Tensor& b, at::Tensor& rm, at::Tensor& rv, at::Tensor& nbt, bool training, float momentum,
                     float eps, bool relu, bool stats_ready, const SyncBN* sync) {
  const Geometry g = geometry(x);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const float* sums = forward_sums<T>(x, g, work, training && !stats_ready, sync, st);
  using K = decltype(&bn_apply_kernel<T, false, false>);
  static constexpr K kernels[2][2][2] = {             // [sync][relu][res]
      {{bn_apply_kernel<T, false, false>, bn_apply_kernel<T, false, true>}, {bn_apply_kernel<T, true, false>, bn_apply_kernel<T, true, true>}},
      {{bn_apply_sync_kernel<T, false, false>, bn_apply_sync_kernel<T, false, true>},
       {bn_apply_sync_kernel<T, true, false>, bn_apply_sync_kernel<T, true, true>}}};
  kernels[sync != nullptr][relu][res != nullptr]<<<apply_grid(g), kBnThreads, 0, st>>>(
      reinterpret_cast<const T*>(x.data_ptr()), res ? reinterpret_cast<const T*>(res->data_ptr()) : nullptr, reinterpret_cast<T*>(y.data_ptr()),
      ptr_or_null<uint8_t>(mask), sums, w.data_ptr(), b.data_ptr(), wdtype(w), ptr_or_null<float>(rm), ptr_or_null<float>(rv),
      ptr_or_null<int64_t>(nbt), ptr_or_null<float>(saved), g.M, g.C, eps, momentum, training ? 1 : 0);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// returns {y, saved(mean|invstd), relu_mask}; `work` = the zeroed accumulator slice supplied by the caller (host.h: check_work)
std::vector<at::Tensor> bn_act_forward(const at::Tensor& x, const c10::optional<at::Tensor>& residual, const at::Tensor& weight,
                                       const at::Tensor& bias, at::Tensor running_mean, at::Tensor running_var,
                                       c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum, double eps, bool relu,
                                       bool need_mask, at::Tensor work, bool stats_ready, const SyncBN* sync) {
  check_nhwc(x, "x");
  TORCH_CHECK(!sync || training, "eval-mode BatchNorm is never synchronised");
  TORCH_CHECK(weight.scalar_type() == bias.scalar_type() && weight.is_contiguous() && bias.is_contiguous());
  if (running_mean.defined()) TORCH_CHECK(running_mean.scalar_type() == at::kFloat && running_var.scalar_type() == at::kFloat, "running stats must be fp32");
  TORCH_CHECK(training || running_mean.defined(), "eval mode needs running statistics");
  const at::Tensor* res = nullptr;
  if (residual.has_value() && residual->defined()) {
    check_nhwc(*residual, "residual");
    TORCH_CHECK(residual->sizes() == x.sizes() && residual->scalar_type() == x.scalar_type(), "residual must match x");
    res = &*residual;
  }
  c10::cuda::CUDAGuard guard(x.device());
  const int C = (int)x.size(1);
  at::Tensor y = at::empty_like(x, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  at::Tensor saved, mask, nbt;
  if (num_batches_tracked.has_value() && num_batches_tracked->defined()) {
    nbt = *num_batches_tracked;
    TORCH_CHECK(nbt.scalar_type() == at::kLong && nbt.is_cuda());
  }
  if (training) {
    check_work(work, C, sync);
    saved = at::empty({2 * C}, x.options().dtype(at::kFloat));
  }
  if (relu && need_mask) mask = at::empty({x.numel() / 8}, x.options().dtype(at::kByte));
  for_act_dtype(x, [&](auto t) {
    fwd_impl<typename decltype(t)::type>(x, res, y, mask, work, saved, weight, bias, running_mean, running_var, nbt, training, (float)momentum,
                                         (float)eps, relu, stats_ready, sync);
  });
  return {y, saved, mask};
}

// Second pass of a BatchNorm backward: finish the reduction pass's partials, then dx (and dres = dz with `dres`) from
// dz = dy (x the ReLU mask bits with `relu`).
template <typename T>
static void bwd_apply(const Geometry& g, const at::Tensor& part, const T* dy, const uint8_t* mask, const at::Tensor& x, const at::Tensor& saved,
                      at::Tensor& work, const at::Tensor& w, at::Tensor& dx, T* dres, at::Tensor& dw, at::Tensor& db, bool relu,
                      const SyncBN* sync, cudaStream_t st) {
  using K = decltype(&bn_bwd_apply_kernel<T, false, false>);
  static constexpr K kernels[2][2][2] = {             // [sync][relu][res]
      {{bn_bwd_apply_kernel<T, false, false>, bn_bwd_apply_kernel<T, false, true>},
       {bn_bwd_apply_kernel<T, true, false>, bn_bwd_apply_kernel<T, true, true>}},
      {{bn_bwd_apply_sync_kernel<T, false, false>, bn_bwd_apply_sync_kernel<T, false, true>},
       {bn_bwd_apply_sync_kernel<T, true, false>, bn_bwd_apply_sync_kernel<T, true, true>}}};
  const int wdt = wdtype(w);
  const float* sums = finish_sums(part.data_ptr<float>(), (int)part.size(0), g.C, g.M, work.data_ptr<float>(), sync, st);
  kernels[sync != nullptr][relu][dres != nullptr]<<<apply_grid(g), kBnThreads, 0, st>>>(
      dy, mask, reinterpret_cast<const T*>(x.data_ptr()), saved.data_ptr<float>(), sums, w.data_ptr(), wdt, reinterpret_cast<T*>(dx.data_ptr()),
      dres, dw.data_ptr(), db.data_ptr(), g.M, g.C);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// First pass of a BatchNorm backward: the per-CTA partials of sum dz and sum dz * xhat, dz = dy (x the ReLU bits with `mask`)
template <typename T>
static at::Tensor bwd_reduce(const Geometry& g, const T* dy, const uint8_t* mask, const at::Tensor& x, const at::Tensor& saved, cudaStream_t st) {
  const auto reduce = mask ? bn_bwd_reduce_kernel<T, true> : bn_bwd_reduce_kernel<T, false>;
  int rpb;
  const int rgrid = reduce_grid(g, &rpb, resident_ctas(reduce, g.smem));
  at::Tensor part = partials(x, rgrid, g.C);
  reduce<<<rgrid, kBnThreads, g.smem, st>>>(dy, mask, reinterpret_cast<const T*>(x.data_ptr()), saved.data_ptr<float>(), part.data_ptr<float>(),
                                            g.M, g.C, rpb);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return part;
}

template <typename T>
static void bwd_impl(const at::Tensor& dy, const at::Tensor& mask, const at::Tensor& x, const at::Tensor& saved, at::Tensor& work,
                     const at::Tensor& w, at::Tensor& dx, at::Tensor& dres, at::Tensor& dw, at::Tensor& db, bool relu, bool write_res,
                     const SyncBN* sync) {
  const Geometry g = geometry(x);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const T* dyp = reinterpret_cast<const T*>(dy.data_ptr());
  const uint8_t* mk = relu ? mask.data_ptr<uint8_t>() : nullptr;
  at::Tensor part = bwd_reduce<T>(g, dyp, mk, x, saved, st);
  bwd_apply<T>(g, part, dyp, mk, x, saved, work, w, dx, write_res ? reinterpret_cast<T*>(dres.data_ptr()) : nullptr, dw, db, relu, sync, st);
}

// returns {dx, dres (undefined if !has_residual), dweight, dbias}
std::vector<at::Tensor> bn_act_backward(const at::Tensor& dy_in, const at::Tensor& x, const c10::optional<at::Tensor>& mask_opt,
                                        const at::Tensor& weight, const at::Tensor& saved, bool relu, bool has_residual, at::Tensor work,
                                        const SyncBN* sync) {
  check_nhwc(x, "x");
  at::Tensor dy = dy_in.is_contiguous(at::MemoryFormat::ChannelsLast) ? dy_in : dy_in.contiguous(at::MemoryFormat::ChannelsLast);
  TORCH_CHECK(dy.scalar_type() == x.scalar_type() && dy.sizes() == x.sizes());
  at::Tensor mask;
  if (relu) {
    TORCH_CHECK(mask_opt.has_value() && mask_opt->defined() && mask_opt->scalar_type() == at::kByte && mask_opt->numel() == x.numel() / 8,
                "ReLU backward needs the forward's bit mask");
    mask = *mask_opt;
  }
  check_work(work, x.size(1), sync);
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor dx = at::empty_like(x, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  at::Tensor dres;
  if (has_residual) dres = (!relu) ? dy : at::empty_like(x, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  at::Tensor dw = at::empty_like(weight), db = at::empty_like(weight);
  const bool write_res = has_residual && relu;  // without ReLU the residual gradient IS dy: no copy
  for_act_dtype(x, [&](auto t) { bwd_impl<typename decltype(t)::type>(dy, mask, x, saved, work, weight, dx, dres, dw, db, relu, write_res, sync); });
  return {dx, dres, dw, db};
}

// ------------------------------------------------------------------ backward with a split incoming gradient
// A block output feeds two consumers (next conv1 and the skip connection), so autograd would first materialise
// dy = dy_a + dy_b with an ATen add (16 of them per ResNet-50 step, 1.2 ms) and this op would then read dy twice and
// write the masked residual gradient again.  Here the first pass does the add, the ReLU mask and the reductions at
// once and writes g = (dy_a + dy_b) * mask ONCE; g is both the residual gradient and the second pass's input:
//   eager : add 2R+1W, reduce 2R, apply 2R+2W  = 9 tensor passes      here : reduce 3R+1W, apply 2R+1W = 7
// The sum is rounded to T before it is used, i.e. bit-identical to what the ATen add would have produced.
template <typename T, bool RELU>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_reduce_sum_kernel(const T* __restrict__ dya, const T* __restrict__ dyb,
                                                                       const uint8_t* __restrict__ mask, const T* __restrict__ x,
                                                                       const float* __restrict__ saved, T* __restrict__ gout,
                                                                       float* __restrict__ part, int64_t M, int C, int rows_per_block) {
  extern __shared__ float sm[];
  const RowMap m = row_map(C);
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block, r1 = min(M, r0 + (int64_t)rows_per_block);
  for (int cgb = 0; cgb < m.cgs; cgb += m.tpr) {
    const int cg = cgb + m.cg0;
    float s[8], q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] = 0.f; q[k] = 0.f; }
    if (m.active && cg < m.cgs) {
      float mean[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) mean[k] = saved[cg * 8 + k];
      const int64_t coff = cg * 8;
      int64_t r = r0 + m.rlocal;
      for (; r + (int64_t)m.rpp < r1; r += 2 * (int64_t)m.rpp) {
        float d[2][8], e[2][8], v[2][8];
        unsigned bits[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int64_t row = r + (int64_t)u * m.rpp;
          load8<T>(dya + row * C + coff, d[u]);
          load8<T>(dyb + row * C + coff, e[u]);
          load8<T>(x + row * C + coff, v[u]);
          if constexpr (RELU) bits[u] = mask[row * m.cgs + cg];
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            float dz = to_f32<T>(from_f32<T>(d[u][k] + e[u][k]));
            if constexpr (RELU) dz = (bits[u] >> k) & 1u ? dz : 0.f;
            d[u][k] = dz;
            s[k] += dz;
            q[k] += dz * (v[u][k] - mean[k]);
          }
          store8<T>(gout + (r + (int64_t)u * m.rpp) * C + coff, d[u]);
        }
      }
      for (; r < r1; r += m.rpp) {
        float d[8], e[8], v[8];
        load8<T>(dya + r * C + coff, d);
        load8<T>(dyb + r * C + coff, e);
        load8<T>(x + r * C + coff, v);
        unsigned bits = 0;
        if constexpr (RELU) bits = mask[r * m.cgs + cg];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float dz = to_f32<T>(from_f32<T>(d[k] + e[k]));
          if constexpr (RELU) dz = (bits >> k) & 1u ? dz : 0.f;
          d[k] = dz;
          s[k] += dz;
          q[k] += dz * (v[k] - mean[k]);
        }
        store8<T>(gout + r * C + coff, d);
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) q[k] *= saved[C + cg * 8 + k];
    }
    cta_combine(m, cgb, s, q, sm, part, C);
  }
}

// First pass with a split incoming gradient: writes g = (dy_a + dy_b) (x the ReLU bits) and returns the per-CTA partials
template <typename T>
static at::Tensor bwd_reduce_sum(const Geometry& g, const at::Tensor& dya, const at::Tensor& dyb, const uint8_t* mask, const at::Tensor& x,
                                 const at::Tensor& saved, T* gout, cudaStream_t st) {
  const auto reduce = mask ? bn_bwd_reduce_sum_kernel<T, true> : bn_bwd_reduce_sum_kernel<T, false>;
  int rpb;
  const int rgrid = reduce_grid(g, &rpb, resident_ctas(reduce, g.smem));
  at::Tensor part = partials(x, rgrid, g.C);
  reduce<<<rgrid, kBnThreads, g.smem, st>>>(reinterpret_cast<const T*>(dya.data_ptr()), reinterpret_cast<const T*>(dyb.data_ptr()), mask,
                                            reinterpret_cast<const T*>(x.data_ptr()), saved.data_ptr<float>(), gout, part.data_ptr<float>(),
                                            g.M, g.C, rpb);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return part;
}

template <typename T>
static void bwd2_impl(const at::Tensor& dya, const at::Tensor& dyb, const at::Tensor& mask, const at::Tensor& x, const at::Tensor& saved,
                      at::Tensor& work, const at::Tensor& w, at::Tensor& g_out, at::Tensor& dx, at::Tensor& dw, at::Tensor& db, bool relu,
                      const SyncBN* sync) {
  const Geometry g = geometry(x);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  T* gp = reinterpret_cast<T*>(g_out.data_ptr());
  at::Tensor part = bwd_reduce_sum<T>(g, dya, dyb, relu ? mask.data_ptr<uint8_t>() : nullptr, x, saved, gp, st);
  // second pass: g already carries the mask, and it IS the residual gradient -> the plain (no ReLU, no dres) apply variant
  bwd_apply<T>(g, part, gp, nullptr, x, saved, work, w, dx, nullptr, dw, db, false, sync, st);
}

// returns {dx, g = (dy_a + dy_b) * relu_mask (the residual gradient), dweight, dbias}
std::vector<at::Tensor> bn_act_backward2(const at::Tensor& dy_a_in, const at::Tensor& dy_b_in, const at::Tensor& x,
                                         const c10::optional<at::Tensor>& mask_opt, const at::Tensor& weight, const at::Tensor& saved,
                                         bool relu, at::Tensor work, const SyncBN* sync) {
  check_nhwc(x, "x");
  const auto cl = at::MemoryFormat::ChannelsLast;
  at::Tensor dya = dy_a_in.is_contiguous(cl) ? dy_a_in : dy_a_in.contiguous(cl);
  at::Tensor dyb = dy_b_in.is_contiguous(cl) ? dy_b_in : dy_b_in.contiguous(cl);
  TORCH_CHECK(dya.scalar_type() == x.scalar_type() && dya.sizes() == x.sizes() && dya.device() == x.device(), "dy_a must match x");
  TORCH_CHECK(dyb.scalar_type() == x.scalar_type() && dyb.sizes() == x.sizes() && dyb.device() == x.device(), "dy_b must match x");
  at::Tensor mask;
  if (relu) {
    TORCH_CHECK(mask_opt.has_value() && mask_opt->defined() && mask_opt->scalar_type() == at::kByte && mask_opt->numel() == x.numel() / 8,
                "ReLU backward needs the forward's bit mask");
    mask = *mask_opt;
  }
  const int C = (int)x.size(1);
  check_work(work, C, sync);
  TORCH_CHECK(saved.defined() && saved.scalar_type() == at::kFloat && saved.numel() >= 2 * C, "saved statistics missing");
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor g = at::empty_like(x, x.options().memory_format(cl));
  at::Tensor dx = at::empty_like(x, x.options().memory_format(cl));
  at::Tensor dw = at::empty_like(weight), db = at::empty_like(weight);
  for_act_dtype(x, [&](auto t) { bwd2_impl<typename decltype(t)::type>(dya, dyb, mask, x, saved, work, weight, g, dx, dw, db, relu, sync); });
  return {dx, g, dw, db};
}

// ------------------------------------------------------------------ 1x1 conv -> BatchNorm pair: backward with the fused data gradient
// The reduction pass as in bn_act_backward (dy_b undefined) or bn_act_backward2, then the wgmma data-gradient GEMM that forms
// dx from g and y in shared memory as it loads them (gemm_bnstats.cu), instead of the apply pass followed by cuDNN's dgrad.
// y: the BatchNorm input (the conv output); conv_weight: [C_out, C_in, 1, 1]; this rank alone (no synchronised statistics).
// returns {d conv input, dx (d conv output, for the weight gradient), g (the residual gradient with dy_b, else undefined),
//          dweight, dbias}
std::vector<at::Tensor> conv1x1_bn_backward(const at::Tensor& dy_a_in, const c10::optional<at::Tensor>& dy_b_in, const at::Tensor& y,
                                            const c10::optional<at::Tensor>& mask_opt, const at::Tensor& weight, const at::Tensor& saved,
                                            const at::Tensor& conv_weight, bool relu, at::Tensor work) {
  check_nhwc(y, "y");
  const auto cl = at::MemoryFormat::ChannelsLast;
  TORCH_CHECK(y.scalar_type() == at::kBFloat16 || y.scalar_type() == at::kHalf, "conv1x1_bn_backward: bf16 or fp16 activations");
  at::Tensor dya = dy_a_in.is_contiguous(cl) ? dy_a_in : dy_a_in.contiguous(cl);
  TORCH_CHECK(dya.scalar_type() == y.scalar_type() && dya.sizes() == y.sizes() && dya.device() == y.device(), "dy_a must match y");
  const bool split = dy_b_in.has_value() && dy_b_in->defined();
  at::Tensor dyb;
  if (split) {
    dyb = dy_b_in->is_contiguous(cl) ? *dy_b_in : dy_b_in->contiguous(cl);
    TORCH_CHECK(dyb.scalar_type() == y.scalar_type() && dyb.sizes() == y.sizes() && dyb.device() == y.device(), "dy_b must match y");
  }
  const uint8_t* mk = nullptr;
  if (relu) {
    TORCH_CHECK(mask_opt.has_value() && mask_opt->defined() && mask_opt->scalar_type() == at::kByte && mask_opt->numel() == y.numel() / 8,
                "ReLU backward needs the forward's bit mask");
    mk = mask_opt->data_ptr<uint8_t>();
  }
  const int C = (int)y.size(1);
  check_work(work, C, nullptr);
  TORCH_CHECK(saved.defined() && saved.scalar_type() == at::kFloat && saved.numel() >= 2 * C, "saved statistics missing");
  c10::cuda::CUDAGuard guard(y.device());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const Geometry g = geometry(y);
  at::Tensor gt;                                  // the apply's input: dy_a, or the masked sum of the two gradients
  at::Tensor part;
  for_act_dtype(y, [&](auto t) {
    using T = typename decltype(t)::type;
    if (split) {
      gt = at::empty_like(y, y.options().memory_format(cl));
      part = bwd_reduce_sum<T>(g, dya, dyb, mk, y, saved, reinterpret_cast<T*>(gt.data_ptr()), st);
      mk = nullptr;                               // g already carries the mask
    } else {
      gt = dya;
      part = bwd_reduce<T>(g, reinterpret_cast<const T*>(dya.data_ptr()), mk, y, saved, st);
    }
  });
  const float* sums = finish_sums(part.data_ptr<float>(), (int)part.size(0), C, g.M, work.data_ptr<float>(), nullptr, st);
  at::Tensor dx = at::empty_like(y, y.options().memory_format(cl));
  at::Tensor din = at::empty({y.size(0), conv_weight.size(1), y.size(2), y.size(3)}, y.options().memory_format(cl));
  at::Tensor dw = at::empty_like(weight), db = at::empty_like(weight);
  conv1x1_dgrad_bn(gt, y, mk, saved, sums, weight, wdtype(weight), dw, db, conv_weight, dx, din);
  return {din, dx, split ? gt : at::Tensor(), dw, db};
}

}  // namespace ptd

// ====================================================================================================================
// Fused ResNet stem: BatchNorm + ReLU + MaxPool(3x3, stride 2, pad 1), NHWC.
//
// torchvision's stem (/root/reference/distributed.py:136-139 -> resnet.conv1/bn1/relu/maxpool) writes the full
// 112x112 activation, re-reads it for the pool, and in backward runs ATen's max_pool_backward_nhwc with int64 indices
// (int64 index traffic).  Here the normalised activation never touches HBM:
//   forward : one pass over the conv output: BN -> ReLU -> 3x3 max -> pooled output + a 4-bit arg-max code per element
//             (code 15 = "all candidates <= 0": the ReLU killed the gradient)
//   backward: two passes over the INPUT domain; each input position gathers the (at most 4) pooled gradients whose
//             window selected it, which yields dz for the BN backward reductions / apply without ever materialising
//             the 112x112 gradient of the pool.
namespace ptd {

struct PoolGeom { int H, W, OH, OW; };

__device__ __forceinline__ void stem_scale_shift(const float* gsum, const float* rm, const float* rv, const void* w, const void* b, int wdt,
                                                 int cg, int C, float inv_m, float eps, int training, float (&sc)[8], float (&sh)[8],
                                                 float (&mean)[8], float (&var)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = cg * 8 + k;
    if (training) {
      mean[k] = gsum[c] * inv_m;
      var[k] = fmaxf(gsum[C + c] * inv_m - mean[k] * mean[k], 0.f);
    } else {
      mean[k] = rm[c];
      var[k] = rv[c];
    }
    const float invstd = rsqrtf(var[k] + eps);
    sc[k] = ld_w(w, wdt, c) * invstd;
    sh[k] = ld_w(b, wdt, c) - mean[k] * sc[k];
  }
}

#define STEM_FWD_PARAMS                                                                                                    \
  const T *__restrict__ x, T *__restrict__ y, uint2 *__restrict__ code, const float *__restrict__ gsum,                   \
      const void *__restrict__ w, const void *__restrict__ b, int wdt, float *__restrict__ running_mean,                  \
      float *__restrict__ running_var, int64_t *__restrict__ nbt, float *__restrict__ saved, int64_t M, int N, int C,     \
      PoolGeom g, float eps, float momentum, int training
#define STEM_FWD_ARGS x, y, code, gsum, w, b, wdt, running_mean, running_var, nbt, saved, M, N, C, g, eps, momentum, training
template <typename T, bool SYNC>
__device__ __forceinline__ void stem_fwd_body(STEM_FWD_PARAMS) {
  const int cgs = C >> 3;
  const int cg = threadIdx.x % cgs;                 // host guarantees blockDim.x % cgs == 0
  const int64_t rows = stat_rows<SYNC>(gsum, C, M);
  float sc[8], sh[8], mean[8], var[8];
  stem_scale_shift(gsum, running_mean, running_var, w, b, wdt, cg, C, 1.f / (float)rows, eps, training, sc, sh, mean, var);
  if (training && blockIdx.x == 0 && threadIdx.x < cgs) {
    if (threadIdx.x == 0 && nbt) *nbt += 1;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = cg * 8 + k;
      saved[c] = mean[k];
      saved[C + c] = rsqrtf(var[k] + eps);
      if (running_mean) {
        const float unbiased = rows > 1 ? var[k] * ((float)rows / (float)(rows - 1)) : var[k];
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean[k];
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
      }
    }
  }
  const int64_t total = (int64_t)N * g.OH * g.OW;
  const int ppb = blockDim.x / cgs;                  // output pixels per CTA pass
  // 32-bit index math (host checks the pixel counts fit): 64-bit div/mod would dominate the instruction stream
  for (int p = blockIdx.x * ppb + threadIdx.x / cgs; p < (int)total; p += gridDim.x * ppb) {
    const int ow = p % g.OW;
    const int t_ = p / g.OW;
    const int oh = t_ % g.OH;
    const int64_t n = t_ / g.OH;
    float best[8];
    uint32_t sel[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { best[k] = 0.f; sel[k] = 15u; }
    const T* base = x + n * g.H * g.W * C + cg * 8;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = 2 * oh - 1 + kh;
      if (ih < 0 || ih >= g.H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int iw = 2 * ow - 1 + kw;
        if (iw < 0 || iw >= g.W) continue;
        float f[8];
        load8<T>(base + ((int64_t)ih * g.W + iw) * C, f);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float v = f[k] * sc[k] + sh[k];
          if (v > best[k]) { best[k] = v; sel[k] = (uint32_t)(kh * 3 + kw); }
        }
      }
    }
    store8<T>(y + (int64_t)p * C + cg * 8, best);
    if (code) {   // one byte per channel: the backward compares 4 channels per instruction (vcmpeq4)
      uint2 word;
      word.x = sel[0] | (sel[1] << 8) | (sel[2] << 16) | (sel[3] << 24);
      word.y = sel[4] | (sel[5] << 8) | (sel[6] << 16) | (sel[7] << 24);
      code[(int64_t)p * cgs + cg] = word;
    }
  }
}
template <typename T>
__global__ void __launch_bounds__(kBnThreads) stem_fwd_kernel(STEM_FWD_PARAMS) { stem_fwd_body<T, false>(STEM_FWD_ARGS); }
template <typename T>
__global__ void __launch_bounds__(kBnThreads) stem_fwd_sync_kernel(STEM_FWD_PARAMS) { stem_fwd_body<T, true>(STEM_FWD_ARGS); }
#undef STEM_FWD_PARAMS
#undef STEM_FWD_ARGS

// dz (gradient w.r.t. the BN+ReLU output at one input position) = sum of the pooled gradients that selected it.
// 16-bit dtypes stay packed: vcmpeq4 turns the 8 arg-max bytes into byte masks, PRMT widens them to 16-bit lane masks,
// the masked bf16x2/half2 pairs are accumulated with packed adds (at most 4 terms) and widened to fp32 once.
template <typename T> struct Pair;
template <> struct Pair<__nv_bfloat16> {
  using P = __nv_bfloat162;
  static __device__ __forceinline__ uint32_t add(uint32_t a, uint32_t b) {
    P r = __hadd2(*reinterpret_cast<P*>(&a), *reinterpret_cast<P*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
  }
  static __device__ __forceinline__ float2 widen(uint32_t a) { return __bfloat1622float2(*reinterpret_cast<P*>(&a)); }
};
template <> struct Pair<__half> {
  using P = __half2;
  static __device__ __forceinline__ uint32_t add(uint32_t a, uint32_t b) {
    P r = __hadd2(*reinterpret_cast<P*>(&a), *reinterpret_cast<P*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
  }
  static __device__ __forceinline__ float2 widen(uint32_t a) { return __half22float2(*reinterpret_cast<P*>(&a)); }
};

template <typename T>
__device__ __forceinline__ void stem_gather_dz(const T* __restrict__ dp, const uint2* __restrict__ code, int64_t n, int ih, int iw, int cg,
                                               int cgs, int C, const PoolGeom& g, float (&dz)[8]) {
  const int oh0 = ih >> 1, oh1 = min((ih + 1) >> 1, g.OH - 1);
  const int ow0 = iw >> 1, ow1 = min((iw + 1) >> 1, g.OW - 1);
  if constexpr (sizeof(T) == 2) {
    uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;      // +0.0 pairs
    for (int oh = oh0; oh <= oh1; ++oh) {
      const int kh = ih - (2 * oh - 1);
      for (int ow = ow0; ow <= ow1; ++ow) {
        const uint32_t pat = (uint32_t)(kh * 3 + iw - (2 * ow - 1)) * 0x01010101u;
        const int64_t p = (n * g.OH + oh) * g.OW + ow;
        const uint2 cw = code[p * cgs + cg];
        const V4 d = ld_stream(dp + p * C + cg * 8);
        const uint32_t m0 = __vcmpeq4(cw.x, pat), m1 = __vcmpeq4(cw.y, pat);
        a0 = Pair<T>::add(a0, d.x & __byte_perm(m0, 0, 0x1100));
        a1 = Pair<T>::add(a1, d.y & __byte_perm(m0, 0, 0x3322));
        a2 = Pair<T>::add(a2, d.z & __byte_perm(m1, 0, 0x1100));
        a3 = Pair<T>::add(a3, d.w & __byte_perm(m1, 0, 0x3322));
      }
    }
    float2 t;
    t = Pair<T>::widen(a0); dz[0] = t.x; dz[1] = t.y;
    t = Pair<T>::widen(a1); dz[2] = t.x; dz[3] = t.y;
    t = Pair<T>::widen(a2); dz[4] = t.x; dz[5] = t.y;
    t = Pair<T>::widen(a3); dz[6] = t.x; dz[7] = t.y;
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) dz[k] = 0.f;
    for (int oh = oh0; oh <= oh1; ++oh) {
      const int kh = ih - (2 * oh - 1);
      for (int ow = ow0; ow <= ow1; ++ow) {
        const uint32_t want = (uint32_t)(kh * 3 + iw - (2 * ow - 1));
        const int64_t p = (n * g.OH + oh) * g.OW + ow;
        const uint2 cw = code[p * cgs + cg];
        float d[8];
        load8<T>(dp + p * C + cg * 8, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t sel = ((k < 4 ? cw.x : cw.y) >> (8 * (k & 3))) & 255u;
          dz[k] += sel == want ? d[k] : 0.f;
        }
      }
    }
  }
}

// Backward over 2x2 QUADS of input positions.  The four positions (2k..2k+1, 2j..2j+1) are covered by exactly four
// pooling windows A=(k,j) B=(k,j+1) C=(k+1,j) D=(k+1,j+1); each window's (arg-max bytes, pooled gradient) is loaded ONCE
// per quad and matched against the nine (window, position) slots:
//     dz00 = A@4        dz01 = A@5 + B@3        dz10 = A@7 + C@1        dz11 = A@8 + B@6 + C@2 + D@0
// so every lane does the same work (no parity divergence) and the per-position instruction count drops ~5x versus a
// per-position gather.  A CTA owns `rows_per_block` quad rows (n, k): n and k are CTA-uniform scalars.
template <typename T>
struct QuadDz {                                         // packed accumulators: 4 positions x 4 pair-words
  uint32_t a[4][4];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) a[i][j] = 0u;
  }
  __device__ __forceinline__ void hit(int pos, const uint2& cw, const V4& d, uint32_t want) {
    const uint32_t pat = want * 0x01010101u;
    const uint32_t m0 = __vcmpeq4(cw.x, pat), m1 = __vcmpeq4(cw.y, pat);
    a[pos][0] = Pair<T>::add(a[pos][0], d.x & __byte_perm(m0, 0, 0x1100));
    a[pos][1] = Pair<T>::add(a[pos][1], d.y & __byte_perm(m0, 0, 0x3322));
    a[pos][2] = Pair<T>::add(a[pos][2], d.z & __byte_perm(m1, 0, 0x1100));
    a[pos][3] = Pair<T>::add(a[pos][3], d.w & __byte_perm(m1, 0, 0x3322));
  }
  __device__ __forceinline__ void widen(int pos, float (&dz)[8]) const {
    float2 t;
    t = Pair<T>::widen(a[pos][0]); dz[0] = t.x; dz[1] = t.y;
    t = Pair<T>::widen(a[pos][1]); dz[2] = t.x; dz[3] = t.y;
    t = Pair<T>::widen(a[pos][2]); dz[4] = t.x; dz[5] = t.y;
    t = Pair<T>::widen(a[pos][3]); dz[6] = t.x; dz[7] = t.y;
  }
};

// dz of the quad (n, k, j) for channel group cg; 16-bit dtypes only (fp32 uses the per-position gather)
template <typename T>
__device__ __forceinline__ void stem_quad_dz(const T* __restrict__ dp, const uint2* __restrict__ code, int64_t n, int k, int j, int cg, int cgs,
                                             int C, const PoolGeom& g, QuadDz<T>& qd) {
  qd.clear();
  const bool has_r = (j + 1) < g.OW, has_b = (k + 1) < g.OH;
  const int64_t pA = (n * g.OH + k) * g.OW + j;
  {
    const uint2 cw = code[pA * cgs + cg];
    const V4 d = ld_stream(dp + pA * C + cg * 8);
    qd.hit(0, cw, d, 4u); qd.hit(1, cw, d, 5u); qd.hit(2, cw, d, 7u); qd.hit(3, cw, d, 8u);
  }
  if (has_r) {
    const uint2 cw = code[(pA + 1) * cgs + cg];
    const V4 d = ld_stream(dp + (pA + 1) * C + cg * 8);
    qd.hit(1, cw, d, 3u); qd.hit(3, cw, d, 6u);
  }
  if (has_b) {
    const int64_t pC = pA + g.OW;
    const uint2 cw = code[pC * cgs + cg];
    const V4 d = ld_stream(dp + pC * C + cg * 8);
    qd.hit(2, cw, d, 1u); qd.hit(3, cw, d, 2u);
    if (has_r) {
      const uint2 cw2 = code[(pC + 1) * cgs + cg];
      const V4 d2 = ld_stream(dp + (pC + 1) * C + cg * 8);
      qd.hit(3, cw2, d2, 0u);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads, 4) stem_bwd_reduce_kernel(const T* __restrict__ dp, const uint2* __restrict__ code,
                                                                     const T* __restrict__ x, const float* __restrict__ saved,
                                                                     float* __restrict__ part, int64_t M, int C, PoolGeom g,
                                                                     int rows_per_block) {
  extern __shared__ float sm[];
  const RowMap m = row_map(C);                       // tpr == cgs (host guarantees cgs divides the CTA size)
  const int cg = m.cg0;
  const int QH = (g.H + 1) >> 1, QW = (g.W + 1) >> 1;
  const int nrows = (int)(M / ((int64_t)g.H * g.W)) * QH;   // quad rows
  const int row0 = blockIdx.x * rows_per_block, row1 = min(nrows, row0 + rows_per_block);
  float s[8], q[8], mean[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { s[k] = 0.f; q[k] = 0.f; mean[k] = saved[cg * 8 + k]; }
  for (int row = row0; row < row1; ++row) {
    const int n = row / QH, k = row - n * QH;
    for (int j = m.rlocal; j < QW; j += m.rpp) {
      if constexpr (sizeof(T) == 2) {
        QuadDz<T> qd;
        stem_quad_dz<T>(dp, code, n, k, j, cg, m.cgs, C, g, qd);
#pragma unroll
        for (int pos = 0; pos < 4; ++pos) {
          const int ih = 2 * k + (pos >> 1), iw = 2 * j + (pos & 1);
          if (ih < g.H && iw < g.W) {
            float dz[8], v[8];
            qd.widen(pos, dz);
            load8<T>(x + (((int64_t)n * g.H + ih) * g.W + iw) * C + cg * 8, v);
#pragma unroll
            for (int c = 0; c < 8; ++c) { s[c] += dz[c]; q[c] += dz[c] * (v[c] - mean[c]); }
          }
        }
      } else {
#pragma unroll
        for (int pos = 0; pos < 4; ++pos) {
          const int ih = 2 * k + (pos >> 1), iw = 2 * j + (pos & 1);
          if (ih < g.H && iw < g.W) {
            float dz[8], v[8];
            stem_gather_dz<T>(dp, code, n, ih, iw, cg, m.cgs, C, g, dz);
            load8<T>(x + (((int64_t)n * g.H + ih) * g.W + iw) * C + cg * 8, v);
#pragma unroll
            for (int c = 0; c < 8; ++c) { s[c] += dz[c]; q[c] += dz[c] * (v[c] - mean[c]); }
          }
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) q[k] *= saved[C + cg * 8 + k];
  cta_combine(m, 0, s, q, sm, part, C);
}

#define STEM_BWD_APPLY_PARAMS                                                                                              \
  const T *__restrict__ dp, const uint2 *__restrict__ code, const T *__restrict__ x, const float *__restrict__ saved,      \
      const float *__restrict__ gsum, const void *__restrict__ w, int wdt, T *__restrict__ dx, void *__restrict__ dw,     \
      void *__restrict__ db, int64_t M, int C, PoolGeom g, int rows_per_block
#define STEM_BWD_APPLY_ARGS dp, code, x, saved, gsum, w, wdt, dx, dw, db, M, C, g, rows_per_block
template <typename T, bool SYNC>
__device__ __forceinline__ void stem_bwd_apply_body(STEM_BWD_APPLY_PARAMS) {
  const RowMap m = row_map(C);
  const int cg = m.cg0;
  const float inv_m = 1.f / (float)stat_rows<SYNC>(gsum, C, M);
  float ka[8], kb[8], kd[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = cg * 8 + k;
    const float mean = saved[c], invstd = saved[C + c];
    const float sdz = gsum[c], sdzx = gsum[C + c];
    ka[k] = ld_w(w, wdt, c) * invstd;
    kb[k] = -ka[k] * invstd * sdzx * inv_m;
    kd[k] = -ka[k] * sdz * inv_m - kb[k] * mean;
    if (blockIdx.x == 0 && m.rlocal == 0) {
      if constexpr (SYNC) {                  // dgamma / dbeta: this rank's sums (see bn_bwd_apply_body)
        st_w(dw, wdt, c, gsum[c - C]);
        st_w(db, wdt, c, gsum[c - 2 * C]);
      } else {
        st_w(dw, wdt, c, sdzx);
        st_w(db, wdt, c, sdz);
      }
    }
  }
  const int QH = (g.H + 1) >> 1, QW = (g.W + 1) >> 1;
  const int nrows = (int)(M / ((int64_t)g.H * g.W)) * QH;
  const int row0 = blockIdx.x * rows_per_block, row1 = min(nrows, row0 + rows_per_block);
  for (int row = row0; row < row1; ++row) {
    const int n = row / QH, k = row - n * QH;
    for (int j = m.rlocal; j < QW; j += m.rpp) {
      QuadDz<T> qd;
      if constexpr (sizeof(T) == 2) stem_quad_dz<T>(dp, code, n, k, j, cg, m.cgs, C, g, qd);
#pragma unroll
      for (int pos = 0; pos < 4; ++pos) {
        const int ih = 2 * k + (pos >> 1), iw = 2 * j + (pos & 1);
        if (ih < g.H && iw < g.W) {
          float dz[8], v[8];
          if constexpr (sizeof(T) == 2) qd.widen(pos, dz);
          else stem_gather_dz<T>(dp, code, n, ih, iw, cg, m.cgs, C, g, dz);
          const int64_t off = (((int64_t)n * g.H + ih) * g.W + iw) * C + cg * 8;
          load8<T>(x + off, v);
#pragma unroll
          for (int c = 0; c < 8; ++c) v[c] = ka[c] * dz[c] + kb[c] * v[c] + kd[c];
          store8<T>(dx + off, v);
        }
      }
    }
  }
}
template <typename T>
__global__ void __launch_bounds__(kBnThreads, 4) stem_bwd_apply_kernel(STEM_BWD_APPLY_PARAMS) {
  stem_bwd_apply_body<T, false>(STEM_BWD_APPLY_ARGS);
}
template <typename T>
__global__ void __launch_bounds__(kBnThreads) stem_bwd_apply_sync_kernel(STEM_BWD_APPLY_PARAMS) {   // no spills at 4 CTAs/SM
  stem_bwd_apply_body<T, true>(STEM_BWD_APPLY_ARGS);
}
#undef STEM_BWD_APPLY_PARAMS
#undef STEM_BWD_APPLY_ARGS

static PoolGeom pool_geom(const at::Tensor& x) {
  PoolGeom g;
  g.H = (int)x.size(2);
  g.W = (int)x.size(3);
  g.OH = (g.H + 2 - 3) / 2 + 1;
  g.OW = (g.W + 2 - 3) / 2 + 1;
  return g;
}

template <typename T>
static void stem_fwd_impl(const at::Tensor& x, at::Tensor& y, at::Tensor& code, at::Tensor& work, at::Tensor& saved, const at::Tensor& w,
                          const at::Tensor& b, at::Tensor& rm, at::Tensor& rv, at::Tensor& nbt, bool training, float momentum, float eps,
                          bool stats_ready, const SyncBN* sync) {
  const Geometry g = geometry(x);
  const PoolGeom pg = pool_geom(x);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const float* sums = forward_sums<T>(x, g, work, training && !stats_ready, sync, st);
  const int cgs = g.C / 8;
  const int64_t total = x.size(0) * pg.OH * pg.OW;
  const int ppb = kBnThreads / cgs;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((total + ppb - 1) / ppb, (int64_t)g.sms * 16));
  static constexpr decltype(&stem_fwd_kernel<T>) kernels[2] = {stem_fwd_kernel<T>, stem_fwd_sync_kernel<T>};   // [sync]
  kernels[sync != nullptr]<<<grid, kBnThreads, 0, st>>>(
      reinterpret_cast<const T*>(x.data_ptr()), reinterpret_cast<T*>(y.data_ptr()), reinterpret_cast<uint2*>(ptr_or_null<uint8_t>(code)), sums,
      w.data_ptr(), b.data_ptr(), wdtype(w), ptr_or_null<float>(rm), ptr_or_null<float>(rv), ptr_or_null<int64_t>(nbt),
      ptr_or_null<float>(saved), g.M, (int)x.size(0), g.C, pg, eps, momentum, training ? 1 : 0);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// relu(bn(x)) -> maxpool 3x3/2/1.  returns {y_pool, saved, code}
static std::vector<at::Tensor> stem_forward_common(const at::Tensor& x, const at::Tensor& weight, const at::Tensor& bias,
                                                   at::Tensor running_mean, at::Tensor running_var,
                                                   c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum, double eps,
                                                   bool need_code, at::Tensor work, bool stats_ready, const SyncBN* sync) {
  check_nhwc(x, "x");
  TORCH_CHECK(!sync || training, "eval-mode BatchNorm is never synchronised");
  const int C = (int)x.size(1);
  TORCH_CHECK(C % 8 == 0 && kBnThreads % (C / 8) == 0, "fused stem needs C/8 to divide ", kBnThreads);
  TORCH_CHECK(x.numel() / C < (int64_t)1 << 30, "fused stem: too many pixels for 32-bit indexing");
  TORCH_CHECK(training || running_mean.defined(), "eval mode needs running statistics");
  c10::cuda::CUDAGuard guard(x.device());
  const PoolGeom pg = pool_geom(x);
  at::Tensor y = at::empty({x.size(0), C, pg.OH, pg.OW}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  at::Tensor saved, code, nbt;
  if (num_batches_tracked.has_value() && num_batches_tracked->defined()) nbt = *num_batches_tracked;
  if (training) {
    check_work(work, C, sync);
    saved = at::empty({2 * C}, x.options().dtype(at::kFloat));
  }
  if (need_code) code = at::empty({y.numel()}, x.options().dtype(at::kByte));
  for_act_dtype(x, [&](auto t) {
    stem_fwd_impl<typename decltype(t)::type>(x, y, code, work, saved, weight, bias, running_mean, running_var, nbt, training, (float)momentum,
                                              (float)eps, stats_ready, sync);
  });
  return {y, saved, code};
}

std::vector<at::Tensor> stem_forward(const at::Tensor& x, const at::Tensor& weight, const at::Tensor& bias, at::Tensor running_mean,
                                     at::Tensor running_var, c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum,
                                     double eps, bool need_code, at::Tensor work, const SyncBN* sync) {
  return stem_forward_common(x, weight, bias, running_mean, running_var, num_batches_tracked, training, momentum, eps, need_code, work, false,
                             sync);
}
// same, with the per-channel sum / sum of squares of x already accumulated in work[0:2C] (stem convolution run as a GEMM;
// synchronised: the GEMM's exchange already filled the whole work slice)
std::vector<at::Tensor> stem_forward_pre(const at::Tensor& x, const at::Tensor& weight, const at::Tensor& bias, at::Tensor running_mean,
                                         at::Tensor running_var, c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum,
                                         double eps, bool need_code, at::Tensor work, const SyncBN* sync) {
  return stem_forward_common(x, weight, bias, running_mean, running_var, num_batches_tracked, training, momentum, eps, need_code, work, true,
                             sync);
}

template <typename T>
static void stem_bwd_impl(const at::Tensor& dp, const at::Tensor& code, const at::Tensor& x, const at::Tensor& saved, at::Tensor& work,
                          const at::Tensor& w, at::Tensor& dx, at::Tensor& dw, at::Tensor& db, const SyncBN* sync) {
  const Geometry g = geometry(x);
  const PoolGeom pg = pool_geom(x);
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const T* dpp = reinterpret_cast<const T*>(dp.data_ptr());
  const uint2* cp = reinterpret_cast<const uint2*>(code.data_ptr());
  const T* xp = reinterpret_cast<const T*>(x.data_ptr());
  const int nrows = (int)(x.size(0) * ((pg.H + 1) / 2));               // quad rows
  const int rpb = std::max(1, std::min(4, nrows / (g.sms * 8)));       // quad rows per CTA
  const int grid = (nrows + rpb - 1) / rpb;
  at::Tensor part = partials(x, grid, g.C);
  stem_bwd_reduce_kernel<T><<<grid, kBnThreads, g.smem, st>>>(dpp, cp, xp, saved.data_ptr<float>(), part.data_ptr<float>(), g.M, g.C, pg, rpb);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  const float* sums = finish_sums(part.data_ptr<float>(), grid, g.C, g.M, work.data_ptr<float>(), sync, st);
  static constexpr decltype(&stem_bwd_apply_kernel<T>) kernels[2] = {stem_bwd_apply_kernel<T>, stem_bwd_apply_sync_kernel<T>};   // [sync]
  kernels[sync != nullptr]<<<grid, kBnThreads, 0, st>>>(dpp, cp, xp, saved.data_ptr<float>(), sums, w.data_ptr(), wdtype(w),
                                                        reinterpret_cast<T*>(dx.data_ptr()), dw.data_ptr(), db.data_ptr(), g.M, g.C, pg, rpb);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// returns {dx, dweight, dbias}
std::vector<at::Tensor> stem_backward(const at::Tensor& dp_in, const at::Tensor& x, const at::Tensor& code, const at::Tensor& weight,
                                      const at::Tensor& saved, at::Tensor work, const SyncBN* sync) {
  check_nhwc(x, "x");
  at::Tensor dp = dp_in.is_contiguous(at::MemoryFormat::ChannelsLast) ? dp_in : dp_in.contiguous(at::MemoryFormat::ChannelsLast);
  const int C = (int)x.size(1);
  TORCH_CHECK(dp.scalar_type() == x.scalar_type() && dp.size(1) == C && code.scalar_type() == at::kByte && code.numel() == dp.numel());
  check_work(work, C, sync);
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor dx = at::empty_like(x, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  at::Tensor dw = at::empty_like(weight), db = at::empty_like(weight);
  for_act_dtype(x, [&](auto t) { stem_bwd_impl<typename decltype(t)::type>(dp, code, x, saved, work, weight, dx, dw, db, sync); });
  return {dx, dw, db};
}

}  // namespace ptd
