// 1x1 convolution (NHWC) as a wgmma GEMM with the BatchNorm statistics fused into the epilogue (sm_90a).
//
//   C[M, N] (T) = A[M, K] (T activations, K = C_in contiguous) x B[N, K]^T (T weights [C_out, C_in]),  T = bf16 or fp16
//   gsum[0:N]  += sum_m C[m, n]          gsum[N:2N] += sum_m C[m, n]^2          (fp32, over the stored 16-bit values)
//
// In a ResNet-50 step the 1x1 convolutions are HBM-bound, so the only way to make them cheaper is to do more per byte:
// the per-channel sum / sum-of-squares that BatchNorm needs are reduced here from the output tile while it sits in
// shared memory on its way out, which removes BN's separate statistics pass (one full re-read of the conv output).
// Call site: every conv1x1 -> bn pair of the Bottleneck blocks (models/resnet.py, ops/conv_bn.py) and the stem GEMM.
//
// Hopper structure: persistent CTAs, one per SM, each with a FIXED n-tile (so its per-channel partial sums stay in
// registers for the CTA's lifetime and reach global memory once) and m-tiles strided by the number of CTAs per n-tile;
// CTAs with adjacent ids share the same m-tile sequence, so an A tile is fetched from HBM once and hit in L2 by the
// other n-tiles.
//   warp 8        TMA producer : cp.async.bulk.tensor.2d (128B-swizzled 128x64 A tile, BLOCK_Nx64 B tile) -> smem ring,
//                                completion on an mbarrier (expect_tx); runs ahead across tile boundaries
//   warpgroups 0,1 consumers   : warpgroup c owns rows [64c, 64c+64) of the 128-row tile; wgmma.mma_async m64nXk16
//                                (T x T -> fp32 registers) straight from the swizzled smem stages; epilogue packs
//                                T into a 128B-swizzled staging tile, one TMA store per 64x64 box (clipped at the M
//                                tail by the tensor map), column owners reduce the statistics from the staged values.
//
// bf16 and fp16 share everything but the wgmma operand type, the tensor-map element type and the pack / unpack of the
// epilogue (both are 2-byte elements with the same swizzled layout).  Products of two fp16 (or two bf16) values are exact
// in fp32, so both accumulate the same way.  fp16 output is rounded to nearest even (__floats2half2_rn): a value of
// magnitude >= 65520 is stored as +-inf, and the sums of that channel become inf / nan - what cuDNN followed by a separate
// statistics pass over the stored tensor gives.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda.h>
#include <torch/extension.h>

#include "bn_combine.cuh"
#include "common.cuh"
#include "host.h"

namespace ptd {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;          // 64 16-bit elements = one 128-byte swizzle row
constexpr int kConsumerThreads = 256;
constexpr int kGemmThreads = kConsumerThreads + 32;

template <int BLOCK_N> struct GemmCfg {
  static constexpr int kStages = BLOCK_N == 256 ? 3 : 4;
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kCBytes = kBlockM * BLOCK_N * 2;               // 16-bit output staging, [BLOCK_N / 64] 64-column boxes
  static constexpr int kStatFloats = 2 * 4 * 128;                     // [2 warpgroups][4 sums][128 threads]
  static constexpr int kSmem = 1024 + kStages * (kABytes + kBBytes) + kCBytes + kStatFloats * 4 + 2 * kStages * 8;
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done, spins = 0;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    if (!done && ++spins > (1u << 24)) __trap();      // a lost arrival must not hang the GPU
  } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void named_barrier(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 bytes apart (SBO), LBO unused (=1).
// The tile is 1024-byte aligned; +2 in the (>>4) start-address field advances K by 16 elements (32 bytes).
__device__ __forceinline__ uint64_t gmma_desc(const void* smem_tile) {
  const uint64_t addr = (uint64_t)(smem_u32(smem_tile) >> 4) & 0x3FFFull;
  return addr | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

#define PTD_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, fp32 accumulators in d[32]; TY: the operand type, "bf16" or "f16"
#define PTD_WGMMA_N64(TY)                                                                                             \
  asm volatile(                                                                                                       \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                              \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " "                                                     \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                       \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}" \
      : PTD_F8(0), PTD_F8(8), PTD_F8(16), PTD_F8(24)                                                                  \
      : "l"(adesc), "l"(bdesc), "r"(accumulate))
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, fp32 accumulators in d[64]
#define PTD_WGMMA_N128(TY)                                                                                            \
  asm volatile(                                                                                                       \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                              \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                    \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                       \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                              \
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                              \
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}" \
      : PTD_F8(0), PTD_F8(8), PTD_F8(16), PTD_F8(24), PTD_F8(32), PTD_F8(40), PTD_F8(48), PTD_F8(56)                  \
      : "l"(adesc), "l"(bdesc), "r"(accumulate))

template <typename T> __device__ __forceinline__ void wgmma_n64(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
  if constexpr (std::is_same<T, __half>::value) PTD_WGMMA_N64("f16");
  else PTD_WGMMA_N64("bf16");
}
template <typename T> __device__ __forceinline__ void wgmma_n128(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
  if constexpr (std::is_same<T, __half>::value) PTD_WGMMA_N128("f16");
  else PTD_WGMMA_N128("bf16");
}
#undef PTD_WGMMA_N64
#undef PTD_WGMMA_N128
#undef PTD_F8

// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <typename T, int BLOCK_N>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_bnstats_kernel(const __grid_constant__ CUtensorMap tmap_a,
                                                                       const __grid_constant__ CUtensorMap tmap_b,
                                                                       const __grid_constant__ CUtensorMap tmap_c,
                                                                       float* __restrict__ part, int N, int K, int m_tiles,
                                                                       int n_tiles, int ctas_per_n) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kInstN = BLOCK_N >= 128 ? 128 : 64;                  // wgmma N per instruction
  constexpr int kBoxes = BLOCK_N / 64;                               // 64-column output boxes
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smem_a = smem;                                            // [kStages][128 x 64] T, 128B swizzle
  uint8_t* smem_b = smem_a + kStages * Cfg::kABytes;                 // [kStages][BLOCK_N x 64]
  uint8_t* smem_c = smem_b + kStages * Cfg::kBBytes;                 // [2 warpgroups][kBoxes][64 x 64] T, 128B swizzle
  float* smem_stats = reinterpret_cast<float*>(smem_c + Cfg::kCBytes);   // [2 warpgroups][s0 s1 q0 q1][128 threads]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_stats + Cfg::kStatFloats);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x % n_tiles;           // fixed for this CTA
  const int m_first = blockIdx.x / n_tiles;          // first m-tile, then += ctas_per_n
  const int n0 = n_tile * BLOCK_N;
  const int num_kb = K / kBlockK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerThreads / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    // ===== TMA producer
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
      uint32_t it = 0;
      for (int mt = m_first; mt < m_tiles; mt += ctas_per_n) {
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
          mbar_expect_tx(&full_bar[s], Cfg::kABytes + Cfg::kBBytes);
          tma_load_2d(smem_a + s * Cfg::kABytes, &tmap_a, &full_bar[s], kb * kBlockK, mt * kBlockM);
          tma_load_2d(smem_b + s * Cfg::kBBytes, &tmap_b, &full_bar[s], kb * kBlockK, n0);
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg computes rows [64 wg, 64 wg + 64) of every tile
  const int wg = warp >> 2, t = threadIdx.x & 127, w = warp & 3;
  uint8_t* stg = smem_c + wg * (Cfg::kCBytes / 2);
  float acc[BLOCK_N / 2] = {};
  // accumulator acc[4j + e] holds row 16w + (lane >> 2) + 8 (e >> 1), column 8j + 2 (lane & 3) + (e & 1) of the
  // warpgroup's 64 x BLOCK_N block, whichever wgmma width produced it
  const int r0 = 16 * w + (lane >> 2);
  // statistics: thread t owns column pair p = t % (BLOCK_N / 2) over a 1 / kParts share of the 64 rows
  constexpr int kPairs = BLOCK_N / 2, kParts = 128 / kPairs, kRows = 64 / kParts;
  const int p = t % kPairs, rpart = t / kPairs;
  const int p_box = p >> 5, p_gran = (p & 31) >> 2, p_byte = (p & 3) * 4;
  float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;

  uint32_t it = 0;
  for (int mt = m_first; mt < m_tiles; mt += ctas_per_n) {
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const int s = it % kStages;
      mbar_wait(&full_bar[s], (it / kStages) & 1);
      const uint64_t adesc = gmma_desc(smem_a + s * Cfg::kABytes + wg * 64 * 128);
      const uint64_t bdesc = gmma_desc(smem_b + s * Cfg::kBBytes);
      fence_regs(acc);
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
#pragma unroll
        for (int h = 0; h < BLOCK_N / kInstN; ++h) {
          // B rows [h * kInstN, ...) start h * kInstN * 128 bytes further: +8 * kInstN in the (>>4) address field
          if constexpr (kInstN == 128) wgmma_n128<T>(acc + h * 64, adesc + 2 * k, bdesc + h * 8 * kInstN + 2 * k, (kb | k) != 0);
          else wgmma_n64<T>(acc + h * 32, adesc + 2 * k, bdesc + h * 8 * kInstN + 2 * k, (kb | k) != 0);
        }
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
      fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[s]);                   // this warp has finished reading the stage
    }

    // ---- epilogue: the staging tile may be refilled once the previous tile's TMA store has read it
    if (t == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    named_barrier(1 + wg, 128);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      // 16-byte granule g of row r sits at slot g ^ (r & 7) (the TMA SWIZZLE_128B layout): conflict-free here and below
      uint8_t* box = stg + (j >> 3) * 8192 + (lane & 3) * 4;
      const int g = j & 7;
      *reinterpret_cast<uint32_t*>(box + r0 * 128 + ((g ^ (r0 & 7)) << 4)) = Wire<T>::pack2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<uint32_t*>(box + (r0 + 8) * 128 + ((g ^ (r0 & 7)) << 4)) =
          Wire<T>::pack2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the TMA engine
    named_barrier(1 + wg, 128);
    if (t == 0) {
#pragma unroll
      for (int b = 0; b < kBoxes; ++b)
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                     ::"l"(&tmap_c), "r"(smem_u32(stg + b * 8192)), "r"(n0 + b * 64), "r"(mt * kBlockM + wg * 64) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    // The statistics are taken from the rounded 16-bit values - exactly what a separate BatchNorm pass over the stored
    // tensor would see.  Rows past M were zero-filled by TMA: they contribute 0 to both sums.
    const uint8_t* src = stg + p_box * 8192 + p_byte;
#pragma unroll 8
    for (int r = rpart * kRows; r < rpart * kRows + kRows; ++r) {
      const float2 f = Wire<T>::unpack2(*reinterpret_cast<const uint32_t*>(src + r * 128 + ((p_gran ^ (r & 7)) << 4)));
      s0 += f.x; q0 += f.x * f.x;
      s1 += f.y; q1 += f.y * f.y;
    }
  }
  if (t == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // outstanding output stores have landed
  // Fixed-order combine (no atomics, so the statistics are the same bits on every run): the per-thread sums go to shared
  // memory, then one thread per (sum, column) adds the warpgroups and row parts in order and writes this CTA's row of
  // the partials, part[m_first][0:N] (sums) / [N:2N] (sums of squares); combine_partials() adds the rows.
  float* my = smem_stats + wg * 4 * 128 + t;
  my[0] = s0; my[128] = s1; my[256] = q0; my[384] = q1;
  named_barrier(3, kConsumerThreads);
  for (int i = threadIdx.x; i < 2 * BLOCK_N; i += kConsumerThreads) {
    const int half = i >= BLOCK_N, col = i - half * BLOCK_N;
    const int pair = col >> 1, which = half * 2 + (col & 1);        // which: s0, s1, q0, q1
    float v = 0.f;
    for (int w2 = 0; w2 < 2; ++w2)
      for (int pt = 0; pt < kParts; ++pt) v += smem_stats[w2 * 4 * 128 + which * 128 + pt * kPairs + pair];
    part[(size_t)m_first * 2 * N + half * N + n0 + col] = v;
  }
}

// ------------------------------------------------------------------ data gradient with the BatchNorm backward apply on the A side
//   dx[M, K]  = A_k * dz + B_k * y + D_k   (dz = g, times the ReLU bit with RELU; rounded to T: bn_bwd_dx, the bits of bn_bwd_apply)
//   dIn[M, N] = dx x W                     (W = [K = C_out, N = C_in], the conv weight as stored: wgmma's transposed-B mode)
// The backward of a 1x1 conv -> BN pair otherwise writes dx in the BN apply pass and reads it back in the dgrad GEMM; here
// each stage's g tile is turned into the dx tile in place in shared memory before the wgmma reads it.  dx still reaches
// global memory once (the weight gradient needs it): the CTAs of n-tile 0 TMA-store the transformed tiles, the others
// re-read g / y from L2 like the forward kernel's A tiles.  wgmma group n-1 stays in flight while stage n is transformed.
constexpr int kCoefMaxK = 2048;            // A / B / D of up to 2048 channels in shared memory

template <int BLOCK_N> struct DgradCfg {
  static constexpr int kStages = BLOCK_N == 128 ? 3 : 4;
  static constexpr int kTileBytes = kBlockM * kBlockK * 2;            // one g or y tile
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;               // [BLOCK_N / 64] boxes of 64 k-rows x 64 n
  static constexpr int kCBytes = kBlockM * BLOCK_N * 2;
  static constexpr int kSmem = 1024 + kStages * (2 * kTileBytes + kBBytes) + kCBytes + 2 * kStages * 8 + 3 * kCoefMaxK * 4;
};

// K-major A as in gmma_desc; MN-major 128B-swizzled B: 64-wide n atoms 8 KB apart (LBO), 8-row k groups 1 KB apart (SBO)
__device__ __forceinline__ uint64_t gmma_desc_mn(const void* smem_tile) {
  const uint64_t addr = (uint64_t)(smem_u32(smem_tile) >> 4) & 0x3FFFull;
  return addr | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

#define PTD_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// as PTD_WGMMA_N64 / N128 with the transpose bit of B set (B read N-major)
#define PTD_WGMMA_T64(TY)                                                                                             \
  asm volatile(                                                                                                       \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                              \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " "                                                     \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                       \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 1;\n\t}" \
      : PTD_F8(0), PTD_F8(8), PTD_F8(16), PTD_F8(24)                                                                  \
      : "l"(adesc), "l"(bdesc), "r"(accumulate))
#define PTD_WGMMA_T128(TY)                                                                                            \
  asm volatile(                                                                                                       \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                              \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                    \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                       \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                              \
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                              \
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 1;\n\t}" \
      : PTD_F8(0), PTD_F8(8), PTD_F8(16), PTD_F8(24), PTD_F8(32), PTD_F8(40), PTD_F8(48), PTD_F8(56)                  \
      : "l"(adesc), "l"(bdesc), "r"(accumulate))
template <typename T> __device__ __forceinline__ void wgmma_t64(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
  if constexpr (std::is_same<T, __half>::value) PTD_WGMMA_T64("f16");
  else PTD_WGMMA_T64("bf16");
}
template <typename T> __device__ __forceinline__ void wgmma_t128(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
  if constexpr (std::is_same<T, __half>::value) PTD_WGMMA_T128("f16");
  else PTD_WGMMA_T128("bf16");
}
#undef PTD_WGMMA_T64
#undef PTD_WGMMA_T128
#undef PTD_F8

template <typename T, int BLOCK_N, bool RELU>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_bnbwd_dgrad_kernel(
    const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_y, const __grid_constant__ CUtensorMap tmap_w,
    const __grid_constant__ CUtensorMap tmap_dx, const __grid_constant__ CUtensorMap tmap_c, const uint8_t* __restrict__ mask,
    const float* __restrict__ saved, const float* __restrict__ gsum, const void* __restrict__ bnw, int wdt, void* __restrict__ dw,
    void* __restrict__ db, int M, int K, int m_tiles, int n_tiles, int ctas_per_n) {
  using Cfg = DgradCfg<BLOCK_N>;
  static_assert(BLOCK_N == 64 || BLOCK_N == 128, "one wgmma per k16 step");
  constexpr int kStages = Cfg::kStages;
  constexpr int kBoxes = BLOCK_N / 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smem_g = smem;                                            // [kStages][128 x 64] T: g, rewritten to dx in place
  uint8_t* smem_y = smem_g + kStages * Cfg::kTileBytes;              // [kStages][128 x 64] T: the BN input y
  uint8_t* smem_b = smem_y + kStages * Cfg::kTileBytes;              // [kStages][kBoxes][64 k x 64 n] T
  uint8_t* smem_c = smem_b + kStages * Cfg::kBBytes;                 // [2 warpgroups][kBoxes][64 x 64] T
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_c + Cfg::kCBytes);
  uint64_t* empty_bar = full_bar + kStages;
  float* coef = reinterpret_cast<float*>(empty_bar + kStages);       // [A | B | D][K]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x % n_tiles;
  const int m_first = blockIdx.x / n_tiles;
  const int n0 = n_tile * BLOCK_N;
  const int num_kb = K / kBlockK;
  const bool store_dx = n_tile == 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerThreads / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    // ===== TMA producer
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_g) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_y) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
      uint32_t it = 0;
      for (int mt = m_first; mt < m_tiles; mt += ctas_per_n) {
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
          mbar_expect_tx(&full_bar[s], 2 * Cfg::kTileBytes + Cfg::kBBytes);
          tma_load_2d(smem_g + s * Cfg::kTileBytes, &tmap_g, &full_bar[s], kb * kBlockK, mt * kBlockM);
          tma_load_2d(smem_y + s * Cfg::kTileBytes, &tmap_y, &full_bar[s], kb * kBlockK, mt * kBlockM);
#pragma unroll
          for (int b = 0; b < kBoxes; ++b)
            tma_load_2d(smem_b + s * Cfg::kBBytes + b * 8192, &tmap_w, &full_bar[s], n0 + b * 64, kb * kBlockK);
        }
      }
    }
    return;
  }

  // ===== consumers: the coefficients of all K channels once per CTA (block 0 also writes dgamma / dbeta, as bn_bwd_apply)
  const float inv_m = 1.f / (float)(int64_t)M;
  for (int c = threadIdx.x; c < K; c += kConsumerThreads) {
    const float sdz = gsum[c], sdzx = gsum[K + c];
    const BnBwdCoef q = bn_bwd_coef(ld_w(bnw, wdt, c), saved[c], saved[K + c], sdz, sdzx, inv_m, (c & 7) == 7);
    coef[c] = q.a; coef[K + c] = q.b; coef[2 * K + c] = q.d;
    if (blockIdx.x == 0) { st_w(dw, wdt, c, sdzx); st_w(db, wdt, c, sdz); }
  }
  named_barrier(3, kConsumerThreads);

  const int wg = warp >> 2, t = threadIdx.x & 127, w = warp & 3;
  uint8_t* stg = smem_c + wg * (Cfg::kCBytes / 2);
  float acc[BLOCK_N / 2] = {};
  const int r0 = 16 * w + (lane >> 2);
  // transform: thread t owns 16-byte granule j = t % 8 (channels 8j..8j+7 of the k-block) of rows t / 8 + 16 i of its warpgroup
  const int j = t & 7, rbase = wg * 64 + (t >> 3);
  const int mgroups = K / 8;

  uint32_t it = 0;
  for (int mt = m_first; mt < m_tiles; mt += ctas_per_n) {
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const int s = it % kStages;
      uint32_t bits[4] = {0u, 0u, 0u, 0u};
      if constexpr (RELU) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = mt * kBlockM + rbase + 16 * i;
          if (row < M) bits[i] = mask[(size_t)row * mgroups + kb * 8 + j];
        }
      }
      float ca[8], cb[8], cd[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int c = kb * kBlockK + j * 8 + e;
        ca[e] = coef[c]; cb[e] = coef[K + c]; cd[e] = coef[2 * K + c];
      }
      mbar_wait(&full_bar[s], (it / kStages) & 1);
      uint8_t* gt = smem_g + s * Cfg::kTileBytes;
      const uint8_t* yt = smem_y + s * Cfg::kTileBytes;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = rbase + 16 * i;
        const int off = r * 128 + ((j ^ (r & 7)) << 4);
        uint4 gv = *reinterpret_cast<const uint4*>(gt + off);
        const uint4 yv = *reinterpret_cast<const uint4*>(yt + off);
        uint32_t* gw = reinterpret_cast<uint32_t*>(&gv);
        const uint32_t* yw = reinterpret_cast<const uint32_t*>(&yv);
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const float2 g2 = Wire<T>::unpack2(gw[h]), y2 = Wire<T>::unpack2(yw[h]);
          float dz0 = g2.x, dz1 = g2.y;
          if constexpr (RELU) {
            dz0 = (bits[i] >> (2 * h)) & 1u ? dz0 : 0.f;
            dz1 = (bits[i] >> (2 * h + 1)) & 1u ? dz1 : 0.f;
          }
          gw[h] = Wire<T>::pack2(bn_bwd_dx(ca[2 * h], cb[2 * h], cd[2 * h], dz0, y2.x),
                                 bn_bwd_dx(ca[2 * h + 1], cb[2 * h + 1], cd[2 * h + 1], dz1, y2.y));
        }
        *reinterpret_cast<uint4*>(gt + off) = gv;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // dx tile -> visible to wgmma and the TMA store
      named_barrier(1 + wg, 128);
      if (store_dx && t == 0) {
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                     ::"l"(&tmap_dx), "r"(smem_u32(gt + wg * 64 * 128)), "r"(kb * kBlockK), "r"(mt * kBlockM + wg * 64) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      const uint64_t adesc = gmma_desc(gt + wg * 64 * 128);
      const uint64_t bdesc = gmma_desc_mn(smem_b + s * Cfg::kBBytes);
      fence_regs(acc);
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
        // one instruction covers the whole BLOCK_N; 16 k-rows of B are 2048 bytes further (+128 in the >>4 address field)
        if constexpr (BLOCK_N == 128) wgmma_t128<T>(acc, adesc + 2 * k, bdesc + 128 * k, (kb | k) != 0);
        else wgmma_t64<T>(acc, adesc + 2 * k, bdesc + 128 * k, (kb | k) != 0);
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");   // the previous stage's MMAs are done
      fence_regs(acc);
      if (kb > 0) {
        if (store_dx && t == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // its dx store has read it
        if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);
      }
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    fence_regs(acc);
    if (t == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // last dx store and previous staging store
    if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);

    // ---- epilogue: the staged TMA store of gemm_bnstats_kernel, without the statistics
    named_barrier(1 + wg, 128);
#pragma unroll
    for (int jj = 0; jj < BLOCK_N / 8; ++jj) {
      uint8_t* box = stg + (jj >> 3) * 8192 + (lane & 3) * 4;
      const int g = jj & 7;
      *reinterpret_cast<uint32_t*>(box + r0 * 128 + ((g ^ (r0 & 7)) << 4)) = Wire<T>::pack2(acc[4 * jj], acc[4 * jj + 1]);
      *reinterpret_cast<uint32_t*>(box + (r0 + 8) * 128 + ((g ^ (r0 & 7)) << 4)) = Wire<T>::pack2(acc[4 * jj + 2], acc[4 * jj + 3]);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    named_barrier(1 + wg, 128);
    if (t == 0) {
#pragma unroll
      for (int b = 0; b < kBoxes; ++b)
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                     ::"l"(&tmap_c), "r"(smem_u32(stg + b * 8192)), "r"(n0 + b * 64), "r"(mt * kBlockM + wg * 64) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (t == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    TORCH_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p, "cuTensorMapEncodeTiled not found");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// row-major [rows, cols] matrix of 16-bit elements (dtype: BFLOAT16 / FLOAT16), box = box_rows x 64 columns, 128-byte swizzle
static CUtensorMap make_map(CUtensorMapDataType dtype, const void* ptr, int64_t rows, int64_t cols, int box_rows,
                            CUtensorMapL2promotion promo) {
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&m, dtype, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: ", (int)r);
  return m;
}

template <typename T> struct TypeTag { using type = T; };

template <typename T, int BLOCK_N>
static void launch_gemm(const at::Tensor& a, const at::Tensor& b, at::Tensor& c, at::Tensor& gsum, int M, int N, int K, const SyncBN* sync) {
  constexpr int smem = GemmCfg<BLOCK_N>::kSmem;
  static bool configured[64] = {};                 // the attribute is per device (DataParallel drives several from one process)
  const int dev = a.get_device();
  if (!configured[dev & 63]) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(gemm_bnstats_kernel<T, BLOCK_N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured[dev & 63] = true;
  }
  constexpr CUtensorMapDataType dt = std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const CUtensorMap ma = make_map(dt, a.data_ptr(), M, K, kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  const CUtensorMap mb = make_map(dt, b.data_ptr(), N, K, BLOCK_N, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  const CUtensorMap mc = make_map(dt, c.data_ptr(), M, N, 64, CU_TENSOR_MAP_L2_PROMOTION_NONE);   // 64 x 64 store boxes
  const int m_tiles = (M + kBlockM - 1) / kBlockM, n_tiles = N / BLOCK_N;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int ctas_per_n = std::max(1, std::min(m_tiles, sms / n_tiles));
  const int grid = ctas_per_n * n_tiles;
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  at::Tensor part = at::empty({ctas_per_n, 2 * N}, gsum.options());
  gemm_bnstats_kernel<T, BLOCK_N><<<grid, kGemmThreads, smem, st>>>(ma, mb, mc, part.data_ptr<float>(), N, K, m_tiles, n_tiles, ctas_per_n);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  finish_sums(part.data_ptr<float>(), ctas_per_n, N, M, gsum.data_ptr<float>(), sync, st);
}

template <typename T>
static void launch_gemm_for(const at::Tensor& a, const at::Tensor& b, at::Tensor& c, at::Tensor& gsum, int M, int N, int K, const SyncBN* sync) {
  static const int max_bn = getenv("PTD_GEMM_BLOCK_N") ? atoi(getenv("PTD_GEMM_BLOCK_N")) : 256;
  if (N % 256 == 0 && max_bn >= 256) launch_gemm<T, 256>(a, b, c, gsum, M, N, K, sync);
  else if (N % 128 == 0 && max_bn >= 128) launch_gemm<T, 128>(a, b, c, gsum, M, N, K, sync);
  else launch_gemm<T, 64>(a, b, c, gsum, M, N, K, sync);
}

// x: [B, K, H, W] channels_last bf16 or fp16; weight: [N, K, 1, 1] of x's dtype (any dense layout); gsum: zeroed float[2N].
// returns y [B, N, H, W] channels_last in x's dtype; gsum accumulates the per-channel sum and sum of squares of y.
// sync: gsum is a synchronised work slice (host.h kSyncWork) and the epilogue partials go through the cross-rank exchange.
at::Tensor conv1x1_bnstats(const at::Tensor& x, const at::Tensor& weight, at::Tensor gsum, const SyncBN* sync) {
  const bool is16 = x.scalar_type() == at::kBFloat16 || x.scalar_type() == at::kHalf;
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && is16 && x.is_contiguous(at::MemoryFormat::ChannelsLast),
              "conv1x1_bnstats: x must be a channels_last bf16 or fp16 CUDA tensor");
  TORCH_CHECK(weight.dim() == 4 && weight.size(2) == 1 && weight.size(3) == 1 && weight.scalar_type() == x.scalar_type(),
              "conv1x1_bnstats: weight must be [N, K, 1, 1] with x's dtype (both bf16 or both fp16)");
  const int64_t M64 = x.size(0) * x.size(2) * x.size(3);
  const int K = (int)x.size(1), N = (int)weight.size(0);
  TORCH_CHECK(weight.size(1) == K && K % kBlockK == 0 && N % 64 == 0 && M64 < (int64_t)1 << 31, "conv1x1_bnstats: unsupported shape");
  check_work(gsum, N, sync);
  TORCH_CHECK((reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0, "x must be 16-byte aligned");
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor w2 = weight.reshape({N, K}).contiguous();       // [N, K] K-major (a view for both NCHW and NHWC 1x1 weights)
  at::Tensor y = at::empty({x.size(0), N, x.size(2), x.size(3)}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  const int M = (int)M64;
  if (x.scalar_type() == at::kHalf) launch_gemm_for<__half>(x, w2, y, gsum, M, N, K, sync);
  else launch_gemm_for<__nv_bfloat16>(x, w2, y, gsum, M, N, K, sync);
  return y;
}

template <typename T, int BLOCK_N, bool RELU>
static void launch_dgrad(const at::Tensor& g, const at::Tensor& y, const uint8_t* mask, const at::Tensor& saved, const float* sums,
                         const at::Tensor& bnw, int wdt, at::Tensor& dw, at::Tensor& db, const at::Tensor& w2, at::Tensor& dx, at::Tensor& din,
                         int M, int N, int K) {
  constexpr int smem = DgradCfg<BLOCK_N>::kSmem;
  auto kernel = gemm_bnbwd_dgrad_kernel<T, BLOCK_N, RELU>;
  static bool configured[64] = {};
  const int dev = g.get_device();
  if (!configured[dev & 63]) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured[dev & 63] = true;
  }
  constexpr CUtensorMapDataType dt = std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const CUtensorMap mg = make_map(dt, g.data_ptr(), M, K, kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  const CUtensorMap my = make_map(dt, y.data_ptr(), M, K, kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  const CUtensorMap mw = make_map(dt, w2.data_ptr(), K, N, 64, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);    // [K, N]: 64 k-rows x 64 n
  const CUtensorMap mdx = make_map(dt, dx.data_ptr(), M, K, 64, CU_TENSOR_MAP_L2_PROMOTION_NONE);
  const CUtensorMap mc = make_map(dt, din.data_ptr(), M, N, 64, CU_TENSOR_MAP_L2_PROMOTION_NONE);
  const int m_tiles = (M + kBlockM - 1) / kBlockM, n_tiles = N / BLOCK_N;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int ctas_per_n = std::max(1, std::min(m_tiles, sms / n_tiles));
  kernel<<<ctas_per_n * n_tiles, kGemmThreads, smem, at::cuda::getCurrentCUDAStream()>>>(
      mg, my, mw, mdx, mc, mask, saved.data_ptr<float>(), sums, bnw.data_ptr(), wdt, dw.data_ptr(), db.data_ptr(), M, K, m_tiles, n_tiles,
      ctas_per_n);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void conv1x1_dgrad_bn(const at::Tensor& g, const at::Tensor& y, const uint8_t* mask, const at::Tensor& saved, const float* sums,
                      const at::Tensor& bnw, int wdt, at::Tensor& dw, at::Tensor& db, const at::Tensor& conv_w, at::Tensor& dx, at::Tensor& din) {
  const int64_t M64 = y.size(0) * y.size(2) * y.size(3);
  const int K = (int)y.size(1), N = (int)conv_w.size(1);
  TORCH_CHECK(conv_w.dim() == 4 && conv_w.size(0) == K && conv_w.size(2) == 1 && conv_w.size(3) == 1 && conv_w.scalar_type() == y.scalar_type(),
              "conv1x1_bn_backward: the conv weight must be [C_out, C_in, 1, 1] with the activations' dtype");
  TORCH_CHECK(K % kBlockK == 0 && K <= kCoefMaxK && N % 64 == 0 && M64 < (int64_t)1 << 31, "conv1x1_bn_backward: unsupported shape");
  at::Tensor w2 = conv_w.reshape({K, N});
  TORCH_CHECK(w2.is_contiguous(), "conv1x1_bn_backward: the conv weight must be dense [C_out, C_in]");
  const int M = (int)M64;
  auto run = [&](auto tag) {
    using T = typename decltype(tag)::type;
    if (N % 128 == 0) {
      if (mask) launch_dgrad<T, 128, true>(g, y, mask, saved, sums, bnw, wdt, dw, db, w2, dx, din, M, N, K);
      else launch_dgrad<T, 128, false>(g, y, mask, saved, sums, bnw, wdt, dw, db, w2, dx, din, M, N, K);
    } else {
      if (mask) launch_dgrad<T, 64, true>(g, y, mask, saved, sums, bnw, wdt, dw, db, w2, dx, din, M, N, K);
      else launch_dgrad<T, 64, false>(g, y, mask, saved, sums, bnw, wdt, dw, db, w2, dx, din, M, N, K);
    }
  };
  if (y.scalar_type() == at::kHalf) run(TypeTag<__half>{});
  else run(TypeTag<__nv_bfloat16>{});
}

}  // namespace ptd
