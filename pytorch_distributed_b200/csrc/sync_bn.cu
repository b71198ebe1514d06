// Synchronised BatchNorm: the cross-rank exchange of the per-channel sums (sm_90a).
//
// One kernel replaces combine_partials() when a layer is synchronised.  Per call it
//   1. combines this rank's per-CTA partial rows in combine_partials' order (bn_combine.cuh), so the
//      local [2C] sums are the bits the unsynchronised op computes, and adds them to work[0:2C] as that op does;
//   2. publishes them, followed by the local row count (two 32-bit halves, exact), into slot `rank` of every peer's
//      exchange area as 8-byte LL words {payload, seq} (one relaxed .sys vector store: value and flag land together);
//   3. reads slots 0..W-1 of its own area in rank order, spinning on the sequence, and adds them in fp32 from 0 (the
//      counts as 64-bit integers), so every rank holds the same global sums and count, bit for bit;
//   4. writes work[2C:4C] = the global sums and work[4C:4C+2] = the global count, where the apply kernels read them.
//
// Work split: CTA b owns the 32-word tiles b, b + grid, ... of the 2C + 2 words on every rank, and the grid depends on C
// only, so CTA b of one rank depends only on CTA b of the others; at most kMaxBlocks CTAs, all co-resident.
//
// Buffer reuse: call `seq` writes parity seq & 1.  The previous writes of that parity are from call seq - 2.  A rank
// enters call seq only after its call seq - 1 read a word every peer published in call seq - 1, and a peer publishes
// call seq - 1 only after its call seq - 2 kernel (including all its reads) has finished, in stream order.  So no word a
// peer may still read is overwritten - the argument of ll_allreduce_kernel.  A stale word carries a smaller sequence, and
// the reader waits for equality.
#include <ATen/cuda/CUDAContext.h>
#include <torch/extension.h>

#include "bn_combine.cuh"
#include "common.cuh"
#include "host.h"

namespace ptd {

__global__ void __launch_bounds__(1024) sync_bn_kernel(const __grid_constant__ CommCtx c, const float* __restrict__ part, int nblocks,
                                                       int C, int64_t rows, float* __restrict__ work, int64_t xoff,
                                                       uint32_t* __restrict__ calls) {
  __shared__ float sm[32][33];
  __shared__ uint32_t word[kMaxWorld][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n = 2 * C, nw = n + 2;
  const uint32_t seq = calls[blockIdx.x] + 1;
  const int par = seq & 1;
  // [par][src][word] uint2 words; my slot in every peer's area starts at slot_off
  const int64_t area_off = xoff + (int64_t)par * kMaxWorld * kSyncBnSlotWords * 8;
  const int64_t slot_off = area_off + (int64_t)c.rank * kSyncBnSlotWords * 8;
  const uint64_t t0 = globaltimer_ns();
  for (int tile = blockIdx.x; tile * 32 < nw; tile += gridDim.x) {
    const int i = tile * 32 + tx;
    sm[ty][tx] = combine_slice(part, nblocks, n, i, ty);
    __syncthreads();
    if (ty == 0) {
      uint32_t w = 0;
      if (i < n) {
        const float l = work[i] + combine_fold(sm, tx);   // combine_partials: gsum[i] += t
        work[i] = l;
        w = __float_as_uint(l);
      } else if (i == n) {
        w = (uint32_t)(uint64_t)rows;
      } else if (i == n + 1) {
        w = (uint32_t)((uint64_t)rows >> 32);
      }
      word[0][tx] = w;
    }
    __syncthreads();
    const uint32_t mine = word[0][tx];
    __syncthreads();
    if (ty < c.world && i < nw) {
      // publish: thread (ty, tx) stores word i into peer ty's area, then reads source ty's word i from its own
      uint2* dst = reinterpret_cast<uint2*>(c.base[ty] + slot_off) + i;
      asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1,%2};" ::"l"(dst), "r"(mine), "r"(seq) : "memory");
      const uint2* src = reinterpret_cast<const uint2*>(c.base[c.rank] + area_off + (int64_t)ty * kSyncBnSlotWords * 8) + i;
      uint2 v;
      while (true) {
        asm volatile("ld.relaxed.sys.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(src) : "memory");
        if (v.y == seq) break;
        if (c.timeout_ms && globaltimer_ns() - t0 > (uint64_t)c.timeout_ms * 1000000ull) {
          if (c.status) { *reinterpret_cast<volatile uint32_t*>(c.status) = 0xDEAD3000u | (uint32_t)c.rank; __threadfence_system(); }
          __trap();
        }
      }
      word[ty][tx] = v.x;
    }
    __syncthreads();
    if (ty == 0) {
      if (i < n) {
        float g = 0.f;
        for (int k = 0; k < c.world; ++k) g += __uint_as_float(word[k][tx]);
        work[n + i] = g;
      } else if (i == n) {            // 2C is a multiple of 16: both count halves sit in this tile
        uint64_t cnt = 0;
        for (int k = 0; k < c.world; ++k) cnt += (uint64_t)word[k][tx] | ((uint64_t)word[k][tx + 1] << 32);
        *reinterpret_cast<int64_t*>(work + 2 * n) = (int64_t)cnt;
      }
    }
    __syncthreads();                  // sm / word are refilled by the next tile
  }
  if (threadIdx.x == 0) {
    calls[blockIdx.x] = seq;
    if (blockIdx.x == 0)              // counters of CTAs this grid does not have: every entry stays at the same call count
      for (int b = gridDim.x; b < kMaxBlocks; ++b) calls[b] = seq;
  }
}

void sync_bn_exchange(const float* part, int nblocks, int C, int64_t rows, float* work, const SyncBN& s, cudaStream_t st) {
  TORCH_CHECK(C > 0 && C % 8 == 0 && C <= kSyncBnMaxC, "synchronised BatchNorm needs C % 8 == 0 and C <= ", kSyncBnMaxC, " (got ", C, ")");
  TORCH_CHECK(s.ctx.world >= 1 && s.ctx.world <= kMaxWorld && s.calls != nullptr, "invalid synchronised BatchNorm handle");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(work) & 7) == 0, "synchronised BatchNorm work slice must be 8-byte aligned");
  const int tiles = (2 * C + 2 + 31) / 32;
  const int grid = std::min(tiles, kMaxBlocks);
  sync_bn_kernel<<<grid, 1024, 0, st>>>(s.ctx, part, nblocks, C, rows, work, s.xoff, s.calls);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void check_work(const at::Tensor& work, int64_t C, const SyncBN* sync) {
  TORCH_CHECK(work.defined() && work.scalar_type() == at::kFloat && work.is_contiguous() && work.numel() >= 2 * C, "work buffer too small");
  TORCH_CHECK(!sync || work.numel() >= kSyncWork(C), "synchronised BatchNorm needs a work slice of ", kSyncWork(C), " floats");
}

float* work_sums(float* work, int C, const SyncBN* sync) { return sync ? work + 2 * C : work; }

float* finish_sums(const float* part, int nblocks, int C, int64_t rows, float* work, const SyncBN* sync, cudaStream_t st) {
  if (sync) sync_bn_exchange(part, nblocks, C, rows, work, *sync, st);
  else combine_partials(part, nblocks, 2 * C, work, st);
  return work_sums(work, C, sync);
}

}  // namespace ptd
