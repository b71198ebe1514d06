// Plain-C++ types shared by host code and kernels (no device code here: symm.cpp/bindings.cpp include this).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptd {

constexpr int kMaxWorld = 16;
constexpr int kMaxBlocks = 64;     // max CTAs of a cross-GPU kernel (all must be co-resident)
constexpr int kMaxChannels = 16;   // independent signal channels (one per stream / engine)
constexpr int kMaxPtrs = 384;      // tensors per bucket launch (pointer pack lives in kernel params)

// Layout of the per-rank signal pad (lives at the start of the symmetric arena).
//   flags[channel][block][src_rank]  : written by peer `src_rank`, read by the owner
//   inbox (LL protocol, metrics)     : see metrics kernels
struct SignalPad {
  uint32_t flags[kMaxChannels][kMaxBlocks][kMaxWorld];
  // low-latency inbox: [parity][src_rank][slot] of {payload bits, sequence}
  uint2 inbox[2][kMaxWorld][8];
};

// Everything a cross-GPU kernel needs to address its peers.  Passed by value.
struct CommCtx {
  int rank;
  int world;
  int channel;
  uint32_t timeout_ms;          // 0 = wait forever
  char* base[kMaxWorld];        // per-rank arena base (base[rank] is local); SignalPad sits at offset 0
  char* mc_base;                // multicast alias of the same arena (nullptr => no NVLS)
  uint32_t* seq;                // local (non-symmetric) [kMaxChannels][kMaxBlocks] sequence counters
  uint32_t* status;             // host-mapped status word: non-zero => a wait timed out
};

enum DType : int { kF32 = 0, kBF16 = 1, kF16 = 2 };

// Synchronised BatchNorm (sync_bn.cu).  Exchange area, at the same arena offset on every rank:
//   uint2 words[2 parities][kMaxWorld source ranks][kSyncBnSlotWords] of {payload bits, sequence}
// A slot carries one rank's [2C] local sums followed by its row count as two 32-bit halves.
constexpr int kSyncBnMaxC = 8192;
constexpr int kSyncBnSlotWords = 2 * kSyncBnMaxC + 2;
constexpr int64_t kSyncBnAreaBytes = (int64_t)2 * kMaxWorld * kSyncBnSlotWords * 8;

// What a synchronised BatchNorm call needs to reach its peers.  `calls`: this handle's local [kMaxBlocks] call counters
// (all entries advance together, one per exchange).
struct SyncBN {
  CommCtx ctx;
  int64_t xoff;        // arena byte offset of the exchange area
  uint32_t* calls;
};

}  // namespace ptd
