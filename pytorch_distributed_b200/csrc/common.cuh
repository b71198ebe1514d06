// Device-side building blocks shared by every sm_90a kernel in this extension:
//  * 16-byte vector load/store with explicit cache policy
//  * NVLS multimem.ld_reduce / multimem.st wrappers (in-switch reduction / multicast over NVSwitch)
//  * system-scope signal flags (monotonic sequence numbers, no reset) + block barrier across GPUs
//  * bounded spin-waits: a peer that never arrives traps the kernel instead of hanging the box
//
// Reference parity: these replace what the reference reaches through NCCL
// (/root/reference/distributed.py:105-109,256 all_reduce + barrier) with peer-memory code.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "comm_types.h"

namespace ptd {

__device__ __forceinline__ SignalPad* pad_of(const CommCtx& c, int r) {
  return reinterpret_cast<SignalPad*>(c.base[r]);
}

// ------------------------------------------------------------------ scalar sys-scope ops
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Spin until *flag has reached `want` (monotonic counters, wrap-safe compare).
__device__ __forceinline__ void wait_flag(const CommCtx& c, const uint32_t* flag, uint32_t want) {
  if ((int32_t)(ld_acquire_sys(flag) - want) >= 0) return;
  const uint64_t t0 = globaltimer_ns();
  const uint64_t budget = (uint64_t)c.timeout_ms * 1000000ull;
  while ((int32_t)(ld_acquire_sys(flag) - want) < 0) {
    __nanosleep(40);
    if (budget && globaltimer_ns() - t0 > budget) {
      if (c.status) { *reinterpret_cast<volatile uint32_t*>(c.status) = 0xDEAD0000u | (uint32_t)c.rank; __threadfence_system(); }
      __trap();
    }
  }
}

// Cross-GPU barrier between the CTAs with the same blockIdx.x on every rank.
// `seq` is the caller's register copy of this (channel, block) sequence number.
// Semantics: release of everything this CTA wrote before, acquire of everything the peer CTAs wrote before.
__device__ __forceinline__ void block_barrier(const CommCtx& c, uint32_t& seq) {
  __syncthreads();
  ++seq;
  if (threadIdx.x < (unsigned)c.world) {
    const int peer = threadIdx.x;
    st_release_sys(&pad_of(c, peer)->flags[c.channel][blockIdx.x][c.rank], seq);
    wait_flag(c, &pad_of(c, c.rank)->flags[c.channel][blockIdx.x][peer], seq);
  }
  __syncthreads();
}

__device__ __forceinline__ uint32_t load_seq(const CommCtx& c) {
  return c.seq[c.channel * kMaxBlocks + blockIdx.x];
}
__device__ __forceinline__ void store_seq(const CommCtx& c, uint32_t seq) {
  if (threadIdx.x == 0) c.seq[c.channel * kMaxBlocks + blockIdx.x] = seq;
}

// ------------------------------------------------------------------ 16-byte vector memory ops
struct __align__(16) V4 { uint32_t x, y, z, w; };

__device__ __forceinline__ V4 ld_stream(const void* p) {  // read-once data: keep out of L1
  V4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ V4 ld_sys(const void* p) {  // data another GPU may have just written
  V4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_v4(void* p, const V4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_sys(void* p, const V4& v) {  // store that a peer will read
  asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------ NVLS multimem
// ld_reduce: the switch fetches the 16 bytes at this multicast address from EVERY bound GPU,
// adds them (fp32 accumulation for 16-bit types) and returns one result.
template <typename T> struct Multimem;
template <> struct Multimem<__nv_bfloat16> {
  static __device__ __forceinline__ V4 ld_reduce(const void* mc) {
    V4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
  }
};
template <> struct Multimem<__half> {
  static __device__ __forceinline__ V4 ld_reduce(const void* mc) {
    V4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
  }
};
template <> struct Multimem<float> {
  static __device__ __forceinline__ V4 ld_reduce(const void* mc) {
    V4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
  }
};
// st: one store, replicated by the switch into every bound GPU's copy.
__device__ __forceinline__ void multimem_st(void* mc, const V4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------ dtype helpers (8 elements <-> registers)
template <typename T> struct Wire;  // T in {bf16, half, float}: how 8 consecutive elements are held
template <> struct Wire<__nv_bfloat16> {
  static constexpr int kVecElems = 8;  // per 16-byte vector
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  }
};
template <> struct Wire<__half> {
  static constexpr int kVecElems = 8;
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
};

// Eight fp32 values <-> storage of type T at `p` (p 16-byte aligned for 16-bit T, 32-byte for fp32).
template <typename T> __device__ __forceinline__ void load8(const T* p, float (&f)[8], bool sys = false);
template <> __device__ __forceinline__ void load8<float>(const float* p, float (&f)[8], bool sys) {
  V4 a = sys ? ld_sys(p) : ld_stream(p), b = sys ? ld_sys(p + 4) : ld_stream(p + 4);
  f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
  f[4] = __uint_as_float(b.x); f[5] = __uint_as_float(b.y); f[6] = __uint_as_float(b.z); f[7] = __uint_as_float(b.w);
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&f)[8], bool sys) {
  V4 a = sys ? ld_sys(p) : ld_stream(p);
  float2 t;
  t = Wire<__nv_bfloat16>::unpack2(a.x); f[0] = t.x; f[1] = t.y;
  t = Wire<__nv_bfloat16>::unpack2(a.y); f[2] = t.x; f[3] = t.y;
  t = Wire<__nv_bfloat16>::unpack2(a.z); f[4] = t.x; f[5] = t.y;
  t = Wire<__nv_bfloat16>::unpack2(a.w); f[6] = t.x; f[7] = t.y;
}
template <> __device__ __forceinline__ void load8<__half>(const __half* p, float (&f)[8], bool sys) {
  V4 a = sys ? ld_sys(p) : ld_stream(p);
  float2 t;
  t = Wire<__half>::unpack2(a.x); f[0] = t.x; f[1] = t.y;
  t = Wire<__half>::unpack2(a.y); f[2] = t.x; f[3] = t.y;
  t = Wire<__half>::unpack2(a.z); f[4] = t.x; f[5] = t.y;
  t = Wire<__half>::unpack2(a.w); f[6] = t.x; f[7] = t.y;
}
template <typename T> __device__ __forceinline__ void store8(T* p, const float (&f)[8], bool sys = false);
template <> __device__ __forceinline__ void store8<float>(float* p, const float (&f)[8], bool sys) {
  V4 a{__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3])};
  V4 b{__float_as_uint(f[4]), __float_as_uint(f[5]), __float_as_uint(f[6]), __float_as_uint(f[7])};
  if (sys) { st_sys(p, a); st_sys(p + 4, b); } else { st_v4(p, a); st_v4(p + 4, b); }
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&f)[8], bool sys) {
  using W = Wire<__nv_bfloat16>;
  V4 a{W::pack2(f[0], f[1]), W::pack2(f[2], f[3]), W::pack2(f[4], f[5]), W::pack2(f[6], f[7])};
  if (sys) st_sys(p, a); else st_v4(p, a);
}
template <> __device__ __forceinline__ void store8<__half>(__half* p, const float (&f)[8], bool sys) {
  using W = Wire<__half>;
  V4 a{W::pack2(f[0], f[1]), W::pack2(f[2], f[3]), W::pack2(f[4], f[5]), W::pack2(f[6], f[7])};
  if (sys) st_sys(p, a); else st_v4(p, a);
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

}  // namespace ptd
