// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fences, shared-memory
// descriptors, accumulator fragments). Hand-written; the descriptor layout follows the PTX ISA "matrix descriptor"
// table of wgmma.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace fvit {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (error surfaces on the host) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // (try_wait suspends in hardware for a bounded time per poll; after 2^16 polls the loop backs off so that a long
  // but legitimate wait -- profiler replay, SM time-slicing next to a collective -- cannot reach the bound: 2^24
  // polls with back-off are many seconds)
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 16)) {
      __nanosleep(200);
      if (spins > (1u << 24)) __trap();
    }
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (one warpgroup = 128 threads)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// Shared-memory matrix descriptor (64 bit):
//  [0,14) start address >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4
//  [49,52) base offset | [62,64) layout (0 none, 1 128B, 2 64B, 3 32B swizzle)
// The base offset stays 0: the swizzle phase of a row comes from the address bits themselves, so a K-major SW128
// matrix may start at any 128-byte row of a buffer that TMA wrote from a 1024-byte boundary (measured on H100:
// setting the field to (start >> 7) & 7 for such a start shifts the phase twice and gives wrong products).
// K-major SW128: SBO = 1024 (8 rows x 128 B), LBO unused; MN-major SW128: LBO = next 64-wide MN atom, SBO = next
// 8 K rows. The SWZ_* values below are the layout field shifted to bit 61.
enum : uint32_t { SWZ_NONE = 0, SWZ_128B = 2, SWZ_64B = 4, SWZ_32B = 6 };

__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes, uint32_t swizzle) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(swizzle & 7) << 61;
  return d;
}

// Accumulator fragment of an m64nN wgmma <-> rows [0, 64) of a row-major fp32 tile in shared memory: thread t of
// the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8), columns 8j + 2*(t%4) (+1).
template <int N>
__device__ __forceinline__ void acc_store(float* buf, int ld, const float (&d)[N / 2]) {
  const int t = threadIdx.x & 127;
  float* r0 = buf + ((t >> 5) * 16 + ((t & 31) >> 2)) * ld + 2 * (t & 3);
  float* r1 = r0 + 8 * ld;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(r1 + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
template <int N>
__device__ __forceinline__ void acc_load(const float* buf, int ld, float (&d)[N / 2]) {
  const int t = threadIdx.x & 127;
  const float* r0 = buf + ((t >> 5) * 16 + ((t & 31) >> 2)) * ld + 2 * (t & 3);
  const float* r1 = r0 + 8 * ld;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const float2 a = *reinterpret_cast<const float2*>(r0 + 8 * j);
    const float2 b = *reinterpret_cast<const float2*>(r1 + 8 * j);
    d[4 * j] = a.x, d[4 * j + 1] = a.y, d[4 * j + 2] = b.x, d[4 * j + 3] = b.y;
  }
}

// D[128 x N] (+)= sum_k A_k B_k (fp16 operands, fp32 accumulate), computed by the calling warpgroup as two m64
// halves and left in buf (row-major fp32, leading dimension ld), K = 16 * KSTEPS. adesc(h, k) is the descriptor of
// rows [64h, 64h + 64) of A for K step k, bdesc(k) that of B. With accumulate, buf holds the previous D.
// Every thread of the warpgroup calls this; the caller synchronises the warpgroup before others read buf.
template <int N, int TA, int TB, int KSTEPS, class FA, class FB>
__device__ __forceinline__ void wg_mma_128(float* buf, int ld, FA adesc, FB bdesc, bool accumulate) {
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    float d[N / 2];
    if (accumulate) {
      acc_load<N>(buf + h * 64 * ld, ld, d);
    } else {
#pragma unroll
      for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) Wgmma<N, TA, TB, 0>::mma(d, adesc(h, k), bdesc(k), 1u);
    wgmma_commit();
    wgmma_wait0();
    acc_store<N>(buf + h * 64 * ld, ld, d);
  }
}

// 32 / 16 consecutive fp32 values of an accumulator row (row-per-thread reads of a tile left by wg_mma_128)
__device__ __forceinline__ void ld_row32(const float* src, uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    r[4 * i] = __float_as_uint(v.x), r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z), r[4 * i + 3] = __float_as_uint(v.w);
  }
}
__device__ __forceinline__ void ld_row16(const float* src, uint32_t (&r)[16]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    r[4 * i] = __float_as_uint(v.x), r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z), r[4 * i + 3] = __float_as_uint(v.w);
  }
}
// Per-thread register budget of the calling warpgroup (every warp of the group executes it): dec returns registers
// to the CTA's pool, inc waits until the pool has them.
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace fvit
