// Thin inline-PTX wrappers for the sm_90a features the engine uses:
// mbarrier, TMA (tiled + im2col), wgmma ordering (the MMA instructions themselves are in wgmma.cuh).
// Everything here is a 1:1 spelling of a PTX instruction; no policy lives in this file.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

#include "wgmma.cuh"

namespace sfb {

#ifndef SFB_WATCHDOG_SPINS
// A hung mbarrier wait traps instead of wedging the GPU (a wedged box is a lost lease).
#define SFB_WATCHDOG_SPINS (1u << 26)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      " .reg .pred p;\n"
      " elect.sync _|p, 0xffffffff;\n"
      " selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      " .reg .pred p;\n"
      " mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      " selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > SFB_WATCHDOG_SPINS) __trap();
  }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}
// 2-D tiled load: box -> smem, completes on mbarrier with the box byte count.
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 5-D im2col load over an NDHWC tensor (dims given to the map as C,W,H,D,N).
// (c,w,h,d,n) is the channel offset and the input coordinate of filter tap 0 for the first pixel of the
// column; (ow,oh,od) is the filter-tap offset (tap * dilation). The unit walks pixelsPerColumn output pixels
// W-fastest inside the map's bounding box; out-of-tensor pixels are zero-filled.
__device__ __forceinline__ void tma_load_im2col_5d(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c,
                                                   int32_t w, int32_t h, int32_t d, int32_t n, uint16_t ow,
                                                   uint16_t oh, uint16_t od) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2], {%8, %9, %10};"
      ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "h"(ow),
        "h"(oh), "h"(od)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma
// Ordering of register accesses against the asynchronous warpgroup MMAs (all 128 threads of the warpgroup execute these).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor (sm_90 format): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) |
// layout type [62,64) (0 none, 1 = 128B swizzle, 2 = 64B, 3 = 32B).  The callers pass the layout as 0 / 2 / 4 / 6,
// i.e. the same field shifted one bit down ([61,64)).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t layout_type) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout_type & 6) << 61;
  return d;
}

// ----------------------------------------------------------------------------- accumulator tile hand-off
// The MMA warpgroups keep a [64 x n] fp32 accumulator in registers (wgmma fragment layout, wgmma.cuh); the epilogue warps
// read it from a row-major shared-memory tile of `pitch` floats per row.  acc_store writes the calling warpgroup's
// fragment to rows [0, 64) of `tile`; every thread of the warpgroup calls it.
template <int MAXN>
__device__ __forceinline__ void acc_store(const float* d, int n, float* tile, int pitch) {
  const int t = threadIdx.x & 127;
  const int r = (t >> 5) * 16 + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < MAXN / 8; ++j) {
    if (8 * j < n) {
      *reinterpret_cast<float2*>(tile + r * pitch + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2*>(tile + (r + 8) * pitch + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  }
}
// 16 consecutive columns of one row of an accumulator tile (16-byte aligned).
__device__ __forceinline__ void acc_ld_x16(const float* src, uint32_t (&v)[16]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 x = reinterpret_cast<const float4*>(src)[j];
    v[4 * j] = __float_as_uint(x.x);
    v[4 * j + 1] = __float_as_uint(x.y);
    v[4 * j + 2] = __float_as_uint(x.z);
    v[4 * j + 3] = __float_as_uint(x.w);
  }
}

// named barrier among a subset of warps
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// signal a named barrier without waiting on it (nthreads counts the arriving and the waiting threads)
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------- register reallocation
// Lower / raise the calling warpgroup's per-thread register limit (all 128 threads execute it).  N is a multiple of 8
// in [24, 256]; a raise waits until other warpgroups of the CTA have released enough registers.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

}  // namespace sfb
