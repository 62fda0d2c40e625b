// Split-bf16 operand planes: an fp32 value v is stored as hi = bf16(v) and lo = bf16(v - hi), and read back as hi + lo.
// The lo plane may be null (single-plane operands).  Scalar helpers address element i; the vector helpers move 8
// (16-byte) or 4 (8-byte) consecutive elements.
#pragma once
#include <cstdint>
#include <cuda_bf16.h>

namespace sfb {

struct alignas(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void put_split(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t i, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}
__device__ __forceinline__ float get_split(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t i) {
  float v = __bfloat162float(hi[i]);
  if (lo) v += __bfloat162float(lo[i]);
  return v;
}

// split 8 fp32 values into hi = bf16(x), lo = bf16(x - hi) and store both planes (lo may be null)
__device__ __forceinline__ void store_split8(__nv_bfloat16* hi, __nv_bfloat16* lo, const float (&x)[8]) {
  bf16x8 h, l;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat16 h0 = __float2bfloat16_rn(x[2 * i]), h1 = __float2bfloat16_rn(x[2 * i + 1]);
    h.v[i] = __halves2bfloat162(h0, h1);
    l.v[i] = __halves2bfloat162(__float2bfloat16_rn(x[2 * i] - __bfloat162float(h0)),
                                __float2bfloat16_rn(x[2 * i + 1] - __bfloat162float(h1)));
  }
  *reinterpret_cast<bf16x8*>(hi) = h;
  if (lo) *reinterpret_cast<bf16x8*>(lo) = l;
}
__device__ __forceinline__ void load_planes8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, float (&x)[8]) {
  const bf16x8 h = *reinterpret_cast<const bf16x8*>(hi);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[2 * i] = __bfloat162float(__low2bfloat16(h.v[i]));
    x[2 * i + 1] = __bfloat162float(__high2bfloat16(h.v[i]));
  }
  if (lo) {
    const bf16x8 l = *reinterpret_cast<const bf16x8*>(lo);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      x[2 * i] += __bfloat162float(__low2bfloat16(l.v[i]));
      x[2 * i + 1] += __bfloat162float(__high2bfloat16(l.v[i]));
    }
  }
}

__device__ __forceinline__ uint32_t pack_bf2(float a, float b) {
  const __nv_bfloat162 t = __halves2bfloat162(__float2bfloat16_rn(a), __float2bfloat16_rn(b));
  return *reinterpret_cast<const uint32_t*>(&t);
}
// the 4 values of v split into planes at element offset off
__device__ __forceinline__ void store_planes4(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t off, float4 v) {
  const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z),
                      h3 = __float2bfloat16_rn(v.w);
  uint2 h;
  {
    const __nv_bfloat162 a = __halves2bfloat162(h0, h1), b = __halves2bfloat162(h2, h3);
    h.x = *reinterpret_cast<const uint32_t*>(&a);
    h.y = *reinterpret_cast<const uint32_t*>(&b);
  }
  *reinterpret_cast<uint2*>(hi + off) = h;
  if (lo) {
    uint2 l;
    l.x = pack_bf2(v.x - __bfloat162float(h0), v.y - __bfloat162float(h1));
    l.y = pack_bf2(v.z - __bfloat162float(h2), v.w - __bfloat162float(h3));
    *reinterpret_cast<uint2*>(lo + off) = l;
  }
}

}  // namespace sfb
