// Fused pooled attention for MViT's MultiScaleAttention (attention.py:355-385) on wgmma, per (clip*head, 64-query tile):
//
//   forward   S = q k^T (wgmma 64 x 80 x 16 per key tile, 5 tiles = 400 keys)  -> fp32 score block in shared memory
//             t = scale*S + rel-pos bias(q, k)  (cal_rel_pos_spatial / _temporal, attention.py:64-147, from RQ = q.[Rh;Rw;Rt]^T)
//             P = softmax(t)  (exact: the whole key axis is resident), written to global memory as split planes (the
//                              backward reads them) and staged 64 keys at a time as 128B-swizzled K-major bf16 planes
//             O = P v   (wgmma 64 x 96 x 16, accumulator in registers; v arrives by TMA as MN-major atoms)
//   backward  dP = dO v^T (same tile loop as S), dS = P (dP - sum_k P dP) -> split planes, dRQ = the rel-pos bias gradient
//
// Neither S nor dP goes to HBM.  Key grids with Nk <= 400 and head_dim 96 (MViTv2-S: 8 x 7 x 7 keys in 12 of 16 blocks);
// other grids keep the unfused sequence (sfb_gemm_batched -> sfb_softmax_relpos_* -> sfb_gemm_batched).
// One warpgroup per CTA: warp-uniform TMA issue by thread 0, every wgmma waited before its shared-memory operands are
// reused.  The row passes repeat the arithmetic of softmax_relpos_fwd / _bwd (mvit_ops.cu) on the resident block.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "tmap.h"

namespace sfb {

constexpr int AF_BM = 64;          // queries per CTA (one warpgroup, wgmma M)
constexpr int AF_BN = 80;          // keys per score tile (wgmma N)
constexpr int AF_NKT = 5;          // score tiles: 400 keys
constexpr int AF_NK_MAX = AF_BN * AF_NKT;
constexpr int AF_HD = 96;          // head dim
constexpr int AF_SP = AF_NK_MAX + 4;                // floats per score row
constexpr uint32_t AF_QT_BYTES = AF_BM * 128;       // [64 rows x 64 dims] bf16 K-major SW128 tile (q / dO / P k-block)
constexpr uint32_t AF_KT_BYTES = AF_BN * 128;       // [80 keys x 64 dims] bf16 K-major SW128 tile
constexpr uint32_t AF_VA_BYTES = 64 * 128;          // [64 keys x 64 dims] MN-major SW128 atom of v
// shared memory: A operand (2 planes x 2 k-blocks), key tile (2 planes x 2 k-blocks, reused for v: 2 planes x 2 atoms),
// P staging (2 planes), score block, barriers
constexpr uint32_t AF_OFF_A = 0;
constexpr uint32_t AF_OFF_K = AF_OFF_A + 4 * AF_QT_BYTES;
constexpr uint32_t AF_OFF_P = AF_OFF_K + 4 * AF_KT_BYTES;
constexpr uint32_t AF_OFF_S = AF_OFF_P + 2 * AF_QT_BYTES;
constexpr uint32_t AF_OFF_BINS = AF_OFF_S + AF_BM * AF_SP * 4;
constexpr uint32_t AF_BINS_FLOATS = 256;            // per warp: Lh + Lw + Lt (checked on the host)
constexpr uint32_t AF_OFF_BAR = AF_OFF_BINS + 4 * AF_BINS_FLOATS * 4;
constexpr uint32_t AF_SMEM = AF_OFF_BAR + 64 + 1024;

struct AttnParams {
  CUtensorMap tmA[2], tmK[2], tmV[2];   // fwd: q, k, v;  bwd: dO, v (as the K-major key operand), unused
  int BH, Nq, Nk, q_tiles;
  const float* rq; int64_t rq_pitch;    // fwd: RQ [BH*(Nq-1), rq_pitch] or null
  int qt, qh, qw, kt, kh, kw, Lh, Lw, Lt;
  float rh_q, rh_k, rw_q, rw_k, rt_q, rt_k;
  float scale;
  float* out;                           // fwd: O [BH, Nq, 96]
  float* lse;                           // fwd: [BH*Nq] or null
  __nv_bfloat16* p_hi; __nv_bfloat16* p_lo; int64_t p_pitch;     // fwd: written; bwd: read
  __nv_bfloat16* ds_hi; __nv_bfloat16* ds_lo; int64_t ds_pitch;  // bwd
  float* drq;                           // bwd: [BH*(Nq-1), rq_pitch] or null
};

__device__ __forceinline__ void af_tma_3d(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void af_put_split(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t i, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}
__device__ __forceinline__ float af_get_split(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t i) {
  return __bfloat162float(hi[i]) + (lo ? __bfloat162float(lo[i]) : 0.f);
}
__device__ __forceinline__ float af_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int af_rel_index(int i, int j, float rq, float rk, int nk) {
  return int(floorf(float(i) * rq - float(j) * rk + float(nk - 1) * rk));
}

// S[64 x 400] (fp32, shared) = A[64 x 96] . B[keys x 96]^T for the CTA's query tile; A (q or dO) is loaded here too.
// `phase` tracks the single TMA barrier.  Keys past Nk read as zero (TMA out-of-bounds fill).
template <int NSPLIT>
__device__ __forceinline__ void af_scores(const AttnParams& p, uint8_t* smem, uint64_t* bar, uint32_t& phase, int bh, int q0) {
  constexpr int NP = NSPLIT == 3 ? 2 : 1;
  float* S = reinterpret_cast<float*>(smem + AF_OFF_S);
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, NP * 2 * AF_QT_BYTES);
    for (int pl = 0; pl < NP; ++pl)
      for (int kb = 0; kb < 2; ++kb)
        af_tma_3d(smem + AF_OFF_A + (pl * 2 + kb) * AF_QT_BYTES, &p.tmA[pl], bar, kb * 64, q0, bh);
  }
  mbar_wait(bar, phase);
  phase ^= 1;
  const uint32_t a_base = smem_u32(smem + AF_OFF_A), k_base = smem_u32(smem + AF_OFF_K);
  for (int t = 0; t < AF_NKT; ++t) {
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar, NP * 2 * AF_KT_BYTES);
      for (int pl = 0; pl < NP; ++pl)
        for (int kb = 0; kb < 2; ++kb)
          af_tma_3d(smem + AF_OFF_K + (pl * 2 + kb) * AF_KT_BYTES, &p.tmK[pl], bar, kb * 64, t * AF_BN, bh);
    }
    mbar_wait(bar, phase);
    phase ^= 1;
    float d[AF_BN / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < AF_HD / 16; ++ks) {
      const uint32_t off = uint32_t(ks >> 2) * AF_QT_BYTES + uint32_t(ks & 3) * 32u;
      const uint32_t koff = uint32_t(ks >> 2) * AF_KT_BYTES + uint32_t(ks & 3) * 32u;
      const uint64_t a_hi = make_smem_desc(a_base + off, 16, 1024, 2);
      const uint64_t b_hi = make_smem_desc(k_base + koff, 16, 1024, 2);
      const uint32_t acc = ks != 0;
      if (NSPLIT == 3) {
        const uint64_t a_lo = make_smem_desc(a_base + 2 * AF_QT_BYTES + off, 16, 1024, 2);
        const uint64_t b_lo = make_smem_desc(k_base + 2 * AF_KT_BYTES + koff, 16, 1024, 2);
        wgmma_m64n80<0, 0>(d, a_lo, b_hi, acc);
        wgmma_m64n80<0, 0>(d, a_hi, b_lo, 1u);
        wgmma_m64n80<0, 0>(d, a_hi, b_hi, 1u);
      } else {
        wgmma_m64n80<0, 0>(d, a_hi, b_hi, acc);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_store<AF_BN>(d, AF_BN, S + t * AF_BN, AF_SP);
    __syncthreads();   // every thread's MMAs have read the key tile before the next load overwrites it
  }
}

template <int NSPLIT>
__global__ void __launch_bounds__(128, 1) attn_fwd_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + AF_OFF_BAR);
  float* S = reinterpret_cast<float*>(smem + AF_OFF_S);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bh = blockIdx.x / p.q_tiles, q0 = (blockIdx.x % p.q_tiles) * AF_BM;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  uint32_t phase = 0;
  af_scores<NSPLIT>(p, smem, bar, phase, bh, q0);

  // ---- biased softmax, one warp per row (softmax_relpos_fwd arithmetic); P replaces the scores, zero past Nk
  const int khw = p.kh * p.kw;
  for (int rr = warp; rr < AF_BM; rr += 4) {
    float* s = S + rr * AF_SP;
    const int q = q0 + rr;
    if (q >= p.Nq) {
      for (int k = lane; k < AF_NK_MAX; k += 32) s[k] = 0.f;
      continue;
    }
    const int64_t r = int64_t(bh) * p.Nq + q;
    const float* rq = (p.rq && q > 0) ? p.rq + (int64_t(bh) * (p.Nq - 1) + (q - 1)) * p.rq_pitch : nullptr;
    int qz = 0, qy = 0, qx = 0;
    if (q > 0) {
      int t = q - 1;
      qx = t % p.qw;
      t /= p.qw;
      qy = t % p.qh;
      qz = t / p.qh;
    }
    const float bh0 = float(qy) * p.rh_q + float(p.kh - 1) * p.rh_k;
    const float bw0 = float(qx) * p.rw_q + float(p.kw - 1) * p.rw_k;
    const float bt0 = float(qz) * p.rt_q + float(p.kt - 1) * p.rt_k;
    float mx = -INFINITY;
    for (int k = lane; k < p.Nk; k += 32) {
      float v = s[k] * p.scale;
      if (rq && k > 0) {
        const int t = k - 1;
        const int kz = t / khw;
        const int rem = t - kz * khw;
        const int ky = rem / p.kw;
        const int kx = rem - ky * p.kw;
        v += rq[int(floorf(bh0 - float(ky) * p.rh_k))] + rq[p.Lh + int(floorf(bw0 - float(kx) * p.rw_k))] +
             rq[p.Lh + p.Lw + int(floorf(bt0 - float(kz) * p.rt_k))];
      }
      s[k] = v;
      mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int k = lane; k < p.Nk; k += 32) {
      const float e = expf(s[k] - mx);
      s[k] = e;
      sum += e;
    }
    sum = af_warp_sum(sum);
    const float inv = 1.f / sum;
    for (int k = lane; k < AF_NK_MAX; k += 32) s[k] = k < p.Nk ? s[k] * inv : 0.f;
    if (p.p_hi)
      for (int k = lane; k < p.p_pitch; k += 32) af_put_split(p.p_hi, p.p_lo, r * p.p_pitch + k, k < AF_NK_MAX ? s[k] : 0.f);
    if (p.lse && lane == 0) p.lse[r] = mx + logf(sum);
  }
  __syncthreads();

  // ---- O = P v over 64-key blocks: P block -> swizzled bf16 planes, v block -> MN-major atoms, wgmma 64 x 96
  constexpr int NP = NSPLIT == 3 ? 2 : 1;
  float o[AF_HD / 2];
  const uint32_t p_base = smem_u32(smem + AF_OFF_P), v_base = smem_u32(smem + AF_OFF_K);
  const int nkb = (p.Nk + 63) / 64;
  for (int kb = 0; kb < nkb; ++kb) {
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar, NP * 2 * AF_VA_BYTES);
      for (int pl = 0; pl < NP; ++pl)
        for (int a = 0; a < 2; ++a)
          af_tma_3d(smem + AF_OFF_K + (pl * 2 + a) * AF_VA_BYTES, &p.tmV[pl], bar, a * 64, kb * 64, bh);
    }
    // element (row r, key c) of a K-major 128B-swizzled [64 x 64] tile: byte r*128 + ((c/8) ^ (r%8))*16 + (c%8)*2
    for (int i = threadIdx.x; i < AF_BM * 8; i += 128) {
      const int r = i >> 3, g = i & 7, c0 = kb * 64 + g * 8;
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float x[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) x[e] = (c0 + 2 * j + e) < AF_NK_MAX ? S[r * AF_SP + c0 + 2 * j + e] : 0.f;
        const __nv_bfloat162 h = __floats2bfloat162_rn(x[0], x[1]);
        const float2 hf = __bfloat1622float2(h);
        const __nv_bfloat162 l = __floats2bfloat162_rn(x[0] - hf.x, x[1] - hf.y);
        hw[j] = *reinterpret_cast<const uint32_t*>(&h);
        lw[j] = *reinterpret_cast<const uint32_t*>(&l);
      }
      const uint32_t off = uint32_t(r) * 128u + uint32_t((g ^ (r & 7)) * 16);
      *reinterpret_cast<uint4*>(smem + AF_OFF_P + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      if (NSPLIT == 3) *reinterpret_cast<uint4*>(smem + AF_OFF_P + AF_QT_BYTES + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
    fence_proxy_async_smem();   // the generic-proxy stores above are read by wgmma (async proxy)
    __syncthreads();
    mbar_wait(bar, phase);
    phase ^= 1;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t a_hi = make_smem_desc(p_base + ks * 32, 16, 1024, 2);
      const uint64_t b_hi = make_smem_desc(v_base + ks * 2048, AF_VA_BYTES, 1024, 2);
      const uint32_t acc = (kb | ks) != 0;
      if (NSPLIT == 3) {
        const uint64_t a_lo = make_smem_desc(p_base + AF_QT_BYTES + ks * 32, 16, 1024, 2);
        const uint64_t b_lo = make_smem_desc(v_base + 2 * AF_VA_BYTES + ks * 2048, AF_VA_BYTES, 1024, 2);
        wgmma_m64n96<0, 1>(o, a_lo, b_hi, acc);
        wgmma_m64n96<0, 1>(o, a_hi, b_lo, 1u);
        wgmma_m64n96<0, 1>(o, a_hi, b_hi, 1u);
      } else {
        wgmma_m64n96<0, 1>(o, a_hi, b_hi, acc);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();   // P staging and the v atoms are free for the next block
  }
  // O fragments -> [BH, Nq, 96]
  const int rw = warp * 16 + (lane >> 2), cp = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + rw + 8 * h;
    if (q < p.Nq) {
      float* dst = p.out + (int64_t(bh) * p.Nq + q) * AF_HD + cp;
#pragma unroll
      for (int j = 0; j < AF_HD / 8; ++j)
        *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
    }
  }
}

template <int NSPLIT>
__global__ void __launch_bounds__(128, 1) attn_bwd_ds_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + AF_OFF_BAR);
  float* S = reinterpret_cast<float*>(smem + AF_OFF_S);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bh = blockIdx.x / p.q_tiles, q0 = (blockIdx.x % p.q_tiles) * AF_BM;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  uint32_t phase = 0;
  af_scores<NSPLIT>(p, smem, bar, phase, bh, q0);   // dP = dO v^T

  // ---- dS = P (dP - sum_k P dP), dRQ (softmax_relpos_bwd arithmetic), one warp per row
  const int khw = p.kh * p.kw;
  const int Ltot = p.Lh + p.Lw + p.Lt;
  float* bins = reinterpret_cast<float*>(smem + AF_OFF_BINS) + warp * AF_BINS_FLOATS;
  for (int rr = warp; rr < AF_BM; rr += 4) {
    const int q = q0 + rr;
    if (q >= p.Nq) break;
    float* buf = S + rr * AF_SP;
    const int64_t r = int64_t(bh) * p.Nq + q;
    float dot = 0.f;
    for (int k = lane; k < p.Nk; k += 32) {
      const float pv = af_get_split(p.p_hi, p.p_lo, r * p.p_pitch + k);
      dot = fmaf(pv, buf[k], dot);
    }
    dot = af_warp_sum(dot);
    const bool rel = p.drq != nullptr && q > 0;
    if (rel)
      for (int j = lane; j < Ltot; j += 32) bins[j] = 0.f;
    for (int k = lane; k < p.ds_pitch; k += 32) {
      float ds = 0.f;
      if (k < p.Nk) {
        ds = af_get_split(p.p_hi, p.p_lo, r * p.p_pitch + k) * (buf[k] - dot);
        buf[k] = ds;
      }
      af_put_split(p.ds_hi, p.ds_lo, r * p.ds_pitch + k, ds);
    }
    __syncwarp();
    if (rel) {
      int t = q - 1;
      const int qx = t % p.qw;
      t /= p.qw;
      const int qy = t % p.qh;
      const int qz = t / p.qh;
      const float* g = buf + 1;  // key grid [kt][kh][kw] behind the cls column
      for (int a = lane; a < p.kh + p.kw + p.kt; a += 32) {
        float sum = 0.f;
        int bin;
        if (a < p.kh) {
          for (int kz = 0; kz < p.kt; ++kz)
            for (int kx = 0; kx < p.kw; ++kx) sum += g[kz * khw + a * p.kw + kx];
          bin = af_rel_index(qy, a, p.rh_q, p.rh_k, p.kh);
        } else if (a < p.kh + p.kw) {
          const int kx = a - p.kh;
          for (int kz = 0; kz < p.kt; ++kz)
            for (int ky = 0; ky < p.kh; ++ky) sum += g[kz * khw + ky * p.kw + kx];
          bin = p.Lh + af_rel_index(qx, kx, p.rw_q, p.rw_k, p.kw);
        } else {
          const int kz = a - p.kh - p.kw;
          for (int j = 0; j < khw; ++j) sum += g[kz * khw + j];
          bin = p.Lh + p.Lw + af_rel_index(qz, kz, p.rt_q, p.rt_k, p.kt);
        }
        atomicAdd(&bins[bin], sum);
      }
      __syncwarp();
      float* o = p.drq + (int64_t(bh) * (p.Nq - 1) + (q - 1)) * p.rq_pitch;
      for (int j = lane; j < p.rq_pitch; j += 32) o[j] = j < Ltot ? bins[j] : 0.f;
    }
    __syncwarp();
  }
}

typedef CUresult (*AfEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// 3-D map over bf16 [batch][rows][cols] (cols contiguous), box = [1][box_rows][64], 128B swizzle, out-of-bounds zero
static int af_tmap(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t ld, uint64_t bs,
                   uint32_t box_rows) {
  static AfEncodeFn fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeTiled entry point unavailable");
      return -1;
    }
    fn = reinterpret_cast<AfEncodeFn>(f);
  }
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {ld * 2, bs * 2};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("fused attention: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return -2;
  }
  return 0;
}

static void af_geometry(AttnParams& p, int qt, int qh, int qw, int kt, int kh, int kw) {
  p.qt = qt; p.qh = qh; p.qw = qw; p.kt = kt; p.kh = kh; p.kw = kw;
  p.Lh = 2 * std::max(qh, kh) - 1;
  p.Lw = 2 * std::max(qw, kw) - 1;
  p.Lt = 2 * std::max(qt, kt) - 1;
  auto ratio = [](int a, int b) { const float r = float(a) / float(b); return r > 1.f ? r : 1.f; };
  p.rh_q = ratio(kh, qh); p.rh_k = ratio(qh, kh);
  p.rw_q = ratio(kw, qw); p.rw_k = ratio(qw, kw);
  p.rt_q = ratio(kt, qt); p.rt_k = ratio(qt, kt);
}

template <typename K>
static int af_launch(K kernel, const AttnParams& p, cudaStream_t stream, const char* what) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(AF_SMEM));
  kernel<<<p.BH * p.q_tiles, 128, AF_SMEM, stream>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s launch failed: %s (grid=%d smem=%u)", what, cudaGetErrorString(e), p.BH * p.q_tiles, AF_SMEM);
    return -20;
  }
  return 0;
}

}  // namespace sfb

using namespace sfb;

extern "C" int32_t sfb_attn_fwd_supported(int32_t nk, int32_t hd, int32_t kt, int32_t kh, int32_t kw) {
  static const bool on = [] { const char* e = getenv("SFB_ATTN_FUSED"); return e ? e[0] != '0' : true; }();
  return on && hd == AF_HD && kh == 7 && kw == 7 && kt == 8 && nk == 1 + kt * kh * kw;
}

extern "C" int sfb_attn_fwd(const sfb_attn_fwd_desc* d, void* stream_) {
  if (!sfb_attn_fwd_supported(d->nk, d->hd, d->kt, d->kh, d->kw)) {
    set_error("sfb_attn_fwd: only head_dim 96 with an 8x7x7 key grid (Nk = 393) is fused; use the unfused sequence otherwise");
    return -10;
  }
  if (d->nsplit != 1 && d->nsplit != 3) {
    set_error("sfb_attn_fwd: nsplit must be 1 or 3");
    return -10;
  }
  if (!d->q_hi || !d->k_hi || !d->v_hi || !d->out || (d->nsplit == 3 && (!d->q_lo || !d->k_lo || !d->v_lo))) {
    set_error("sfb_attn_fwd: null operand pointer");
    return -10;
  }
  if (d->p_hi && (d->p_pitch % 8 || d->p_pitch < d->nk)) {
    set_error("sfb_attn_fwd: p_pitch must be a multiple of 8 and >= nk");
    return -10;
  }
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.BH = d->bh; p.Nq = d->nq; p.Nk = d->nk;
  p.q_tiles = (d->nq + AF_BM - 1) / AF_BM;
  p.rq = d->rq; p.rq_pitch = d->rq_pitch;
  af_geometry(p, d->qt, d->qh, d->qw, d->kt, d->kh, d->kw);
  p.scale = d->scale;
  p.out = d->out; p.lse = d->lse;
  p.p_hi = (__nv_bfloat16*)d->p_hi; p.p_lo = (__nv_bfloat16*)d->p_lo; p.p_pitch = d->p_pitch;
  const int np = d->nsplit == 3 ? 2 : 1;
  for (int pl = 0; pl < np; ++pl) {
    if (int rc = af_tmap(&p.tmA[pl], pl ? d->q_lo : d->q_hi, AF_HD, d->nq, d->bh, AF_HD, uint64_t(d->nq) * AF_HD, AF_BM)) return rc;
    if (int rc = af_tmap(&p.tmK[pl], pl ? d->k_lo : d->k_hi, AF_HD, d->nk, d->bh, AF_HD, uint64_t(d->nk) * AF_HD, AF_BN)) return rc;
    if (int rc = af_tmap(&p.tmV[pl], pl ? d->v_lo : d->v_hi, AF_HD, d->nk, d->bh, AF_HD, uint64_t(d->nk) * AF_HD, 64)) return rc;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  return d->nsplit == 3 ? af_launch(attn_fwd_kernel<3>, p, stream, "sfb_attn_fwd")
                        : af_launch(attn_fwd_kernel<1>, p, stream, "sfb_attn_fwd");
}

extern "C" int sfb_attn_bwd_ds(const sfb_attn_bwd_desc* d, void* stream_) {
  if (!sfb_attn_fwd_supported(d->nk, d->hd, d->kt, d->kh, d->kw)) {
    set_error("sfb_attn_bwd_ds: only head_dim 96 with an 8x7x7 key grid (Nk = 393) is fused");
    return -10;
  }
  if (d->nsplit != 1 && d->nsplit != 3) {
    set_error("sfb_attn_bwd_ds: nsplit must be 1 or 3");
    return -10;
  }
  if (!d->do_hi || !d->v_hi || !d->p_hi || !d->ds_hi || (d->nsplit == 3 && (!d->do_lo || !d->v_lo || !d->p_lo || !d->ds_lo))) {
    set_error("sfb_attn_bwd_ds: null operand pointer");
    return -10;
  }
  AttnParams p;
  memset(&p, 0, sizeof(p));
  af_geometry(p, d->qt, d->qh, d->qw, d->kt, d->kh, d->kw);
  if (d->p_pitch % 8 || d->p_pitch < d->nk || d->ds_pitch % 8 || d->ds_pitch < d->nk || (d->drq && d->rq_pitch % 4) ||
      p.Lh + p.Lw + p.Lt > int(AF_BINS_FLOATS)) {
    set_error("sfb_attn_bwd_ds: pitches must be multiples of 8 holding nk columns (rq_pitch a multiple of 4), rel-pos tables <= %u",
              AF_BINS_FLOATS);
    return -10;
  }
  p.BH = d->bh; p.Nq = d->nq; p.Nk = d->nk;
  p.q_tiles = (d->nq + AF_BM - 1) / AF_BM;
  p.p_hi = (__nv_bfloat16*)d->p_hi; p.p_lo = d->nsplit == 3 ? (__nv_bfloat16*)d->p_lo : nullptr; p.p_pitch = d->p_pitch;
  p.ds_hi = (__nv_bfloat16*)d->ds_hi; p.ds_lo = (__nv_bfloat16*)d->ds_lo; p.ds_pitch = d->ds_pitch;
  p.drq = d->drq; p.rq_pitch = d->rq_pitch;
  const int np = d->nsplit == 3 ? 2 : 1;
  for (int pl = 0; pl < np; ++pl) {
    if (int rc = af_tmap(&p.tmA[pl], pl ? d->do_lo : d->do_hi, AF_HD, d->nq, d->bh, AF_HD, uint64_t(d->nq) * AF_HD, AF_BM)) return rc;
    if (int rc = af_tmap(&p.tmK[pl], pl ? d->v_lo : d->v_hi, AF_HD, d->nk, d->bh, AF_HD, uint64_t(d->nk) * AF_HD, AF_BN)) return rc;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  return d->nsplit == 3 ? af_launch(attn_bwd_ds_kernel<3>, p, stream, "sfb_attn_bwd_ds")
                        : af_launch(attn_bwd_ds_kernel<1>, p, stream, "sfb_attn_bwd_ds");
}
