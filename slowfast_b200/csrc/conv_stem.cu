// Stem convolutions (C_in = 3, stride 2 in W; stem_helper.py:182 ResNetBasicStem, :258 X3DStem) on wgmma
// WITHOUT im2col traffic: "W-shift" implicit GEMM.
//
// The clip is packed channels-last with the W axis folded by the stride: X'[n, t, h, w', 8] holds pixel pairs
// (channels = parity*3 + c, two zero pads), so one pixel is exactly one 16-byte granule and the stride-2, 7-tap W
// filter becomes a stride-1, 4-tap filter over w'.  For an M tile of 128 consecutive output pixels of one output
// row, all W taps read the SAME shared-memory segment, shifted by one granule per tap - expressed purely through
// the UMMA shared-memory descriptor (no-swizzle canonical layout: rows 16 B apart, start address + tap*16 B,
// K-chunk stride 16 B).  One tiled TMA load per (kt, kh) therefore feeds KW' taps: L2->smem operand traffic
// drops KW' x 2 against per-tap im2col with 16-byte rows (the fast-pathway stem went from 12.4 M TMA ops to
// 0.9 M per step) and padding is the unit's zero fill.
//
// fprop:  D[128 pixels, cout]      += sum_{kt,kh} Seg(kt,kh)[pixels + tap, 8] x W[cout, (kt,kh,tap,8)]
// wgrad:  dW[cout, (kt,kh,tap,8)]  += sum_pixels dY[pixels, cout]^T x Seg(kt,kh)[pixels + tap, 8]
//         (both operands MN-major; the N' atoms of the Seg operand are the taps, 16 B apart)
// There is no dgrad: the clip needs no gradient.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "tmap.h"

namespace sfb {

constexpr int ST_MAX_STAGES = 8;
constexpr int ST_SEG_STRIDE = 2304;   // 136 granules (128 pixels + halo) rounded to a 128-byte multiple
constexpr int ST_SEG_PIX = 136;
constexpr int ST_WSEG_STRIDE = 1152;  // wgrad: 72 granules (64 pixels + halo)
constexpr int ST_WSEG_PIX = 72;
constexpr int ST_MMA_WARPS = 8;   // fprop: two warpgroups of 64 pixels; wgrad: the first warpgroup only (64 co rows)
constexpr int ST_FPROP_THREADS = 32 * (ST_MMA_WARPS + 1 + 4);
constexpr int ST_WGRAD_THREADS = 32 * (4 + 1);
constexpr int ST_BN_MAX = 128;
constexpr int ST_NPG_MAX = 4;     // wgrad: pairs per CTA, each a <= 32-column accumulator

__device__ __forceinline__ void tma_load_5d(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2, int32_t c3, int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c0, int32_t c1,
                                             int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

struct StemParams {
  CUtensorMap tmX[2];
  CUtensorMap tmB[2];   // fprop: weights [cout, K]; wgrad: dY {cout, OW, rows}
  int N, OT, OH, OW;
  int st, sh, pt, ph, pw;
  int KT, KH, KW;       // KW = folded taps (2 or 4)
  int pairs, pps, k_blocks;
  int cout, BN, w_tiles, m_tiles;
  int stages;
  uint32_t stage_bytes, a_plane_bytes, b_bytes;
  uint32_t acc_pitch, off_acc, off_staging, off_red, off_bars;
  float* out;
  float* stats;
  // wgrad only
  int npg, n_groups, co_tiles, ktot, kb_total, splits, kb_per_split, w_chunks;
  float* dw;
};

// ------------------------------------------------------------------------------------------------ fprop
template <int NSPLIT>
__global__ void __launch_bounds__(ST_FPROP_THREADS, 1) stem_fprop_kernel(const __grid_constant__ StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + ST_MAX_STAGES;
  uint64_t* tfull = empty + ST_MAX_STAGES;
  uint64_t* tempty = tfull + 1;
  float* acc_tile = reinterpret_cast<float*>(smem + p.off_acc);
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 32 * ST_MMA_WARPS);
    }
    mbar_init(tfull, 32 * ST_MMA_WARPS);
    mbar_init(tempty, 4);
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();
  constexpr uint32_t NP = NSPLIT == 3 ? 2u : 1u;
  const int total_tiles = p.m_tiles;
  const int ksteps_per_pair = p.KW / 2;

  if (warp == ST_MMA_WARPS) {
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int wt = tile % p.w_tiles;
      int r = tile / p.w_tiles;
      const int oh = r % p.OH;
      r /= p.OH;
      const int ot = r % p.OT;
      const int n = r / p.OT;
      const int w0 = wt * 128 - p.pw;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          const int pair0 = kb * p.pps;
          const int nq = min(p.pps, p.pairs - pair0);
          mbar_expect_tx(&full[stage], (uint32_t(nq) * ST_SEG_PIX * 16u + p.b_bytes) * NP);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          for (int qq = 0; qq < nq; ++qq) {
            const int pair = pair0 + qq;
            const int kt = pair / p.KH, kh = pair - kt * p.KH;
            const int h = oh * p.sh - p.ph + kh, t = ot * p.st - p.pt + kt;
            for (uint32_t pl = 0; pl < NP; ++pl)
              tma_load_5d(st + pl * p.a_plane_bytes + qq * ST_SEG_STRIDE, &p.tmX[pl], &full[stage], 0, w0, h, t, n);
          }
          for (uint32_t pl = 0; pl < NP; ++pl)
            tma_load_2d(st + NP * p.a_plane_bytes + pl * p.b_bytes, &p.tmB[pl], &full[stage], kb * 64, 0);
        }
        __syncwarp();
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp < ST_MMA_WARPS) {
    // MMA warpgroup g: pixels 64g .. 64g+63 of the tile = 8 more 128-byte row groups into each segment
    const int g = warp >> 2;
    float d[ST_BN_MAX / 2];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++it) {
      int held = -1;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const int nq = min(p.pps, p.pairs - kb * p.pps);
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + uint32_t(g) * 1024u;
        const uint32_t b_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + NP * p.a_plane_bytes;
        int kstep = 0;
        for (int qq = 0; qq < nq; ++qq) {
          for (int j = 0; j < ksteps_per_pair; ++j, ++kstep) {
            // A: rows = pixels 16 B apart (8-row groups 128 B), the two K chunks are taps 2j and 2j+1 = +16 B
            const uint32_t aa = a_base + qq * ST_SEG_STRIDE + uint32_t(2 * j) * 16u;
            const uint64_t a_hi = make_smem_desc(aa, 16, 128, 0);
            const uint64_t b_hi = make_smem_desc(b_base + uint32_t(kstep) * 32u, 16, 1024, 2);
            const uint32_t acc_flag = (kb | kstep) != 0 ? 1u : 0u;
            if (NSPLIT == 3) {
              const uint64_t a_lo = make_smem_desc(aa + p.a_plane_bytes, 16, 128, 0);
              const uint64_t b_lo = make_smem_desc(b_base + p.b_bytes + uint32_t(kstep) * 32u, 16, 1024, 2);
              wgmma_bf16<ST_BN_MAX, 0, 0>(d, p.BN, a_lo, b_hi, acc_flag);
              wgmma_bf16<ST_BN_MAX, 0, 0>(d, p.BN, a_hi, b_lo, 1u);
              wgmma_bf16<ST_BN_MAX, 0, 0>(d, p.BN, a_hi, b_hi, 1u);
            } else {
              wgmma_bf16<ST_BN_MAX, 0, 0>(d, p.BN, a_hi, b_hi, acc_flag);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0) mbar_arrive(&empty[held]);
        held = stage;
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      mbar_arrive(&empty[held]);
      mbar_wait(tempty, (it & 1) ^ 1);
      acc_store<ST_BN_MAX>(d, p.BN, acc_tile + size_t(g) * 64 * p.acc_pitch, int(p.acc_pitch));
      mbar_arrive(tfull);
    }
  } else {
    const int q = warp - (ST_MMA_WARPS + 1);
    float* stg = reinterpret_cast<float*>(smem + p.off_staging) + q * (32 * 33);
    float* red = reinterpret_cast<float*>(smem + p.off_red);
    const float* arow = acc_tile + size_t(q * 32 + lane) * p.acc_pitch;
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++it) {
      const int acc = it & 1;
      const int wt = tile % p.w_tiles;
      const int rowi = tile / p.w_tiles;  // (n, ot, oh) flattened
      const int ow = wt * 128 + q * 32 + lane;
      const bool rvalid = ow < p.OW;
      const uint32_t rmask = __ballot_sync(0xffffffffu, rvalid);
      float* red_w = red + ((size_t(acc) * 4 + q) * p.BN) * 2;
      mbar_wait(tfull, it & 1);
      for (int c0 = 0; c0 < p.BN; c0 += 32) {
        uint32_t v0[16], v1[16];
        acc_ld_x16(arow + c0, v0);
        const bool second = (c0 + 16) < p.BN;
        if (second) acc_ld_x16(arow + c0 + 16, v1);
        if (c0 + 32 >= p.BN) {  // last read of the accumulator tile: hand it back to the MMA warpgroups
          __syncwarp();
          if (lane == 0) mbar_arrive(tempty);
        }
        // transpose through shared memory: lane L then holds column c0+L of the warp's 32 pixels, so each store
        // instruction writes one contiguous 128-byte line (pixels of an output row are cout floats apart)
#pragma unroll
        for (int j = 0; j < 16; ++j) stg[lane * 33 + j] = rvalid ? __uint_as_float(v0[j]) : 0.f;  // rows past the row end
#pragma unroll
        for (int j = 0; j < 16; ++j) stg[lane * 33 + 16 + j] = (rvalid && second) ? __uint_as_float(v1[j]) : 0.f;
        __syncwarp();
        {
          const int cl = c0 + lane;
          // narrow outputs (the fast pathway's 8 channels): 32 lanes cover 32/W consecutive pixels x W columns, which
          // is one contiguous span because pixels are exactly cout floats apart
          const bool cvalid = cl < min(p.BN, p.cout);
          float* dst = p.out + (static_cast<long long>(rowi) * p.OW + wt * 128 + q * 32) * p.cout + cl;
          if (p.cout <= 16 && (p.cout & (p.cout - 1)) == 0 && p.BN <= 32) {
            const int W = p.cout;          // 8 or 16 (power of two, checked on the host)
            const int R = 32 / W;          // pixels per store instruction
            const int col = lane & (W - 1), rsub = lane / W;
            float s = 0.f, s2 = 0.f;
            float* d2 = p.out + (static_cast<long long>(rowi) * p.OW + wt * 128 + q * 32) * p.cout + col;
            for (int r0 = 0; r0 < 32; r0 += R) {
              const int r = r0 + rsub;
              const float y = stg[r * 33 + col];
              s += y;
              s2 = fmaf(y, y, s2);
              if ((rmask >> r) & 1u) d2[static_cast<long long>(r) * p.cout] = y;
            }
            // fold the R row-groups that share a column
            for (int o = W; o < 32; o <<= 1) {
              s += __shfl_xor_sync(0xffffffffu, s, o);
              s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            }
            if (p.stats != nullptr && lane < W) {
              red_w[lane * 2 + 0] = s;
              red_w[lane * 2 + 1] = s2;
            }
            if (p.stats != nullptr && lane >= W && lane < p.BN) {
              red_w[lane * 2 + 0] = 0.f;
              red_w[lane * 2 + 1] = 0.f;
            }
            __syncwarp();
            continue;
          }
          float s = 0.f, s2 = 0.f;
#pragma unroll 8
          for (int r = 0; r < 32; ++r) {
            const float y = stg[r * 33 + lane];
            s += y;
            s2 = fmaf(y, y, s2);
            if (((rmask >> r) & 1u) && cvalid) dst[static_cast<long long>(r) * p.cout] = y;
          }
          if (p.stats != nullptr && cl < p.BN) {
            red_w[cl * 2 + 0] = s;
            red_w[cl * 2 + 1] = s2;
          }
          __syncwarp();
        }
      }
      if (p.stats != nullptr) {
        named_bar_sync(1, 128);
        const float* rb = red + size_t(acc) * 4 * p.BN * 2;
        for (int cl = q * 32 + lane; cl < p.BN; cl += 128) {
          if (cl < p.cout) {
            float s = 0.f, s2 = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              s += rb[(size_t(w) * p.BN + cl) * 2 + 0];
              s2 += rb[(size_t(w) * p.BN + cl) * 2 + 1];
            }
            p.stats[size_t(cl) * p.m_tiles + tile] = s;
            p.stats[(size_t(p.cout) + cl) * p.m_tiles + tile] = s2;
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ wgrad
__device__ __forceinline__ void st_red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

template <int NSPLIT>
__global__ void __launch_bounds__(ST_WGRAD_THREADS, 1) stem_wgrad_kernel(const __grid_constant__ StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + ST_MAX_STAGES;
  constexpr uint32_t NP = NSPLIT == 3 ? 2u : 1u;

  const int split = blockIdx.x % p.splits;
  const int grp = blockIdx.x / p.splits;  // pair group (co_tiles == 1: cout <= 128)
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
  const int pair_base = grp * p.npg;
  const int npairs = min(p.npg, p.pairs - pair_base);
  const int ncols_pair = p.KW * 8;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 128);
    }
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();
  const uint32_t dy_plane = 8192;  // one [64 pos][64 co] box = the 64 rows of the MMA

  if (kb1 > kb0 && npairs > 0) {
    if (warp == 4) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          const int wc = kb % p.w_chunks;
          int r = kb / p.w_chunks;
          const int rowi = r;
          const int oh = r % p.OH;
          r /= p.OH;
          const int ot = r % p.OT;
          const int n = r / p.OT;
          const int ow0 = wc * 64;
          mbar_expect_tx(&full[stage], (dy_plane + uint32_t(npairs) * ST_WSEG_PIX * 16u) * NP);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          for (uint32_t pl = 0; pl < NP; ++pl) {
            tma_load_3d_(st + pl * dy_plane, &p.tmB[pl], &full[stage], 0, ow0, rowi);
            uint8_t* xb = st + NP * dy_plane + pl * p.a_plane_bytes;
            for (int j = 0; j < npairs; ++j) {
              const int pair = pair_base + j;
              const int kt = pair / p.KH, kh = pair - kt * p.KH;
              tma_load_5d(xb + j * ST_WSEG_STRIDE, &p.tmX[pl], &full[stage], 0, ow0 - p.pw, oh * p.sh - p.ph + kh,
                          ot * p.st - p.pt + kt, n);
            }
          }
        }
        __syncwarp();
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    } else {
      // one MMA warpgroup: accumulator of pair j = registers d[16 j ..] (ncols_pair <= 32 columns)
      float d[ST_NPG_MAX * 16];
      int stage = 0;
      uint32_t phase = 0;
      int held = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes);
        const uint32_t x_base = a_base + NP * dy_plane;
#pragma unroll
        for (int j = 0; j < ST_NPG_MAX; ++j) {
          if (j < npairs) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
              // A' = dY (MN-major, 128B swizzle); B' = segment: tap atoms 16 B apart, positions 16 B apart,
              // 8-position groups 128 B apart (no swizzle)
              const uint64_t a_hi = make_smem_desc(a_base + ks * 2048, 0, 1024, 2);
              const uint64_t b_hi = make_smem_desc(x_base + j * ST_WSEG_STRIDE + ks * 256, 128, 16, 0);
              const uint32_t acc_flag = (kb != kb0 || ks != 0) ? 1u : 0u;
              if (NSPLIT == 3) {
                const uint64_t a_lo = make_smem_desc(a_base + dy_plane + ks * 2048, 0, 1024, 2);
                const uint64_t b_lo =
                    make_smem_desc(x_base + p.a_plane_bytes + j * ST_WSEG_STRIDE + ks * 256, 128, 16, 0);
                wgmma_bf16<32, 1, 1>(d + 16 * j, ncols_pair, a_lo, b_hi, acc_flag);
                wgmma_bf16<32, 1, 1>(d + 16 * j, ncols_pair, a_hi, b_lo, 1u);
                wgmma_bf16<32, 1, 1>(d + 16 * j, ncols_pair, a_hi, b_hi, 1u);
              } else {
                wgmma_bf16<32, 1, 1>(d + 16 * j, ncols_pair, a_hi, b_hi, acc_flag);
              }
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0) mbar_arrive(&empty[held]);
        held = stage;
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      // epilogue straight from the fragments: rows co = 16 w + lane/4 (+8), columns 8 c + 2 (lane % 4) (+1)
      const int co0 = warp * 16 + (lane >> 2);
      const int col_base = pair_base * ncols_pair;
#pragma unroll
      for (int j = 0; j < ST_NPG_MAX; ++j) {
        if (j < npairs) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (8 * c < ncols_pair) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int co = co0 + 8 * h;
                if (co < p.cout) {
                  float* dst = p.dw + size_t(co) * p.ktot + col_base + j * ncols_pair + 8 * c + 2 * (lane & 3);
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(d[16 * j + 4 * c + 2 * h]),
                               "f"(d[16 * j + 4 * c + 2 * h + 1]) : "memory");
                }
              }
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ packing
// NCDHW fp32 clip -> X'[n, t, h, w/2, 8] split planes, channel = parity*cin + c (cin <= 4)
__global__ void stem_input_fold_kernel(const float* __restrict__ x, int n, int cin, int t, int h, int w,
                                       __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int w2 = w / 2;
  const int64_t thw = int64_t(t) * h * w;
  const int64_t items = int64_t(n) * t * h * w2;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int wp = int(i % w2);
    const int64_t rest = i / w2;  // (n*t + tt)*h + hh
    const int64_t nt = rest / h;
    const int hh = int(rest - nt * h);
    const int64_t b = nt / t;
    const int tt = int(nt - b * t);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    for (int par = 0; par < 2; ++par)
      for (int c = 0; c < cin; ++c)
        v[par * cin + c] = x[(b * cin + c) * thw + (int64_t(tt) * h + hh) * w + 2 * wp + par];
    alignas(16) __nv_bfloat16 hv[8], lv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      hv[j] = __float2bfloat16_rn(v[j]);
      lv[j] = __float2bfloat16_rn(v[j] - __bfloat162float(hv[j]));
    }
    *reinterpret_cast<uint4*>(hi + i * 8) = *reinterpret_cast<const uint4*>(hv);
    if (lo) *reinterpret_cast<uint4*>(lo + i * 8) = *reinterpret_cast<const uint4*>(lv);
  }
}

// weight [cout][cin][kt][kh][kw] -> folded filter matrix [cout][kt][kh][kw'][8] (planes), slot (kw', parity, c)
// holds tap kw = 2*(kw' + dmin) + parity + pad  where dmin = floor(-pad / 2); slots without a tap are zero.
// reverse == 1: scatter a folded fp32 gradient matrix back into the parameter layout (dw = gradient).
__global__ void stem_filter_fold_kernel(const float* __restrict__ w, float* __restrict__ dw, int cout, int cin, int kt,
                                        int kh, int kw, int pad, int kwf, __nv_bfloat16* __restrict__ hi,
                                        __nv_bfloat16* __restrict__ lo, const float* __restrict__ gmat, int reverse) {
  const int dmin = (-pad >= 0) ? (-pad) / 2 : -((pad + 1) / 2);  // floor(-pad/2)
  const int64_t items = int64_t(cout) * kt * kh * kwf * 8;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int slot = int(i % 8);
    int64_t r = i / 8;
    const int kwp = int(r % kwf);
    r /= kwf;
    const int ih = int(r % kh);
    r /= kh;
    const int it = int(r % kt);
    const int co = int(r / kt);
    const int par = slot / cin, c = slot - par * cin;
    const int tap = 2 * (kwp + dmin) + par + pad;
    const bool valid = slot < 2 * cin && tap >= 0 && tap < kw;
    const int64_t widx = (((int64_t(co) * cin + c) * kt + it) * kh + ih) * kw + tap;
    if (reverse) {
      if (valid) dw[widx] = gmat[i];
    } else {
      const float v = valid ? w[widx] : 0.f;
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[i] = h;
      if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
  }
}

typedef CUresult (*EncodeTiledFnS)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnS st_encode() {
  static EncodeTiledFnS fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFnS>(f);
  }
  return fn;
}
// X'[n, t, h, w', 8] bf16, box = [1,1,1,pix,8], no swizzle
static int make_tmap_fold(CUtensorMap* out, const void* base, int n, int t, int h, int w2, uint32_t pix) {
  EncodeTiledFnS fn = st_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point unavailable");
    return -1;
  }
  cuuint64_t dims[5] = {8, (cuuint64_t)w2, (cuuint64_t)h, (cuuint64_t)t, (cuuint64_t)n};
  cuuint64_t strides[4] = {16, 16ull * w2, 16ull * w2 * h, 16ull * w2 * h * t};
  cuuint32_t box[5] = {8, pix, 1, 1, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(fold 5d) failed (%d)", (int)r);
    return -2;
  }
  return 0;
}
// dY [rows, OW, cout] bf16 (cout contiguous), box = [1][64 ow][64 co], 128B swizzle
static int make_tmap_dy3(CUtensorMap* out, const void* base, int64_t rows, int ow, int cout) {
  EncodeTiledFnS fn = st_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point unavailable");
    return -1;
  }
  cuuint64_t dims[3] = {(cuuint64_t)cout, (cuuint64_t)ow, (cuuint64_t)rows};
  cuuint64_t strides[2] = {2ull * cout, 2ull * cout * ow};
  cuuint32_t box[3] = {64, 64, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(dy 3d) failed (%d)", (int)r);
    return -2;
  }
  return 0;
}

static int st_sms = 0, st_smem = 0;
static int st_props() {
  if (st_sms) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("cudaGetDevice failed: no CUDA device");
    return -1;
  }
  cudaDeviceGetAttribute(&st_sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&st_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return 0;
}

static int fill_common(StemParams& p, const sfb_stem_desc* d) {
  if (d->kwf != 2 && d->kwf != 4) {
    set_error("sfb_stem: folded W taps must be 2 or 4 (got %d)", d->kwf);
    return -10;
  }
  if (d->cout % 8 || d->cout > 128) {
    set_error("sfb_stem: cout=%d must be a multiple of 8 and <= 128", d->cout);
    return -10;
  }
  p.N = d->n; p.OT = d->out_t; p.OH = d->out_h; p.OW = d->out_w;
  p.st = d->str_t; p.sh = d->str_h; p.pt = d->pad_t; p.ph = d->pad_h; p.pw = d->pad_wf;
  p.KT = d->kt; p.KH = d->kh; p.KW = d->kwf;
  p.pairs = d->kt * d->kh;
  p.cout = d->cout;
  p.ktot = p.pairs * d->kwf * 8;
  return 0;
}

}  // namespace sfb

using namespace sfb;
typedef __nv_bfloat16 bf16s;

extern "C" int sfb_stem_input_fold(const float* x, int32_t n, int32_t cin, int32_t t, int32_t h, int32_t w, void* hi,
                                   void* lo, void* stream) {
  if (cin < 1 || cin > 4 || (w & 1)) {
    set_error("sfb_stem_input_fold: cin=%d must be <= 4 and w=%d even", cin, w);
    return -10;
  }
  const int64_t items = int64_t(n) * t * h * (w / 2);
  int64_t grid = (items + 255) / 256;
  if (grid > 148 * 16) grid = 148 * 16;
  stem_input_fold_kernel<<<int(grid), 256, 0, (cudaStream_t)stream>>>(x, n, cin, t, h, w, (bf16s*)hi, (bf16s*)lo);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem_input_fold launch failed: %s", cudaGetErrorString(e));
    return -20;
  }
  return 0;
}

extern "C" int sfb_stem_filter_fold(const float* w, float* dw, int32_t cout, int32_t cin, int32_t kt, int32_t kh,
                                    int32_t kw, int32_t pad_w, int32_t kwf, void* hi, void* lo, const float* gmat,
                                    int32_t reverse, void* stream) {
  const int64_t items = int64_t(cout) * kt * kh * kwf * 8;
  int64_t grid = (items + 255) / 256;
  if (grid > 148 * 8) grid = 148 * 8;
  stem_filter_fold_kernel<<<int(grid), 256, 0, (cudaStream_t)stream>>>(w, dw, cout, cin, kt, kh, kw, pad_w, kwf,
                                                                       (bf16s*)hi, (bf16s*)lo, gmat, reverse);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem_filter_fold launch failed: %s", cudaGetErrorString(e));
    return -20;
  }
  return 0;
}

extern "C" int64_t sfb_stem_m_tiles(const sfb_stem_desc* d) {
  return int64_t(d->n) * d->out_t * d->out_h * ((d->out_w + 127) / 128);
}

extern "C" int sfb_stem_fprop(const sfb_stem_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (st_props()) return -1;
  StemParams p;
  memset(&p, 0, sizeof(p));
  int rc = fill_common(p, d);
  if (rc) return rc;
  const int np = d->nsplit == 3 ? 2 : 1;
  p.pps = 64 / (d->kwf * 8);
  p.k_blocks = (p.pairs + p.pps - 1) / p.pps;
  p.BN = (d->cout + 15) / 16 * 16;
  if (p.BN > ST_BN_MAX) {
    set_error("sfb_stem_fprop: cout=%d > %d not supported", d->cout, ST_BN_MAX);
    return -10;
  }
  p.w_tiles = (d->out_w + 127) / 128;
  p.m_tiles = int(sfb_stem_m_tiles(d));
  p.a_plane_bytes = p.pps * ST_SEG_STRIDE;
  p.b_bytes = p.BN * 128;
  p.stage_bytes = ((p.a_plane_bytes + p.b_bytes) * np + 1023) / 1024 * 1024;
  // B must start 1024-aligned inside the stage for the 128B swizzle
  p.a_plane_bytes = (p.a_plane_bytes + 1023) / 1024 * 1024;
  p.stage_bytes = (p.a_plane_bytes + p.b_bytes) * np;
  p.acc_pitch = uint32_t(p.BN) + 4;
  const uint32_t acc_bytes = 128u * p.acc_pitch * 4u;
  const uint32_t tail = acc_bytes + 4 * 32 * 33 * 4 + 2 * 4 * p.BN * 2 * 4 + 256;
  p.stages = std::min<int>(ST_MAX_STAGES, (uint32_t(st_smem) - 1024 - tail) / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, p.k_blocks * 2));
  p.off_acc = p.stages * p.stage_bytes;
  p.off_staging = p.off_acc + acc_bytes;
  p.off_red = p.off_staging + 4 * 32 * 33 * 4;
  p.off_bars = p.off_red + 2 * 4 * p.BN * 2 * 4;
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  p.out = d->out;
  p.stats = d->stats;
  for (int pl = 0; pl < np; ++pl) {
    rc = make_tmap_fold(&p.tmX[pl], pl ? d->x_lo : d->x_hi, d->n, d->t, d->h, d->wf, ST_SEG_PIX);
    if (rc) return rc;
    rc = make_tmap_2d_bf16(&p.tmB[pl], pl ? d->f_lo : d->f_hi, d->cout, p.ktot, p.ktot, p.BN, 64, SWZ_128);
    if (rc) return rc;
  }
  const int grid = std::min(p.m_tiles, st_sms);
  if (d->nsplit == 3) {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem_fprop_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, st_smem); a = true; }
    stem_fprop_kernel<3><<<grid, ST_FPROP_THREADS, smem_bytes, stream>>>(p);
  } else {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem_fprop_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, st_smem); a = true; }
    stem_fprop_kernel<1><<<grid, ST_FPROP_THREADS, smem_bytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem_fprop launch failed: %s (smem=%u stages=%d)", cudaGetErrorString(e), smem_bytes, p.stages);
    return -20;
  }
  return 0;
}

extern "C" int sfb_stem_wgrad(const sfb_stem_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (st_props()) return -1;
  if (d->cout > 64) {
    set_error("sfb_stem_wgrad: cout=%d > 64 not supported", d->cout);
    return -10;
  }
  StemParams p;
  memset(&p, 0, sizeof(p));
  int rc = fill_common(p, d);
  if (rc) return rc;
  const int np = d->nsplit == 3 ? 2 : 1;
  const int ncols_pair = d->kwf * 8;
  if (ncols_pair > 32) {
    set_error("sfb_stem_wgrad: %d folded W taps > 4 not supported", d->kwf);
    return -10;
  }
  p.npg = std::min(p.pairs, ST_NPG_MAX);
  p.n_groups = (p.pairs + p.npg - 1) / p.npg;
  p.w_chunks = (d->out_w + 63) / 64;
  p.kb_total = d->n * d->out_t * d->out_h * p.w_chunks;
  int splits = std::max(1, (2 * st_sms) / p.n_groups);
  splits = std::min(splits, std::max(1, p.kb_total / 8));
  p.kb_per_split = (p.kb_total + splits - 1) / splits;
  p.splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  p.a_plane_bytes = (p.npg * ST_WSEG_STRIDE + 127) / 128 * 128;
  p.stage_bytes = ((8192 + p.a_plane_bytes) * np + 1023) / 1024 * 1024;
  // keep the X planes contiguous after the dY planes: offsets used by the kernel are NP*8192 + pl*a_plane_bytes
  p.stages = std::min<int>(ST_MAX_STAGES, (uint32_t(st_smem) - 1024 - 256) / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, p.kb_per_split));
  p.off_bars = p.stages * p.stage_bytes;
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  p.dw = d->dwm;
  const int64_t rows = int64_t(d->n) * d->out_t * d->out_h;
  for (int pl = 0; pl < np; ++pl) {
    rc = make_tmap_fold(&p.tmX[pl], pl ? d->x_lo : d->x_hi, d->n, d->t, d->h, d->wf, ST_WSEG_PIX);
    if (rc) return rc;
    rc = make_tmap_dy3(&p.tmB[pl], pl ? d->dy_lo : d->dy_hi, rows, d->out_w, d->cout);
    if (rc) return rc;
  }
  const int grid = p.n_groups * p.splits;
  if (d->nsplit == 3) {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem_wgrad_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, st_smem); a = true; }
    stem_wgrad_kernel<3><<<grid, ST_WGRAD_THREADS, smem_bytes, stream>>>(p);
  } else {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem_wgrad_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, st_smem); a = true; }
    stem_wgrad_kernel<1><<<grid, ST_WGRAD_THREADS, smem_bytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem_wgrad launch failed: %s (grid=%d smem=%u)", cudaGetErrorString(e), grid, smem_bytes);
    return -20;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ direct (SIMT) wgrad
// The fast pathway's stem (3 -> 8 channels, 5x7x7, stride (1,2,2)) has only 8 output channels: as a tensor-core GEMM
// dW[8, 735] it fills 8 of the 128 UMMA rows and was MMA-issue-bound (4.5 ms per step).  Its 19 GMAC are cheap on the
// fp32 pipes, exact, and the operands are read once: one thread owns 3 of the 735 (ci,kt,kh,kw) taps for all 8 output
// channels (24 register accumulators), a block stages the 5x7 input rows one output row touches (straight from the
// fp32 NCTHW clip) and that row's dY in shared memory, and walks the 112 output pixels: per pixel and thread 2
// broadcast LDS.128 (dY) + 3 LDS (taps) feed 24 FMAs.  Persistent blocks, one atomic add per (tap, channel) and block.
namespace sfb {
constexpr int SD_COUT = 8, SD_CIN = 3, SD_THREADS = 256, SD_TPT = 3;
struct StemDirectParams {
  const float* x;  // [n][3][T][H][W]
  const __nv_bfloat16* dy_hi; const __nv_bfloat16* dy_lo;  // [n][OT][OH][OW][8]
  float* dw;       // [8][3][KT][KH][KW]
  int n, T, H, W, OT, OH, OW, KT, KH, KW, pt, ph, pw;
  int xw;          // padded row length in shared memory
  int rows_total, rows_per_block;
};
__global__ void __launch_bounds__(SD_THREADS) stem_wgrad_direct_kernel(const StemDirectParams p) {
  extern __shared__ float sm[];
  float* xs = sm;                                           // [KT][KH][3][xw]
  float* dys = sm + size_t(p.KT) * p.KH * SD_CIN * p.xw;    // [OW][8]
  const int taps = SD_CIN * p.KT * p.KH * p.KW;
  int toff[SD_TPT], tkw[SD_TPT];
  bool tok[SD_TPT];
#pragma unroll
  for (int j = 0; j < SD_TPT; ++j) {
    const int tap = threadIdx.x + j * SD_THREADS;
    tok[j] = tap < taps;
    const int tt = tok[j] ? tap : 0;
    const int kw = tt % p.KW;
    int r = tt / p.KW;
    const int kh = r % p.KH;
    r /= p.KH;
    const int kt = r % p.KT;
    const int ci = r / p.KT;
    toff[j] = ((kt * p.KH + kh) * SD_CIN + ci) * p.xw + kw;
    tkw[j] = kw;
  }
  float acc[SD_TPT][SD_COUT];
#pragma unroll
  for (int j = 0; j < SD_TPT; ++j)
#pragma unroll
    for (int c = 0; c < SD_COUT; ++c) acc[j][c] = 0.f;
  const int r0 = blockIdx.x * p.rows_per_block;
  const int r1 = min(p.rows_total, r0 + p.rows_per_block);
  const int xrows = p.KT * p.KH * SD_CIN;
  const int w4 = p.W / 4;
  for (int row = r0; row < r1; ++row) {
    const int oh = row % p.OH;
    int r = row / p.OH;
    const int ot = r % p.OT;
    const int n = r / p.OT;
    __syncthreads();  // previous row fully consumed
    // ---- stage the KT x KH x 3 input rows (zero rows / columns where the padding is)
    for (int i = threadIdx.x; i < xrows * (p.xw / 4); i += SD_THREADS) {
      const int q = i % (p.xw / 4);
      int rr = i / (p.xw / 4);
      const int ci = rr % SD_CIN;
      rr /= SD_CIN;
      const int kh = rr % p.KH;
      const int kt = rr / p.KH;
      const int it = ot - p.pt + kt, ih = oh * 2 - p.ph + kh;
      // smem column s holds input column s - pw'; pw' = 4 (>= pw) keeps the float4 copies aligned
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      const int wq = q - 1;  // float4 index into the input row
      if (it >= 0 && it < p.T && ih >= 0 && ih < p.H && wq >= 0 && wq < w4)
        v = *reinterpret_cast<const float4*>(p.x + (((int64_t(n) * SD_CIN + ci) * p.T + it) * p.H + ih) * p.W + wq * 4);
      *reinterpret_cast<float4*>(xs + ((kt * p.KH + kh) * SD_CIN + ci) * p.xw + q * 4) = v;
    }
    for (int i = threadIdx.x; i < p.OW * 2; i += SD_THREADS) {
      const int64_t off = (int64_t(row) * p.OW) * SD_COUT + i * 4;
      const uint2 h = *reinterpret_cast<const uint2*>(p.dy_hi + off);
      float4 v = make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u), __uint_as_float(h.y << 16),
                             __uint_as_float(h.y & 0xffff0000u));
      if (p.dy_lo) {
        const uint2 l = *reinterpret_cast<const uint2*>(p.dy_lo + off);
        v.x += __uint_as_float(l.x << 16); v.y += __uint_as_float(l.x & 0xffff0000u);
        v.z += __uint_as_float(l.y << 16); v.w += __uint_as_float(l.y & 0xffff0000u);
      }
      *reinterpret_cast<float4*>(dys + i * 4) = v;
    }
    __syncthreads();
    // ---- accumulate: input column of tap kw for output pixel ow = 2*ow - pw + kw  -> smem column + 4
    const int cbase = 4 - p.pw;
#pragma unroll 4
    for (int ow = 0; ow < p.OW; ++ow) {
      const float4 d0 = *reinterpret_cast<const float4*>(dys + ow * 8);
      const float4 d1 = *reinterpret_cast<const float4*>(dys + ow * 8 + 4);
#pragma unroll
      for (int j = 0; j < SD_TPT; ++j) {
        const float xv = xs[toff[j] + cbase + 2 * ow];
        acc[j][0] = fmaf(d0.x, xv, acc[j][0]); acc[j][1] = fmaf(d0.y, xv, acc[j][1]);
        acc[j][2] = fmaf(d0.z, xv, acc[j][2]); acc[j][3] = fmaf(d0.w, xv, acc[j][3]);
        acc[j][4] = fmaf(d1.x, xv, acc[j][4]); acc[j][5] = fmaf(d1.y, xv, acc[j][5]);
        acc[j][6] = fmaf(d1.z, xv, acc[j][6]); acc[j][7] = fmaf(d1.w, xv, acc[j][7]);
      }
    }
  }
  (void)tkw;
#pragma unroll
  for (int j = 0; j < SD_TPT; ++j) {
    if (!tok[j]) continue;
    const int tap = threadIdx.x + j * SD_THREADS;  // = ((ci*KT + kt)*KH + kh)*KW + kw: the parameter's own tap order
#pragma unroll
    for (int c = 0; c < SD_COUT; ++c) atomicAdd(p.dw + size_t(c) * taps + tap, acc[j][c]);
  }
}
}  // namespace sfb

extern "C" int sfb_stem_wgrad_direct(const float* x, int32_t n, int32_t cin, int32_t t, int32_t h, int32_t w,
                                     const void* dy_hi, const void* dy_lo, int32_t cout, int32_t kt, int32_t kh,
                                     int32_t kw, int32_t st, int32_t sh, int32_t sw, int32_t pt, int32_t ph, int32_t pw,
                                     float* dw, void* stream) {
  using namespace sfb;
  if (cin != SD_CIN || cout != SD_COUT || st != 1 || sh != 2 || sw != 2 || pw > 4 || w % 4 ||
      cin * kt * kh * kw > SD_THREADS * SD_TPT) {
    set_error("sfb_stem_wgrad_direct: only the 3 -> 8 channel, stride (1,2,2) stem with <= %d taps is supported",
              SD_THREADS * SD_TPT);
    return -10;
  }
  StemDirectParams p;
  p.x = x; p.dy_hi = (const __nv_bfloat16*)dy_hi; p.dy_lo = (const __nv_bfloat16*)dy_lo; p.dw = dw;
  p.n = n; p.T = t; p.H = h; p.W = w;
  p.OT = (t + 2 * pt - kt) / st + 1; p.OH = (h + 2 * ph - kh) / sh + 1; p.OW = (w + 2 * pw - kw) / sw + 1;
  p.KT = kt; p.KH = kh; p.KW = kw; p.pt = pt; p.ph = ph; p.pw = pw;
  // smem row: 4 zero columns, the W input columns, then zeros up to the last column any tap reads, rounded to 4
  const int need = 4 - pw + 2 * (p.OW - 1) + kw;
  p.xw = (std::max(need, w + 4) + 3) / 4 * 4 + 4;
  p.rows_total = n * p.OT * p.OH;
  int blocks = 148 * 2;
  if (blocks > p.rows_total) blocks = p.rows_total;
  p.rows_per_block = (p.rows_total + blocks - 1) / blocks;
  blocks = (p.rows_total + p.rows_per_block - 1) / p.rows_per_block;
  const size_t smem = (size_t(kt) * kh * SD_CIN * p.xw + size_t(p.OW) * SD_COUT) * sizeof(float);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(stem_wgrad_direct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    attr = true;
  }
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemsetAsync(dw, 0, size_t(cout) * cin * kt * kh * kw * sizeof(float), s);
  stem_wgrad_direct_kernel<<<blocks, SD_THREADS, smem, s>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem_wgrad_direct launch failed: %s (smem=%zu)", cudaGetErrorString(e), smem);
    return -20;
  }
  return 0;
}
