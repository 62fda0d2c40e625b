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
#include "planes.cuh"
#include "runtime.h"

namespace sfb {

constexpr int ST_MAX_STAGES = 8;
constexpr int ST_SEG_STRIDE = 2304;   // 136 granules (128 pixels + halo) rounded to a 128-byte multiple
constexpr int ST_SEG_PIX = 136;
constexpr int ST_WSEG_STRIDE = 1152;  // wgrad: 72 granules (64 pixels + halo)
constexpr int ST_WSEG_PIX = 72;
constexpr int ST_MMA_WARPS = 8;   // fprop: two warpgroups of 64 pixels; wgrad: two warpgroups, half the positions each
constexpr int ST_FPROP_THREADS = 32 * (ST_MMA_WARPS + 1 + 4);
constexpr int ST_WGRAD_THREADS = 32 * (ST_MMA_WARPS + 1);
constexpr int ST_BN_MAX = 64;     // the widest stem of the supported models (StemConvBN.supported)
constexpr int ST_KSTEPS = 4;      // k16 steps per k-block: 64 K elements = pps pairs x KW taps x 8 slots
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
  uint32_t a_kstep[ST_KSTEPS];  // fprop: start of k-step ks's A columns in the stage (pair segment + tap), 16-byte units
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
// Every k-block is ST_KSTEPS k16 steps over pps pairs (the producer zero-fills the pairs past the last one, whose filter
// columns the weight map's bounds also zero) and the tile width is the template's BN, so a k-block's wgmmas are
// straight-line code behind one warpgroup arrive.
template <int NSPLIT, int BN>
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
          mbar_expect_tx(&full[stage], (uint32_t(p.pps) * ST_SEG_PIX * 16u + p.b_bytes) * NP);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          for (int qq = 0; qq < p.pps; ++qq) {
            const int pair = pair0 + qq;
            const int kt = pair / p.KH, kh = pair - kt * p.KH;
            // a pair past the last one reads row -1: entirely out of bounds, so the unit fills it with zeros
            const int h = pair < p.pairs ? oh * p.sh - p.ph + kh : -1, t = ot * p.st - p.pt + kt;
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
    float d[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++it) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int held = -1;
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + uint32_t(g) * 1024u;
        const uint32_t b_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + NP * p.a_plane_bytes;
        // A: rows = pixels 16 B apart (8-row groups 128 B); a k-step's two K chunks are two taps of one pair, 16 B apart
        const uint64_t a_hi0 = make_smem_desc(a_base, 16, 128, 0);
        const uint64_t b_hi0 = make_smem_desc(b_base, 16, 1024, 2);
#pragma unroll
        for (int ks = 0; ks < ST_KSTEPS; ++ks) {
          const uint64_t a_hi = a_hi0 + p.a_kstep[ks];
          const uint64_t b_hi = b_hi0 + uint64_t(ks * 2);  // 32 bytes = 16 bf16 of the 128-byte swizzled rows
          if (NSPLIT == 3) {
            const uint64_t a_lo = a_hi + (p.a_plane_bytes >> 4);
            const uint64_t b_lo = b_hi + (p.b_bytes >> 4);
            wgmma_m64n<BN>(d, a_lo, b_hi);
            wgmma_m64n<BN>(d, a_hi, b_lo);
          }
          wgmma_m64n<BN>(d, a_hi, b_hi);
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
      acc_store<BN>(d, BN, acc_tile + size_t(g) * 64 * p.acc_pitch, int(p.acc_pitch));
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

// CTA = (group of NPG pairs, split of the (row, 64-pixel chunk) k-blocks).  Both MMA warpgroups hold the whole
// [64 co, NPG x KW*8] tile: warpgroup g takes k-steps 2g, 2g+1 (positions 32g .. 32g+31) of every stage, and the
// epilogue adds warpgroup 1's tile to warpgroup 0's through shared memory.  NPG and the pair width KW*8 are
// compile-time, so a stage's wgmmas are straight-line code; pairs past the last one are zero-filled and not stored.
template <int NSPLIT, int KWF, int NPG>
__global__ void __launch_bounds__(ST_WGRAD_THREADS, 1) stem_wgrad_kernel(const __grid_constant__ StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + ST_MAX_STAGES;
  constexpr uint32_t NP = NSPLIT == 3 ? 2u : 1u;
  constexpr int NC = KWF * 8;             // accumulator columns per pair
  constexpr int NACC = NPG * NC / 2;      // accumulator registers per thread

  const int split = blockIdx.x % p.splits;
  const int grp = blockIdx.x / p.splits;  // pair group (co_tiles == 1: cout <= 64)
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
  const int pair_base = grp * NPG;
  const int npairs = min(NPG, p.pairs - pair_base);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 32 * ST_MMA_WARPS);
    }
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();
  const uint32_t dy_plane = 8192;  // one [64 pos][64 co] box = the 64 rows of the MMA

  if (kb1 > kb0) {
    if (warp == ST_MMA_WARPS) {
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
          mbar_expect_tx(&full[stage], (dy_plane + uint32_t(NPG) * ST_WSEG_PIX * 16u) * NP);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          for (uint32_t pl = 0; pl < NP; ++pl) {
            tma_load_3d_(st + pl * dy_plane, &p.tmB[pl], &full[stage], 0, ow0, rowi);
            uint8_t* xb = st + NP * dy_plane + pl * p.a_plane_bytes;
            for (int j = 0; j < NPG; ++j) {
              const int pair = pair_base + j;
              const int kt = pair / p.KH, kh = pair - kt * p.KH;
              // a pair past the last one reads row -1: entirely out of bounds, so the unit fills it with zeros
              const int h = j < npairs ? oh * p.sh - p.ph + kh : -1;
              tma_load_5d(xb + j * ST_WSEG_STRIDE, &p.tmX[pl], &full[stage], 0, ow0 - p.pw, h, ot * p.st - p.pt + kt, n);
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
      // accumulator of pair j = registers d[j NC/2 ..]
      const int g = warp >> 2;
      float d[NACC];
#pragma unroll
      for (int i = 0; i < NACC; ++i) d[i] = 0.f;
      int stage = 0;
      uint32_t phase = 0;
      int held = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        // A' = dY (MN-major, 128B swizzle), 16 positions = 2048 B per k-step; B' = segment: tap atoms 16 B apart,
        // positions 16 B apart, 8-position groups 128 B apart (no swizzle)
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + uint32_t(g) * 2u * 2048u;
        const uint32_t x_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + NP * dy_plane + uint32_t(g) * 2u * 256u;
#pragma unroll
        for (int j = 0; j < NPG; ++j) {
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const uint64_t a_hi = make_smem_desc(a_base + ks * 2048, 0, 1024, 2);
            const uint64_t b_hi = make_smem_desc(x_base + j * ST_WSEG_STRIDE + ks * 256, 128, 16, 0);
            if (NSPLIT == 3) {
              const uint64_t a_lo = a_hi + (dy_plane >> 4);
              const uint64_t b_lo = b_hi + (p.a_plane_bytes >> 4);
              wgmma_m64n<NC, 1, 1>(d + j * (NC / 2), a_lo, b_hi);
              wgmma_m64n<NC, 1, 1>(d + j * (NC / 2), a_hi, b_lo);
            }
            wgmma_m64n<NC, 1, 1>(d + j * (NC / 2), a_hi, b_hi);
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
      // warpgroup 1 hands its tile to warpgroup 0 through the stages (every load has landed and both warpgroups' MMAs
      // are done once both pass the first barrier); the same thread of the other warpgroup holds the same elements
      float* red = reinterpret_cast<float*>(smem);
      const int t = threadIdx.x & 127;
      named_bar_sync(1, 32 * ST_MMA_WARPS);
      if (g == 1) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) red[i * 128 + t] = d[i];
      }
      named_bar_sync(1, 32 * ST_MMA_WARPS);
      if (g == 0) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) d[i] += red[i * 128 + t];
        // epilogue straight from the fragments: rows co = 16 w + lane/4 (+8), columns 8 c + 2 (lane % 4) (+1)
        const int co0 = warp * 16 + (lane >> 2);
        const int col_base = pair_base * NC;
#pragma unroll
        for (int j = 0; j < NPG; ++j) {
          if (j < npairs) {
#pragma unroll
            for (int c = 0; c < NC / 8; ++c) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int co = co0 + 8 * h;
                if (co < p.cout) {
                  float* dst = p.dw + size_t(co) * p.ktot + col_base + j * NC + 8 * c + 2 * (lane & 3);
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(d[j * (NC / 2) + 4 * c + 2 * h]),
                               "f"(d[j * (NC / 2) + 4 * c + 2 * h + 1]) : "memory");
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
      put_split(hi, lo, i, valid ? w[widx] : 0.f);
    }
  }
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
  if (grid > kGridSms * 16) grid = kGridSms * 16;
  stem_input_fold_kernel<<<int(grid), 256, 0, (cudaStream_t)stream>>>(x, n, cin, t, h, w, (bf16s*)hi, (bf16s*)lo);
  return launch_status("sfb_stem_input_fold");
}

extern "C" int sfb_stem_filter_fold(const float* w, float* dw, int32_t cout, int32_t cin, int32_t kt, int32_t kh,
                                    int32_t kw, int32_t pad_w, int32_t kwf, void* hi, void* lo, const float* gmat,
                                    int32_t reverse, void* stream) {
  const int64_t items = int64_t(cout) * kt * kh * kwf * 8;
  int64_t grid = (items + 255) / 256;
  if (grid > kGridSms * 8) grid = kGridSms * 8;
  stem_filter_fold_kernel<<<int(grid), 256, 0, (cudaStream_t)stream>>>(w, dw, cout, cin, kt, kh, kw, pad_w, kwf,
                                                                       (bf16s*)hi, (bf16s*)lo, gmat, reverse);
  return launch_status("sfb_stem_filter_fold");
}

extern "C" int64_t sfb_stem_m_tiles(const sfb_stem_desc* d) {
  return int64_t(d->n) * d->out_t * d->out_h * ((d->out_w + 127) / 128);
}

extern "C" int sfb_stem_fprop(const sfb_stem_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int st_sms = 0, st_smem = 0;
  if (device_limits(&st_sms, &st_smem)) return -1;
  StemParams p;
  memset(&p, 0, sizeof(p));
  int rc = fill_common(p, d);
  if (rc) return rc;
  const int np = d->nsplit == 3 ? 2 : 1;
  p.pps = 64 / (d->kwf * 8);
  p.k_blocks = (p.pairs + p.pps - 1) / p.pps;
  for (int ks = 0; ks < ST_KSTEPS; ++ks) {
    const int per_pair = d->kwf / 2;  // k-steps per pair: taps 2j and 2j+1 of pair qq
    const int qq = ks / per_pair, j = ks % per_pair;
    p.a_kstep[ks] = uint32_t(qq * ST_SEG_STRIDE + 2 * j * 16) >> 4;
  }
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
  {
    typedef void (*KernelFn)(const StemParams);
#define SFB_STEM_FNS(S) {stem_fprop_kernel<S, 16>, stem_fprop_kernel<S, 32>, stem_fprop_kernel<S, 48>, \
                         stem_fprop_kernel<S, 64>}
    static const KernelFn fns[2][ST_BN_MAX / 16] = {SFB_STEM_FNS(1), SFB_STEM_FNS(3)};
#undef SFB_STEM_FNS
    static bool attr[2][ST_BN_MAX / 16] = {};
    const int a = d->nsplit == 3 ? 1 : 0, b = p.BN / 16 - 1;
    if (!attr[a][b]) {
      cudaFuncSetAttribute(fns[a][b], cudaFuncAttributeMaxDynamicSharedMemorySize, st_smem);
      attr[a][b] = true;
    }
    fns[a][b]<<<grid, ST_FPROP_THREADS, smem_bytes, stream>>>(p);
  }
  return launch_status("sfb_stem_fprop", "smem=%u stages=%d", smem_bytes, p.stages);
}

extern "C" int sfb_stem_wgrad(const sfb_stem_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int st_sms = 0, st_smem = 0;
  if (device_limits(&st_sms, &st_smem)) return -1;
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
  // 3 or 4 pairs per CTA, whichever issues fewer padded pairs (4 on a tie: fewer groups re-read dY)
  p.npg = ((p.pairs + 2) / 3) * 3 < ((p.pairs + 3) / 4) * 4 ? 3 : ST_NPG_MAX;
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
  // the epilogue passes one warpgroup's [64 co][npg x kwf*8] fp32 tile through the drained stages
  p.off_bars = std::max(p.stages * p.stage_bytes, uint32_t(64 * p.npg * ncols_pair * 4));
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
  {
    typedef void (*KernelFn)(const StemParams);
#define SFB_STEM_FNS(S) {stem_wgrad_kernel<S, 2, 3>, stem_wgrad_kernel<S, 2, 4>, stem_wgrad_kernel<S, 4, 3>, \
                         stem_wgrad_kernel<S, 4, 4>}
    static const KernelFn fns[2][4] = {SFB_STEM_FNS(1), SFB_STEM_FNS(3)};
#undef SFB_STEM_FNS
    static bool attr[2][4] = {};
    const int a = d->nsplit == 3 ? 1 : 0, b = (d->kwf / 2 - 1) * 2 + (p.npg - 3);
    if (!attr[a][b]) {
      cudaFuncSetAttribute(fns[a][b], cudaFuncAttributeMaxDynamicSharedMemorySize, st_smem);
      attr[a][b] = true;
    }
    fns[a][b]<<<grid, ST_WGRAD_THREADS, smem_bytes, stream>>>(p);
  }
  return launch_status("sfb_stem_wgrad", "grid=%d smem=%u", grid, smem_bytes);
}
