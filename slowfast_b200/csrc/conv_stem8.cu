// The fast pathway's stem (stem_helper.py:182 ResNetBasicStem with dim_out = 8: Conv3d 3 -> 8, [kt,7,7], stride (1,2,2),
// pad (kt/2,3,3)) as a "Toeplitz" implicit GEMM on wgmma.
//
// Why: with 8 output channels the W-shift kernels of conv_stem.cu issue 128 x 16 x 16 MMAs whose cost is the 4 KB
// shared-memory read of the A tile, not the math (measured 1.87 ms fprop, 2.1 ms wgrad per SlowFast step = 11 % of it).
// Here one GEMM row is a GROUP OF 8 CONSECUTIVE OUTPUT PIXELS of an output row:
//
//   D[(n,ot,oh,m), (j,co)] = sum_{kt,kh} sum_{g<12,s<8} A_{kt,kh}[(n,ot,oh,m), g*8+s] * Z_{kt,kh}[(j,co), g*8+s]
//
//   A row  = the 11 (+1 pad) folded pixel pairs the 8 outputs touch: A[.., g*8+s] = X'[.., pair' 8m+g, slot s]
//            (X' = clip with W folded by the stride: slot s = parity*cin + c, pair' = pair + 2 so that tap 0 is pair' 0)
//   Z      = the folded filter, Toeplitz-expanded over the 8 pixels of the group: Z[(j,co), g] = Wf[co][kw' = g - j]
//
// N grows from 8 to 64 for the same A bytes: 6 MMAs of 128 x 64 x 16 per (kt,kh) and 1024 outputs instead of 2 per 112.
// Neither expansion is materialised:
//   * X' is stored de-interleaved, R_j[m] = X'[pair' 8m + j] (8 arrays of 16-byte granules per input row), so that the
//     K chunk g of all rows m is the dense array R_{g%8} (shifted one granule for g >= 8): a no-swizzle K-major
//     operand whose "leading byte offset" is the array stride - the same descriptor trick as the W-shift kernels.
//   * Z is ONE zero-flanked copy of the folded filter per (kt,kh): with the pixel order reversed (j' = 7 - j) the core
//     matrix (j', g) is granule g + j' of that copy, i.e. LBO = SBO = 128 bytes (overlapping operand rows).
// Input rows are split by parity (h = 2*h2 + par) so that the 7 H taps of 8 consecutive output rows are slot offsets
// into two resident groups of 11 input rows: one stage = (8 output rows, input frame t) is loaded once per kt and
// feeds 7 x 6 MMAs (x3 split products).
//
// wgrad runs the same operands with the reduction over the row index: dZ[(kt sel, j, co), g*8+s] for the 4 (or 3) H taps
// of one parity class in registers (2 x 64 rows: two T taps share one pass over the clip), then
// dWf[co][kt][kh][kw'][s] = sum_j dZ[(j,co), (j + kw')*8 + s] is folded into the W-shift gradient matrix by atomics.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "tmap.h"

namespace sfb {

constexpr int T8_ROWS = 8;     // output rows per tile
constexpr int T8_SLOTS = 11;   // resident input rows per parity class: 8 + 3
constexpr int T8_KSTEPS = 6;   // 12 granules of 8 slots = 96 K elements per (kt, kh)
constexpr int T8_FPROP_THREADS = 32 * (8 + 1);    // two MMA warpgroups (rows 0..63 / 64..127) + producer warp
constexpr int T8_WGRAD_THREADS = 32 * (16 + 1);   // four MMA warpgroups (row half x tap pair) + producer warp

__device__ __forceinline__ void t8_tma_5d(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c0, int32_t c1,
                                          int32_t c2, int32_t c3, int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

struct Stem8Params {
  CUtensorMap tmX[2];   // X'' [120.. el, j 8, h2, 2T, N]
  CUtensorMap tmB[2];   // fprop: Z planes [kt*G rows, 64 el];  wgrad: dY [64 el, OW/8, OH, OT, N]
  int N, T, OT, OH, OW, MR;   // MR = OW/8 + 1 granule rows per input row and array
  int KT, pt, bands, tiles;
  uint32_t ab;            // bytes of one R_j array in shared memory (11 slots, 128-byte multiple)
  uint32_t a_plane, a_bytes, b_plane, stage_bytes, off_red, off_bars;
  uint32_t zg;            // granules per kt in Z (7*12 + 8)
  float* out;
  float* stats;
  int m_tiles;
  // wgrad
  int splits0, splits1;   // CTAs per (kt group) for class 0 (kh odd: 3 taps) and class 1 (kh even: 4 taps)
  int kt_groups, steps;
  float* dwm;
  int kfold;
};

// ------------------------------------------------------------------------------------------------ fprop
template <int NSPLIT>
__global__ void __launch_bounds__(T8_FPROP_THREADS, 1) stem8_fprop_kernel(const __grid_constant__ Stem8Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + 2;
  constexpr uint32_t NP = NSPLIT == 3 ? 2u : 1u;
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 256);
    }
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp == 8) {
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
      const int band = tile % p.bands;
      int r = tile / p.bands;
      const int ot = r % p.OT;
      const int n = r / p.OT;
      const int oh0 = band * T8_ROWS;
      const int kt_lo = max(0, p.pt - ot), kt_hi = min(p.KT, p.T + p.pt - ot);
      for (int kt = kt_lo; kt < kt_hi; ++kt) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          const int tin = ot + kt - p.pt;
          mbar_expect_tx(&full[stage], NP * (16u * uint32_t(T8_SLOTS * p.MR * 16) + p.b_plane));
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          for (uint32_t pl = 0; pl < NP; ++pl) {
            for (int cls = 0; cls < 2; ++cls) {
              // class 0: even input rows (kh = 1,3,5), first resident row h2 = oh0 - 1; class 1: odd rows (kh = 0,2,4,6), oh0 - 2
              const int h2 = oh0 - 1 - cls;
              for (int j = 0; j < 8; ++j)
                t8_tma_5d(st + pl * p.a_plane + (cls * 8 + j) * p.ab, &p.tmX[pl], &full[stage], 0, j, h2, 2 * tin + cls, n);
            }
            tma_load_2d(st + p.a_bytes + pl * p.b_plane, &p.tmB[pl], &full[stage], 0, kt * int(p.zg));
          }
        }
        __syncwarp();
        if (++stage == 2) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // MMA warpgroup g: GEMM rows 64g .. 64g+63 (8 more 128-byte row groups into each array); its warps then store
    // straight from the fragments: thread = rows 16w + lane/4 (+8), columns 8c + 2(lane%4) (+1) = pixel 7-c, channels
    const int g = warp >> 2;
    float* red = reinterpret_cast<float*>(smem + p.off_red);   // [2][8 warps][16]
    float d[32];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x, ++it) {
      const int band = tile % p.bands;
      const int rowg = tile / p.bands;            // (n, ot) flattened
      const int ot = rowg % p.OT;
      const int kt_lo = max(0, p.pt - ot), kt_hi = min(p.KT, p.T + p.pt - ot);
      int held = -1;
      for (int kt = kt_lo; kt < kt_hi; ++kt) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + uint32_t(g) * 1024u;
        const uint32_t b_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + p.a_bytes;
        for (int kh = 0; kh < 7; ++kh) {
          const int cls = (kh & 1) ^ 1;             // kh even -> odd input rows (class 1)
          const int so = cls ? (kh >> 1) : ((kh - 1) >> 1);   // slot of output row 0's tap
#pragma unroll
          for (int i = 0; i < T8_KSTEPS; ++i) {
            const int arr = i < 4 ? 2 * i : 2 * i - 8;
            const int shift = i < 4 ? 0 : 1;
            const uint32_t aa = a_base + uint32_t(cls * 8 + arr) * p.ab + uint32_t(so * p.MR + shift) * 16u;
            const uint32_t bb = b_base + uint32_t(kh * 12 + 1 + 2 * i) * 128u;
            const uint64_t a_hi = make_smem_desc(aa, p.ab, 128, 0);
            const uint64_t b_hi = make_smem_desc(bb, 128, 128, 0);
            const uint32_t acc_flag = (kt != kt_lo || kh != 0 || i != 0) ? 1u : 0u;
            if (NSPLIT == 3) {
              const uint64_t a_lo = make_smem_desc(aa + p.a_plane, p.ab, 128, 0);
              const uint64_t b_lo = make_smem_desc(bb + p.b_plane, 128, 128, 0);
              wgmma_m64n64<0, 0>(d, a_lo, b_hi, acc_flag);
              wgmma_m64n64<0, 0>(d, a_hi, b_lo, 1u);
              wgmma_m64n64<0, 0>(d, a_hi, b_hi, 1u);
            } else {
              wgmma_m64n64<0, 0>(d, a_hi, b_hi, acc_flag);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0) mbar_arrive(&empty[held]);
        held = stage;
        if (++stage == 2) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (held >= 0) mbar_arrive(&empty[held]);
      const int cp = 2 * (lane & 3);   // channel pair of this thread
      float s[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rr = g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        const int ohl = rr / p.MR, m = rr - ohl * p.MR;
        if (ohl < T8_ROWS && m < p.MR - 1) {
          float* dst = p.out + ((static_cast<long long>(rowg) * p.OH + band * T8_ROWS + ohl) * p.OW + 8 * m) * 8 + cp;
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            // column c*8 + co holds pixel 8m + 7 - c, channel co
            const float y0 = d[4 * c + 2 * h], y1 = d[4 * c + 2 * h + 1];
            *reinterpret_cast<float2*>(dst + (7 - c) * 8) = make_float2(y0, y1);
            s[0] += y0; s[1] += y1;
            s2[0] = fmaf(y0, y0, s2[0]); s2[1] = fmaf(y1, y1, s2[1]);
          }
        }
      }
      if (p.stats != nullptr) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
#pragma unroll
          for (int o = 4; o <= 16; o <<= 1) {
            s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
            s2[c] += __shfl_xor_sync(0xffffffffu, s2[c], o);
          }
        }
        float* rw = red + ((it & 1) * 8 + warp) * 16;
        if (lane < 4) {
          rw[cp] = s[0]; rw[cp + 1] = s[1];
          rw[8 + cp] = s2[0]; rw[8 + cp + 1] = s2[1];
        }
        named_bar_sync(1, 256);
        if (warp == 0 && lane < 16) {
          const float* rb = red + (it & 1) * 8 * 16;
          float tot = 0.f;
#pragma unroll
          for (int w = 0; w < 8; ++w) tot += rb[w * 16 + lane];
          // lane < 8: sum of channel lane; lane >= 8: sum of squares of channel lane - 8   (stats = [2][cout][m_tiles])
          p.stats[size_t(lane) * p.m_tiles + tile] = tot;
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------ wgrad
__device__ __forceinline__ void t8_red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

// CTA = (parity class, group of two T taps, split of the (n, input frame, band) steps).  Stage = the class's 8 arrays of
// the input band + the dY row groups of the two output frames the taps pair this input frame with.
template <int NSPLIT>
__global__ void __launch_bounds__(T8_WGRAD_THREADS, 1) stem8_wgrad_kernel(const __grid_constant__ Stem8Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + 2;
  constexpr uint32_t NP = NSPLIT == 3 ? 2u : 1u;
  constexpr uint32_t DY_TILE = 16384;   // 128 rows x 128 bytes (120 written by the TMA, the rest stay zero)

  // decode the CTA's job
  const int per0 = p.kt_groups * p.splits0;
  int cls, ktg, split, nsplits;
  if (int(blockIdx.x) < per0) {
    cls = 0;
    ktg = blockIdx.x / p.splits0;
    split = blockIdx.x - ktg * p.splits0;
    nsplits = p.splits0;
  } else {
    const int b = blockIdx.x - per0;
    cls = 1;
    ktg = b / p.splits1;
    split = b - ktg * p.splits1;
    nsplits = p.splits1;
  }
  const int ntaps = cls ? 4 : 3;
  const int kta = 2 * ktg, ktb = 2 * ktg + 1;
  const bool has_b = ktb < p.KT;
  const int per = (p.steps + nsplits - 1) / nsplits;
  const int s0 = split * per, s1 = min(p.steps, s0 + per);

  // zero the whole operand area once: rows the TMA never writes (dY rows 120..127, array tails) must be finite
  {
    uint4* z = reinterpret_cast<uint4*>(smem);
    const uint32_t n16 = (2u * p.stage_bytes) / 16u;
    for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 512);
    }
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t x_bytes = NP * 8u * p.ab;       // class arrays, both planes

  if (s1 > s0) {
    if (warp == 16) {
      int stage = 0;
      uint32_t phase = 0;
      for (int step = s0; step < s1; ++step) {
        const int band = step % p.bands;
        int r = step / p.bands;
        const int tin = r % p.T;
        const int n = r / p.T;
        const int oh0 = band * T8_ROWS;
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          const uint32_t dyb = uint32_t(T8_ROWS * p.MR) * 128u;
          mbar_expect_tx(&full[stage], NP * (8u * uint32_t(T8_SLOTS * p.MR * 16) + (has_b ? 2u : 1u) * dyb));
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          const int h2 = oh0 - 1 - cls;
          for (uint32_t pl = 0; pl < NP; ++pl) {
            for (int j = 0; j < 8; ++j)
              t8_tma_5d(st + (pl * 8 + j) * p.ab, &p.tmX[pl], &full[stage], 0, j, h2, 2 * tin + cls, n);
            uint8_t* dyd = st + x_bytes + pl * 2 * DY_TILE;
            t8_tma_5d(dyd, &p.tmB[pl], &full[stage], 0, 0, oh0, tin - kta + p.pt, n);
            if (has_b) t8_tma_5d(dyd + DY_TILE, &p.tmB[pl], &full[stage], 0, 0, oh0, tin - ktb + p.pt, n);
          }
        }
        __syncwarp();
        if (++stage == 2) {
          stage = 0;
          phase ^= 1;
        }
      }
    } else {
      // MMA warpgroup (g, th): 64-row half g (T tap kta / ktb) and H taps tq = 2 th, 2 th + 1; per tap a 64-column
      // accumulator (granules 0..7, B0) and a 32-column one (granules 8..11, B1)
      const int wg = warp >> 2, g = wg & 1, th = wg >> 1;
      float d0[2][32], d1[2][16];
      int stage = 0;
      uint32_t phase = 0;
      int held = -1;
      for (int step = s0; step < s1; ++step) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t x_base = smem_u32(smem + size_t(stage) * p.stage_bytes);
        const uint32_t lbo_a = has_b ? DY_TILE : 0u;       // second 64-row atom = the other T tap's dY (or an alias)
        const uint32_t dy_base = x_base + x_bytes + uint32_t(g) * lbo_a;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int tq = 2 * th + u;   // class 1: kh = 2 tq, slot offset tq; class 0: kh = 2 tq + 1, slot offset tq
          if (tq < ntaps) {
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
              const uint32_t xa = x_base + uint32_t(tq * p.MR) * 16u + uint32_t(ks) * 256u;
              const uint64_t a_hi = make_smem_desc(dy_base + ks * 2048, lbo_a, 1024, 2);
              const uint64_t b0_hi = make_smem_desc(xa, 128, p.ab, 0);
              const uint64_t b1_hi = make_smem_desc(xa + 16u, 128, p.ab, 0);
              const uint32_t acc_flag = (step != s0 || ks != 0) ? 1u : 0u;
              if (NSPLIT == 3) {
                const uint64_t a_lo = make_smem_desc(dy_base + 2 * DY_TILE + ks * 2048, lbo_a, 1024, 2);
                const uint64_t b0_lo = make_smem_desc(xa + 8u * p.ab, 128, p.ab, 0);
                const uint64_t b1_lo = make_smem_desc(xa + 8u * p.ab + 16u, 128, p.ab, 0);
                wgmma_m64n64<1, 1>(d0[u], a_lo, b0_hi, acc_flag);
                wgmma_m64n64<1, 1>(d0[u], a_hi, b0_lo, 1u);
                wgmma_m64n64<1, 1>(d0[u], a_hi, b0_hi, 1u);
                wgmma_m64n32<1, 1>(d1[u], a_lo, b1_hi, acc_flag);
                wgmma_m64n32<1, 1>(d1[u], a_hi, b1_lo, 1u);
                wgmma_m64n32<1, 1>(d1[u], a_hi, b1_hi, 1u);
              } else {
                wgmma_m64n64<1, 1>(d0[u], a_hi, b0_hi, acc_flag);
                wgmma_m64n32<1, 1>(d1[u], a_hi, b1_hi, acc_flag);
              }
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0) mbar_arrive(&empty[held]);
        held = stage;
        if (++stage == 2) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      // fragments -> dWf: row mu = (j, co), column granule gi = kw' + j, slots 2 (lane % 4) (+1)
      const int kt = g ? ktb : kta;
      if (kt < p.KT) {
        const int sl = 2 * (lane & 3);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int tq = 2 * th + u;
          if (tq < ntaps) {
            const int kh = cls ? 2 * tq : 2 * tq + 1;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int mu = (warp & 3) * 16 + (lane >> 2) + 8 * h;
              const int j = mu >> 3, co = mu & 7;
              float* dst = p.dwm + size_t(co) * p.kfold + size_t((kt * 7 + kh) * 4) * 8 + sl;
#pragma unroll
              for (int gi = 0; gi < 12; ++gi) {
                const int kwp = gi - j;   // folded W tap this granule is for pixel j of the group
                if (kwp >= 0 && kwp < 4) {
                  const float y0 = gi < 8 ? d0[u][4 * gi + 2 * h] : d1[u][4 * (gi - 8) + 2 * h];
                  const float y1 = gi < 8 ? d0[u][4 * gi + 2 * h + 1] : d1[u][4 * (gi - 8) + 2 * h + 1];
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + kwp * 8), "f"(y0), "f"(y1) : "memory");
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
// NCTHW fp32 clip -> X''[n][2t + (h&1)][h/2][j][m][8] split planes: granule (j, m) = pixel pair' 8m + j (pair' = pair + 2),
// slots = parity*cin + c; pads and out-of-row pairs are zero.
__global__ void stem8_input_fold_kernel(const float* __restrict__ x, int n, int cin, int t, int h, int w, int mr,
                                        __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int w2 = w / 2, gpr = 8 * mr, h2n = h / 2;
  const int64_t thw = int64_t(t) * h * w;
  const int64_t items = int64_t(n) * t * h * gpr;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int pp = int(i % gpr);
    const int64_t rest = i / gpr;  // (n*t + tt)*h + hh
    const int64_t nt = rest / h;
    const int hh = int(rest - nt * h);
    const int64_t b = nt / t;
    const int tt = int(nt - b * t);
    const int pair = pp - 2;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    if (pair >= 0 && pair < w2)
      for (int par = 0; par < 2; ++par)
        for (int c = 0; c < cin; ++c)
          v[par * cin + c] = x[(b * cin + c) * thw + (int64_t(tt) * h + hh) * w + 2 * pair + par];
    alignas(16) __nv_bfloat16 hv[8], lv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      hv[j] = __float2bfloat16_rn(v[j]);
      lv[j] = __float2bfloat16_rn(v[j] - __bfloat162float(hv[j]));
    }
    const int64_t row = ((b * 2 * t + 2 * tt + (hh & 1)) * h2n + (hh >> 1));
    const int64_t g = (row * 8 + (pp & 7)) * mr + (pp >> 3);
    *reinterpret_cast<uint4*>(hi + g * 8) = *reinterpret_cast<const uint4*>(hv);
    if (lo) *reinterpret_cast<uint4*>(lo + g * 8) = *reinterpret_cast<const uint4*>(lv);
  }
}

// weight [8][cin][kt][7][7] -> Z planes [kt][7*12 + 8 granules][8 co][8 slots]: granule kh*12 + 8 + kw' holds the folded tap
// kw' (slot (parity, c) = original tap kw = 2 kw' + parity - 1), all other granules are zero.
__global__ void stem8_filter_fold_kernel(const float* __restrict__ w, int cin, int kt, int zg,
                                         __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int items = kt * zg * 64;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < items; i += gridDim.x * blockDim.x) {
    const int slot = i & 7, co = (i >> 3) & 7;
    const int g = (i >> 6) % zg, it = (i >> 6) / zg;
    float v = 0.f;
    const int gi = g - 8;
    if (gi >= 0 && (gi % 12) < 4 && gi / 12 < 7 && slot < 2 * cin) {
      const int kh = gi / 12, kwp = gi % 12;
      const int par = slot / cin, c = slot - par * cin;
      const int tap = 2 * kwp + par - 1;
      if (tap >= 0 && tap < 7) v = w[(((int64_t(co) * cin + c) * kt + it) * 7 + kh) * 7 + tap];
    }
    const __nv_bfloat16 hb = __float2bfloat16_rn(v);
    hi[i] = hb;
    if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(hb));
  }
}

typedef CUresult (*EncodeTiledFn8)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn8 t8_encode() {
  static EncodeTiledFn8 fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn8>(f);
  }
  return fn;
}
static int t8_tmap5(CUtensorMap* out, const void* base, const cuuint64_t dims[5], const cuuint64_t strides[4],
                    const cuuint32_t box[5], bool swz128, const char* what) {
  EncodeTiledFn8 fn = t8_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point unavailable");
    return -1;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(%s) failed (%d)", what, (int)r);
    return -2;
  }
  return 0;
}

static int t8_sms = 0, t8_smem = 0;
static int t8_props() {
  if (t8_sms) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("cudaGetDevice failed: no CUDA device");
    return -1;
  }
  cudaDeviceGetAttribute(&t8_sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&t8_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return 0;
}

static bool t8_geometry_ok(const sfb_stem_desc* d) {
  return d->cout == 8 && d->kh == 7 && d->kwf == 4 && d->str_t == 1 && d->str_h == 2 && d->pad_h == 3 && d->pad_wf == 2 &&
         d->kt >= 1 && d->kt <= 8 && d->out_w % 8 == 0 && d->out_w >= 8 && d->out_w <= 120 && d->out_h % T8_ROWS == 0 &&
         d->h == 2 * d->out_h && d->wf == 8 * (d->out_w / 8 + 1) && d->out_t == d->t + 2 * d->pad_t - d->kt + 1;
}

static int t8_fill(Stem8Params& p, const sfb_stem_desc* d) {
  if (!t8_geometry_ok(d)) {
    set_error("sfb_stem8: unsupported geometry (cout=%d k=%dx%dx(%d folded) out=%dx%dx%d wf=%d)", d->cout, d->kt, d->kh,
              d->kwf, d->out_t, d->out_h, d->out_w, d->wf);
    return -10;
  }
  p.N = d->n; p.T = d->t; p.OT = d->out_t; p.OH = d->out_h; p.OW = d->out_w;
  p.MR = d->out_w / 8 + 1;
  p.KT = d->kt; p.pt = d->pad_t;
  p.bands = d->out_h / T8_ROWS;
  p.tiles = d->n * d->out_t * p.bands;
  p.m_tiles = p.tiles;
  p.ab = (uint32_t(T8_SLOTS * p.MR * 16) + 127u) / 128u * 128u;
  p.zg = 7 * 12 + 8;
  p.kfold = d->kt * 7 * 4 * 8;
  return 0;
}

static int t8_xmaps(Stem8Params& p, const sfb_stem_desc* d, int np) {
  const cuuint64_t row = 16ull * 8 * p.MR;     // bytes of one folded input row
  cuuint64_t dims[5] = {(cuuint64_t)(8 * p.MR), 8, (cuuint64_t)(d->h / 2), (cuuint64_t)(2 * d->t), (cuuint64_t)d->n};
  cuuint64_t strides[4] = {16ull * p.MR, row, row * (d->h / 2), row * (d->h / 2) * 2 * d->t};
  cuuint32_t box[5] = {(cuuint32_t)(8 * p.MR), 1, (cuuint32_t)T8_SLOTS, 1, 1};
  for (int pl = 0; pl < np; ++pl) {
    int rc = t8_tmap5(&p.tmX[pl], pl ? d->x_lo : d->x_hi, dims, strides, box, false, "stem8 x");
    if (rc) return rc;
  }
  return 0;
}

}  // namespace sfb

using namespace sfb;
typedef __nv_bfloat16 bf16t;

extern "C" int sfb_stem8_supported(const sfb_stem_desc* d) { return t8_geometry_ok(d) ? 1 : 0; }

extern "C" int64_t sfb_stem8_m_tiles(const sfb_stem_desc* d) {
  return int64_t(d->n) * d->out_t * (d->out_h / T8_ROWS);
}

extern "C" int sfb_stem8_input_fold(const float* x, int32_t n, int32_t cin, int32_t t, int32_t h, int32_t w, void* hi,
                                    void* lo, void* stream) {
  if (cin < 1 || cin > 4 || (w % 16) || (h & 1)) {
    set_error("sfb_stem8_input_fold: cin=%d must be <= 4, w=%d a multiple of 16, h=%d even", cin, w, h);
    return -10;
  }
  const int mr = w / 16 + 1;
  const int64_t items = int64_t(n) * t * h * 8 * mr;
  int64_t grid = (items + 255) / 256;
  if (grid > 148 * 16) grid = 148 * 16;
  stem8_input_fold_kernel<<<int(grid), 256, 0, (cudaStream_t)stream>>>(x, n, cin, t, h, w, mr, (bf16t*)hi, (bf16t*)lo);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem8_input_fold launch failed: %s", cudaGetErrorString(e));
    return -20;
  }
  return 0;
}

extern "C" int sfb_stem8_filter_fold(const float* w, int32_t cin, int32_t kt, void* hi, void* lo, void* stream) {
  const int zg = 7 * 12 + 8;
  const int items = kt * zg * 64;
  stem8_filter_fold_kernel<<<(items + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, cin, kt, zg, (bf16t*)hi, (bf16t*)lo);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem8_filter_fold launch failed: %s", cudaGetErrorString(e));
    return -20;
  }
  return 0;
}

extern "C" int sfb_stem8_fprop(const sfb_stem_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (t8_props()) return -1;
  Stem8Params p;
  memset(&p, 0, sizeof(p));
  int rc = t8_fill(p, d);
  if (rc) return rc;
  const int np = d->nsplit == 3 ? 2 : 1;
  p.a_plane = 16u * p.ab;
  p.a_bytes = np * p.a_plane;
  p.b_plane = p.zg * 128u;
  p.stage_bytes = (p.a_bytes + np * p.b_plane + 1023u) / 1024u * 1024u;
  p.off_red = 2 * p.stage_bytes;
  p.off_bars = p.off_red + 2 * 8 * 16 * 4;
  const uint32_t smem_bytes = p.off_bars + 128 + 1024;
  if (smem_bytes > uint32_t(t8_smem)) {
    set_error("sfb_stem8_fprop: %u bytes of shared memory needed, %d available", smem_bytes, t8_smem);
    return -11;
  }
  p.out = d->out;
  p.stats = d->stats;
  rc = t8_xmaps(p, d, np);
  if (rc) return rc;
  for (int pl = 0; pl < np; ++pl) {
    rc = make_tmap_2d_bf16(&p.tmB[pl], pl ? d->f_lo : d->f_hi, uint64_t(d->kt) * p.zg, 64, 64, p.zg, 64, SWZ_NONE);
    if (rc) return rc;
  }
  const int grid = std::min(p.tiles, t8_sms);
  if (d->nsplit == 3) {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem8_fprop_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, t8_smem); a = true; }
    stem8_fprop_kernel<3><<<grid, T8_FPROP_THREADS, smem_bytes, stream>>>(p);
  } else {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem8_fprop_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, t8_smem); a = true; }
    stem8_fprop_kernel<1><<<grid, T8_FPROP_THREADS, smem_bytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem8_fprop launch failed: %s (smem=%u)", cudaGetErrorString(e), smem_bytes);
    return -20;
  }
  return 0;
}

extern "C" int sfb_stem8_wgrad(const sfb_stem_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (t8_props()) return -1;
  Stem8Params p;
  memset(&p, 0, sizeof(p));
  int rc = t8_fill(p, d);
  if (rc) return rc;
  const int np = d->nsplit == 3 ? 2 : 1;
  p.stage_bytes = (np * 8u * p.ab + np * 2u * 16384u + 1023u) / 1024u * 1024u;
  if ((np * 8u * p.ab) % 1024u) {
    set_error("sfb_stem8_wgrad: operand arrays (%u bytes) do not keep the dY tiles 1024-byte aligned", np * 8u * p.ab);
    return -11;
  }
  p.off_bars = 2 * p.stage_bytes;
  const uint32_t smem_bytes = p.off_bars + 128 + 1024;
  if (smem_bytes > uint32_t(t8_smem)) {
    set_error("sfb_stem8_wgrad: %u bytes of shared memory needed, %d available", smem_bytes, t8_smem);
    return -11;
  }
  p.kt_groups = (d->kt + 1) / 2;
  p.steps = d->n * d->t * p.bands;
  // CTAs: class 1 carries 4 H taps per step, class 0 three -> split the machine 4 : 3
  const int per_group = std::max(2, t8_sms / p.kt_groups);
  p.splits1 = std::max(1, std::min(p.steps, (per_group * 4 + 3) / 7));
  p.splits0 = std::max(1, std::min(p.steps, per_group - p.splits1));
  p.dwm = d->dwm;
  rc = t8_xmaps(p, d, np);
  if (rc) return rc;
  {
    // dY [n, ot, oh, ow, 8] bf16 seen as [64 el = 8 pixels x 8 co, OW/8, OH, OT, N]; box = 8 rows x MR groups (the last one is
    // out of bounds -> zero) x 64 el, 128-byte swizzle
    const cuuint64_t rowb = 16ull * d->out_w;
    cuuint64_t dims[5] = {64, (cuuint64_t)(d->out_w / 8), (cuuint64_t)d->out_h, (cuuint64_t)d->out_t, (cuuint64_t)d->n};
    cuuint64_t strides[4] = {128, rowb, rowb * d->out_h, rowb * d->out_h * d->out_t};
    cuuint32_t box[5] = {64, (cuuint32_t)p.MR, (cuuint32_t)T8_ROWS, 1, 1};
    for (int pl = 0; pl < np; ++pl) {
      rc = t8_tmap5(&p.tmB[pl], pl ? d->dy_lo : d->dy_hi, dims, strides, box, true, "stem8 dy");
      if (rc) return rc;
    }
  }
  const int grid = p.kt_groups * (p.splits0 + p.splits1);
  if (d->nsplit == 3) {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem8_wgrad_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, t8_smem); a = true; }
    stem8_wgrad_kernel<3><<<grid, T8_WGRAD_THREADS, smem_bytes, stream>>>(p);
  } else {
    static bool a = false;
    if (!a) { cudaFuncSetAttribute(stem8_wgrad_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, t8_smem); a = true; }
    stem8_wgrad_kernel<1><<<grid, T8_WGRAD_THREADS, smem_bytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_stem8_wgrad launch failed: %s (grid=%d smem=%u)", cudaGetErrorString(e), grid, smem_bytes);
    return -20;
  }
  return 0;
}
