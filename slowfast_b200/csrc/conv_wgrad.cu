// Convolution weight gradient (wgrad) as an implicit GEMM on wgmma:
//
//   dW[co, (tap, ci)] = sum_m dY[m, co] * X_im2col[m, (tap, ci)]        m over n*ot*oh*ow output positions
//
// The reduction runs over output positions, 64 per k-block (one pipeline stage).  A CTA owns one dW tile in one of two
// orientations, whichever pads the layer less (wgrad_plan):
//   * co-rows:    GEMM rows M' = co, columns N' = (tap, ci).  A' = dY boxes [64 positions][64 co], one per 64 rows;
//                 B' = X chunks [64 positions][CK channels], one TMA load per (tap, channel chunk).
//   * transposed: rows M' = (tap, ci), columns N' = co.  A' = the X chunks (64 / CK of them per 64 rows);
//                 B' = dY boxes [64 positions][DK co].
// Both operands are "MN-major" (the reduction index is the slow axis of the tiles as they sit in shared memory), which
// wgmma reads natively for bf16 A and B.  A tile has 64 or 128 rows: with 128 the two MMA warpgroups take 64 rows each;
// with 64 they take the same rows and different halves of every k-block's positions, and the epilogue adds the two.
// The reduction is split across CTAs (split-K) and combined with vector fp32 reductions into dW, which the caller
// zero-fills.  Padding, the position tail and missing rows/columns are zero-filled by the TMA unit.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "runtime.h"

namespace sfb {

constexpr int WG_BLOCK_K = 64;  // output positions per pipeline stage
constexpr int WG_MAX_STAGES = 8;
constexpr int WG_MMA_WARPS = 8;   // two warpgroups
constexpr int WG_THREADS = 32 * (WG_MMA_WARPS + 1);
constexpr int WG_BN_MAX = 128;
constexpr int WG_ROW_BLOCK_BYTES = 8192;  // 64 rows x 64 positions of either operand

struct WgradParams {
  CUtensorMap tmX[2];
  CUtensorMap tmDy[2];
  int oq, op, oz, nb;
  int sw, sh, sd;
  int lw, lh, ld;
  int kw, kh, kd;
  int dw, dh, dd;
  int CK, cpt, n_chunks;
  int x_chunks;            // (tap, channel chunks) per tile
  int dy_boxes, dy_box_w;  // dY boxes per tile and their width in output channels
  int co_tiles, cout, ktot;
  int x_tiled;  // tap-free stride-1 layer: X loaded with tiled TMA
  int k_blocks, splits;
  int stages;
  uint32_t stage_bytes, x_chunk_bytes, x_plane_bytes, dy_box_bytes, dy_plane_bytes;
  uint32_t x_layout, x_lbo, x_sbo, x_kstep;  // MN-major descriptor fields of the X and dY tiles
  uint32_t dy_layout, dy_lbo, dy_sbo, dy_kstep;
  uint32_t acc_pitch;
  uint32_t off_bars;
  float* dw_out;
};

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

template <int NSPLIT, bool TRANS, int MT, int BN>
__global__ void __launch_bounds__(WG_THREADS, 1) conv_wgrad_kernel(const __grid_constant__ WgradParams p) {
  static_assert(BN % 16 == 0 && BN <= WG_BN_MAX && (MT == 64 || MT == 128), "tile: 64 or 128 rows, 16..128 columns");
  constexpr uint32_t NS = NSPLIT == 3 ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + WG_MAX_STAGES;
  float* acc_tile = reinterpret_cast<float*>(smem);  // the epilogue reuses the drained pipeline stages

  const int split = blockIdx.x % p.splits;
  const int tile = blockIdx.x / p.splits;
  const int co_tile = tile % p.co_tiles;
  const int x_tile = tile / p.co_tiles;
  const int kb0 = int(int64_t(split) * p.k_blocks / p.splits);
  const int kb1 = int(int64_t(split + 1) * p.k_blocks / p.splits);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 32 * WG_MMA_WARPS);
    }
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int chunk_base = x_tile * p.x_chunks;        // first (tap, channel-chunk) of this tile
  const int co_base = co_tile * (TRANS ? BN : MT);   // first output channel of this tile
  if (kb1 <= kb0) return;

  if (warp == WG_MMA_WARPS) {
    // ---------------------------------------------------------------- TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&empty[stage], phase ^ 1);
      if (elect_one()) {
        int t = kb * WG_BLOCK_K;
        const int q0 = t % p.oq;
        t /= p.oq;
        const int p0 = t % p.op;
        t /= p.op;
        const int z0 = t % p.oz;
        const int n0 = t / p.oz;
        const int cw = p.lw + q0 * p.sw, ch = p.lh + p0 * p.sh, cd = p.ld + z0 * p.sd;
        mbar_expect_tx(&full[stage], (p.dy_plane_bytes + p.x_plane_bytes) * NS);
        uint8_t* st = smem + size_t(stage) * p.stage_bytes;
        for (int j = 0; j < p.dy_boxes; ++j) {
          tma_load_2d(st + j * p.dy_box_bytes, &p.tmDy[0], &full[stage], co_base + j * p.dy_box_w, kb * WG_BLOCK_K);
          if (NSPLIT == 3)
            tma_load_2d(st + p.dy_plane_bytes + j * p.dy_box_bytes, &p.tmDy[1], &full[stage], co_base + j * p.dy_box_w,
                        kb * WG_BLOCK_K);
        }
        uint8_t* xb = st + p.dy_plane_bytes * NS;
        for (int j = 0; j < p.x_chunks; ++j) {
          const int idx = chunk_base + j;
          int nn = p.nb, c0 = 0;
          uint16_t ow = 0, oh = 0, od = 0;
          if (idx < p.n_chunks) {
            const int tap = idx / p.cpt;
            c0 = (idx - tap * p.cpt) * p.CK;
            const int tw = tap % p.kw;
            const int t2 = tap / p.kw;
            const int th = t2 % p.kh;
            const int td = t2 / p.kh;
            ow = uint16_t(tw * p.dw);
            oh = uint16_t(th * p.dh);
            od = uint16_t(td * p.dd);
            nn = n0;
          }
          if (p.x_tiled) {
            // tap-free stride-1 layer: X is the plain [M][C] matrix -> tiled TMA (im2col mode is limited by the number
            // of per-pixel requests in flight); a chunk past the last row reads as zeros
            const int row0 = idx < p.n_chunks ? kb * WG_BLOCK_K : p.k_blocks * WG_BLOCK_K;
            tma_load_2d(xb + j * p.x_chunk_bytes, &p.tmX[0], &full[stage], c0, row0);
            if (NSPLIT == 3)
              tma_load_2d(xb + p.x_plane_bytes + j * p.x_chunk_bytes, &p.tmX[1], &full[stage], c0, row0);
            continue;
          }
          tma_load_im2col_5d(xb + j * p.x_chunk_bytes, &p.tmX[0], &full[stage], c0, cw, ch, cd, nn, ow, oh, od);
          if (NSPLIT == 3)
            tma_load_im2col_5d(xb + p.x_plane_bytes + j * p.x_chunk_bytes, &p.tmX[1], &full[stage], c0, cw, ch, cd,
                               nn, ow, oh, od);
        }
      }
      __syncwarp();
      if (++stage == p.stages) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }

  // ---------------------------------------------------------------- MMA warpgroups, then the epilogue
  // MT = 128: warpgroup g owns tile rows 64g .. 64g+63 over whole k-blocks.  MT = 64: both own rows 0..63 and g takes
  // the k16 steps 2g, 2g+1 of each k-block.  The tile width is the template's BN, so a k-block's wgmmas are
  // straight-line code issued back to back.
  const int g = warp >> 2;
  constexpr int KSTEPS = MT == 128 ? WG_BLOCK_K / 16 : WG_BLOCK_K / 32;
  const int ks0 = MT == 128 ? 0 : KSTEPS * g;
  const uint32_t a_row_off = MT == 128 ? uint32_t(g) * WG_ROW_BLOCK_BYTES : 0u;
  const uint32_t a_plane = TRANS ? p.x_plane_bytes : p.dy_plane_bytes;
  const uint32_t b_plane = TRANS ? p.dy_plane_bytes : p.x_plane_bytes;
  const uint32_t a_kstep = TRANS ? p.x_kstep : p.dy_kstep;
  const uint32_t b_kstep = TRANS ? p.dy_kstep : p.x_kstep;
  float d[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  int held = -1;  // stage whose MMAs may still be reading shared memory
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full[stage], phase);
    wgmma_fence();
    const uint32_t dy_base = smem_u32(smem + size_t(stage) * p.stage_bytes);
    const uint32_t x_base = dy_base + p.dy_plane_bytes * NS;
    const uint32_t a_base = (TRANS ? x_base : dy_base) + a_row_off + uint32_t(ks0) * a_kstep;
    const uint32_t b_base = (TRANS ? dy_base : x_base) + uint32_t(ks0) * b_kstep;
    // descriptors of the first k-step; a later k-step adds its offset to the start-address field (16-byte units)
    const uint64_t a_hi0 = TRANS ? make_smem_desc(a_base, p.x_lbo, p.x_sbo, p.x_layout)
                                 : make_smem_desc(a_base, p.dy_lbo, p.dy_sbo, p.dy_layout);
    const uint64_t b_hi0 = TRANS ? make_smem_desc(b_base, p.dy_lbo, p.dy_sbo, p.dy_layout)
                                 : make_smem_desc(b_base, p.x_lbo, p.x_sbo, p.x_layout);
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      const uint64_t a_hi = a_hi0 + uint64_t((ks * a_kstep) >> 4);
      const uint64_t b_hi = b_hi0 + uint64_t((ks * b_kstep) >> 4);
      if (NSPLIT == 3) {
        wgmma_m64n<BN, 1, 1>(d, a_hi + (a_plane >> 4), b_hi);
        wgmma_m64n<BN, 1, 1>(d, a_hi, b_hi + (b_plane >> 4));
      }
      wgmma_m64n<BN, 1, 1>(d, a_hi, b_hi);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage can be refilled
    if (held >= 0) mbar_arrive(&empty[held]);
    held = stage;
    if (++stage == p.stages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  named_bar_sync(1, 32 * WG_MMA_WARPS);  // both warpgroups are done reading the stages the accumulator tile overlays
  acc_store<BN>(d, BN, acc_tile + size_t(g) * 64 * p.acc_pitch, int(p.acc_pitch));
  named_bar_sync(1, 32 * WG_MMA_WARPS);

  // epilogue: red.add into dW rows (output channels), 16 consecutive (tap, ci) columns per thread and pass
  constexpr int CO_N = TRANS ? BN : MT;  // output channels of the tile
  constexpr int K_N = TRANS ? MT : BN;   // dW columns of the tile
  const int col_base = chunk_base * p.CK;
  const uint32_t pitch = p.acc_pitch;
  for (int i = threadIdx.x; i < CO_N * (K_N / 16); i += 32 * WG_MMA_WARPS) {
    const int cl = i % CO_N, k0 = (i / CO_N) * 16;
    const int co = co_base + cl;
    if (co >= p.cout || col_base + k0 >= p.ktot) continue;
    float v[16];
    if constexpr (!TRANS) {
      uint32_t u[16];
      acc_ld_x16(acc_tile + size_t(cl) * pitch + k0, u);
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(u[j]);
      if constexpr (MT == 64) {
        acc_ld_x16(acc_tile + size_t(64 + cl) * pitch + k0, u);
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] += __uint_as_float(u[j]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        v[j] = acc_tile[size_t(k0 + j) * pitch + cl];
        if constexpr (MT == 64) v[j] += acc_tile[size_t(64 + k0 + j) * pitch + cl];
      }
    }
    float* dst = p.dw_out + size_t(co) * p.ktot + col_base + k0;
#pragma unroll
    for (int j = 0; j < 16; j += 4) {
      if (col_base + k0 + j < p.ktot)  // ktot is a multiple of 8, so 4-wide groups never straddle the edge
        red_add_v4(dst + j, v[j], v[j + 1], v[j + 2], v[j + 3]);
    }
  }
}

static int pick_ck(int c) {
  if (c % 64 == 0) return 64;
  if (c % 32 == 0) return 32;
  if (c % 16 == 0) return 16;
  return 8;
}

// Descriptor fields of an MN-major operand held as [64 positions][w channels] boxes (w = 8 / 16 / 32 / 64, 128-byte
// rows swizzled by the box width, SWZ_NONE for w = 8), consecutive boxes `box_bytes` apart along M or N.
struct MnMajor {
  uint32_t layout, lbo, sbo, kstep;
};
static MnMajor mn_major(int w, uint32_t box_bytes) {
  switch (w) {
    case 64: return {2, box_bytes, 1024, 16 * 128};
    case 32: return {4, box_bytes, 512, 16 * 64};
    case 16: return {6, box_bytes, 256, 16 * 32};
    default: return {0, 128, box_bytes, 16 * 16};
  }
}
static SwizzleBytes box_swizzle(int w) { return w == 64 ? SWZ_128 : w == 32 ? SWZ_64 : w == 16 ? SWZ_32 : SWZ_NONE; }

// Split-K: s CTAs per tile, each over a contiguous slice of about k_blocks / s k-blocks.  s minimises the modelled time
// waves(tiles * s) x (ceil(k_blocks / s) + 2) with slices of at least 4 k-blocks, where the 2 k-blocks stand for a
// CTA's pipeline fill and epilogue; the smallest s within 3 % of the best is taken, since every slice also adds one
// tile of red.add traffic into dW.
static double wgrad_slice_cost(int tiles, int k_blocks, int num_sms, int s) {
  return double((int64_t(tiles) * s + num_sms - 1) / num_sms) * double((k_blocks + s - 1) / s + 2);
}
static int wgrad_slices(int tiles, int k_blocks, int num_sms) {
  // past a few waves more slices only add fills: the search stops there, which keeps the host cost of a launch small
  const int smax = std::max(1, std::min(k_blocks / 4, 8 * ((num_sms + tiles - 1) / tiles)));
  auto cost = [&](int s) { return wgrad_slice_cost(tiles, k_blocks, num_sms, s); };
  double best = cost(1);
  for (int s = 2; s <= smax; ++s) best = std::min(best, cost(s));
  int s = 1;
  while (cost(s) > 1.03 * best) ++s;
  return s;
}

// The tiling of a tensor-core launch.  Candidates: co-rows and (cout <= 128) transposed, each with 64- or 128-row tiles.
// Co-rows tiles take the (tap, ci) chunks in balanced groups of at most 128 columns; transposed tiles are one column
// tile as wide as cout rounded up to 16 / 32 / 64 / 128.  The candidate with the least modelled time wins:
// the split-K cost above x (MMA work of a tile k-block + a charge for the bytes it loads), so padded rows and columns,
// idle last waves and narrow tiles' lower intensity all count.
static sfb_wgrad_plan wgrad_plan(const sfb_wgrad_desc* d, int num_sms) {
  sfb_wgrad_plan best;
  memset(&best, 0, sizeof(best));
  const int64_t M = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  const int ck = pick_ck(d->c);
  const int n_chunks = d->kt * d->kh * d->kw * (d->c / ck);
  const int k_blocks = int((M + WG_BLOCK_K - 1) / WG_BLOCK_K);
  double best_cost = 0;
  for (int trans = 0; trans < 2; ++trans) {
    if (trans && d->cout > WG_BN_MAX) continue;
    for (int mt = 128; mt >= 64; mt -= 64) {
      sfb_wgrad_plan c;
      memset(&c, 0, sizeof(c));
      c.transposed = trans;
      c.tile_rows = mt;
      c.ck = ck;
      c.k_blocks = k_blocks;
      if (!trans) {
        const int x_tiles = (n_chunks + WG_BN_MAX / ck - 1) / (WG_BN_MAX / ck);
        int ng = (n_chunks + x_tiles - 1) / x_tiles;
        if ((ng * ck) % 16) ng += 1;  // CK = 8 with an odd chunk count: pad with a zero chunk
        c.bn = ng * ck;
        c.tiles = ((d->cout + mt - 1) / mt) * x_tiles;
      } else {
        c.bn = d->cout <= 16 ? 16 : d->cout <= 32 ? 32 : d->cout <= 64 ? 64 : 128;
        c.tiles = (n_chunks * ck + mt - 1) / mt;
      }
      c.slices = wgrad_slices(c.tiles, k_blocks, num_sms);
      c.ctas = c.tiles * c.slices;
      const double cost = wgrad_slice_cost(c.tiles, k_blocks, num_sms, c.slices) *
                          (double(mt) * c.bn + 32.0 * (mt + c.bn));
      if (best.tiles == 0 || cost < best_cost) {
        best = c;
        best_cost = cost;
      }
    }
  }
  return best;
}

static int wgrad_check(const sfb_wgrad_desc* d) {
  if (d->nsplit != 1 && d->nsplit != 3) {
    set_error("sfb_conv_wgrad: nsplit must be 1 or 3");
    return -10;
  }
  if (d->c <= 0 || d->cout <= 0 || d->c % 8 || d->c_pitch % 8 || d->cout % 8 || d->dy_pitch % 8) {
    set_error("sfb_conv_wgrad: c=%d c_pitch=%lld cout=%d dy_pitch=%lld must be positive multiples of 8", d->c,
              (long long)d->c_pitch, d->cout, (long long)d->dy_pitch);
    return -10;
  }
  const int64_t M64 = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  if (M64 <= 0 || M64 > 0x7fffffffLL) {
    set_error("sfb_conv_wgrad: bad M=%lld", (long long)M64);
    return -10;
  }
  return 0;
}

bool wgrad_direct_takes(const sfb_wgrad_desc* d);
int wgrad_direct_try(const sfb_wgrad_desc* d, int sms, cudaStream_t stream, int* rc_out);

typedef void (*WgradKernel)(const WgradParams);
// The shapes wgrad_plan can choose: co-rows with either row count and any BN, transposed with BN = 16 / 32 / 64 / 128.
template <int S, bool T, int MT>
static WgradKernel kernel_for_bn(int bn) {
  switch (bn) {
    case 16: return conv_wgrad_kernel<S, T, MT, 16>;
    case 32: return conv_wgrad_kernel<S, T, MT, 32>;
    case 64: return conv_wgrad_kernel<S, T, MT, 64>;
    case 128: return conv_wgrad_kernel<S, T, MT, 128>;
    default: break;
  }
  if constexpr (!T) {
    switch (bn) {
      case 48: return conv_wgrad_kernel<S, T, MT, 48>;
      case 80: return conv_wgrad_kernel<S, T, MT, 80>;
      case 96: return conv_wgrad_kernel<S, T, MT, 96>;
      case 112: return conv_wgrad_kernel<S, T, MT, 112>;
      default: break;
    }
  }
  return nullptr;
}
template <int S>
static WgradKernel kernel_for_plan(const sfb_wgrad_plan& pl) {
  if (pl.transposed)
    return pl.tile_rows == 128 ? kernel_for_bn<S, true, 128>(pl.bn) : kernel_for_bn<S, true, 64>(pl.bn);
  return pl.tile_rows == 128 ? kernel_for_bn<S, false, 128>(pl.bn) : kernel_for_bn<S, false, 64>(pl.bn);
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_conv_wgrad_plan(const sfb_wgrad_desc* d, int32_t num_sms, sfb_wgrad_plan* out) {
  if (!d || !out || num_sms <= 0) {
    set_error("sfb_conv_wgrad_plan: null descriptor / output or num_sms <= 0");
    return -10;
  }
  const int rc = wgrad_check(d);
  if (rc) return rc;
  if (wgrad_direct_takes(d)) {
    memset(out, 0, sizeof(*out));
    out->direct = 1;
    return 0;
  }
  *out = wgrad_plan(d, num_sms);
  return 0;
}

extern "C" int sfb_conv_wgrad(const sfb_wgrad_desc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int wg_num_sms = 0, wg_smem_optin = 0;
  if (device_limits(&wg_num_sms, &wg_smem_optin)) return -1;
  int rc = wgrad_check(d);
  if (rc) return rc;
  if (!d->x_hi || !d->dy_hi || !d->dw || (d->nsplit == 3 && (!d->x_lo || !d->dy_lo))) {
    set_error("sfb_conv_wgrad: null operand pointer");
    return -10;
  }
  {
    // narrow layers with many positions: fp32 SIMT body (conv_wgrad_direct.cu), same operands and dW layout
    int rc_direct = 0;
    if (sfb::wgrad_direct_try(d, wg_num_sms, stream, &rc_direct)) return rc_direct;
  }
  const sfb_wgrad_plan pl = wgrad_plan(d, wg_num_sms);
  WgradParams p;
  memset(&p, 0, sizeof(p));
  const uint32_t ns = d->nsplit == 3 ? 2 : 1;
  p.oq = d->out_w; p.op = d->out_h; p.oz = d->out_t; p.nb = d->n;
  p.sw = d->str_w; p.sh = d->str_h; p.sd = d->str_t;
  p.lw = d->low_w; p.lh = d->low_h; p.ld = d->low_t;
  p.kw = d->kw; p.kh = d->kh; p.kd = d->kt;
  p.dw = d->dil_w; p.dh = d->dil_h; p.dd = d->dil_t;
  p.CK = pl.ck;
  p.cpt = d->c / p.CK;
  const int taps = d->kt * d->kh * d->kw;
  p.n_chunks = taps * p.cpt;
  p.ktot = taps * d->c;
  p.cout = d->cout;
  p.k_blocks = pl.k_blocks;
  p.splits = pl.slices;
  // dY boxes: 64 output channels per 64 tile rows (co-rows); the widest of 64 / 32 / 16 / 8 that divides cout
  // (transposed, where they make the tile's columns)
  p.dy_box_w = pl.transposed ? pick_ck(d->cout) : 64;
  p.dy_boxes = pl.transposed ? pl.bn / p.dy_box_w : pl.tile_rows / 64;
  p.co_tiles = (d->cout + (pl.transposed ? pl.bn : pl.tile_rows) - 1) / (pl.transposed ? pl.bn : pl.tile_rows);
  p.x_chunks = pl.transposed ? pl.tile_rows / p.CK : pl.bn / p.CK;
  p.x_chunk_bytes = WG_BLOCK_K * p.CK * 2;
  p.x_plane_bytes = p.x_chunks * p.x_chunk_bytes;
  p.dy_box_bytes = WG_BLOCK_K * p.dy_box_w * 2;
  p.dy_plane_bytes = p.dy_boxes * p.dy_box_bytes;
  p.stage_bytes = (p.dy_plane_bytes + p.x_plane_bytes) * ns;
  p.stage_bytes = (p.stage_bytes + 1023) / 1024 * 1024;
  const MnMajor xd = mn_major(p.CK, p.x_chunk_bytes), yd = mn_major(p.dy_box_w, p.dy_box_bytes);
  p.x_layout = xd.layout; p.x_lbo = xd.lbo; p.x_sbo = xd.sbo; p.x_kstep = xd.kstep;
  p.dy_layout = yd.layout; p.dy_lbo = yd.lbo; p.dy_sbo = yd.sbo; p.dy_kstep = yd.kstep;
  p.acc_pitch = uint32_t(pl.bn) + 4;  // 16-byte rows; the 4-float skew spreads the fragment stores over the banks
  const uint32_t acc_bytes = 128u * p.acc_pitch * 4u;
  const uint32_t budget = uint32_t(wg_smem_optin) - 1024 - 256;
  p.stages = std::min<int>(WG_MAX_STAGES, budget / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, (pl.k_blocks + pl.slices - 1) / pl.slices));
  if (p.stages < 2) {
    set_error("sfb_conv_wgrad: not enough shared memory (stage=%u B)", p.stage_bytes);
    return -11;
  }
  p.off_bars = std::max(uint32_t(p.stages) * p.stage_bytes, acc_bytes);
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  if (smem_bytes > uint32_t(wg_smem_optin)) {
    set_error("sfb_conv_wgrad: %u bytes of shared memory needed, %d available", smem_bytes, wg_smem_optin);
    return -11;
  }
  p.dw_out = d->dw;

  const int lower[3] = {d->low_w, d->low_h, d->low_t};
  const int strd[3] = {d->str_w, d->str_h, d->str_t};
  const int upper[3] = {d->low_w + (d->out_w - 1) * d->str_w + 1 - d->w, d->low_h + (d->out_h - 1) * d->str_h + 1 - d->h,
                        d->low_t + (d->out_t - 1) * d->str_t + 1 - d->d};
  const int64_t M = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  p.x_tiled = (taps == 1 && d->str_w == 1 && d->str_h == 1 && d->str_t == 1 && d->low_w == 0 && d->low_h == 0 &&
               d->low_t == 0 && d->out_w == d->w && d->out_h == d->h && d->out_t == d->d) ? 1 : 0;
  for (uint32_t pn = 0; pn < ns; ++pn) {
    if (p.x_tiled)
      rc = make_tmap_2d_bf16(&p.tmX[pn], pn ? d->x_lo : d->x_hi, uint64_t(M), uint64_t(d->c), uint64_t(d->c_pitch),
                             WG_BLOCK_K, p.CK, box_swizzle(p.CK));
    else
      rc = make_tmap_im2col_bf16(&p.tmX[pn], pn ? d->x_lo : d->x_hi, d->n, d->d, d->h, d->w, d->c, d->c_pitch, lower,
                                 upper, strd, p.CK, WG_BLOCK_K, box_swizzle(p.CK));
    if (rc) return rc;
    rc = make_tmap_2d_bf16(&p.tmDy[pn], pn ? d->dy_lo : d->dy_hi, uint64_t(M), uint64_t(d->cout),
                           uint64_t(d->dy_pitch), WG_BLOCK_K, p.dy_box_w, box_swizzle(p.dy_box_w));
    if (rc) return rc;
  }
  const WgradKernel fn = d->nsplit == 3 ? kernel_for_plan<3>(pl) : kernel_for_plan<1>(pl);
  if (!fn) {
    set_error("sfb_conv_wgrad: no kernel for the tile (transposed=%d rows=%d bn=%d)", pl.transposed, pl.tile_rows,
              pl.bn);
    return -11;
  }
  static WgradKernel configured[64];
  static int n_configured = 0;
  if (std::find(configured, configured + n_configured, fn) == configured + n_configured) {
    cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_optin);
    configured[n_configured++] = fn;
  }
  fn<<<pl.ctas, WG_THREADS, smem_bytes, stream>>>(p);
  return launch_status("sfb_conv_wgrad", "grid=%d smem=%u transposed=%d rows=%d bn=%d", pl.ctas, smem_bytes,
                       pl.transposed, pl.tile_rows, pl.bn);
}
