// Implicit-GEMM 3-D convolution for sm_90a.
//
//   GEMM view: D[M = n*ot*oh*ow, N = cout] = A_im2col[M, K = taps*c] * B[N, K]^T
//
// * A is never materialised: each K chunk (one filter tap x CK channels) of a 128-pixel tile is fetched by ONE
//   TMA im2col load straight into (swizzled) shared memory; padding and the M tail are zero-filled by the unit.
// * B (filter matrix, K-major) arrives through a tiled TMA load (128B swizzle).
// * wgmma (64 x BN x 16 per warpgroup, bf16 -> fp32) accumulates in registers; in parity mode every product is the
//   3-term split  A_lo*B_hi + A_hi*B_lo + A_hi*B_hi.
// * The tile width BN is a template parameter and a k-block is always KSTEPS k16 steps, so the wgmmas of a k-block are
//   issued back to back (a runtime width switch makes ptxas serialise them).
// * Split-K (conv_ksplit): a grid that fills too little of its last wave gives each tile to s CTAs, each over a slice
//   of the k-blocks; the partial tiles meet in the output with red.global.add.
// * Persistent CTAs, warp-specialised: warps 0..7 = two MMA warpgroups (rows 0..63 / 64..127 of the tile),
//   warp 8 = TMA producer, warps 9..16 = epilogue.  The MMA warpgroups hand a finished tile to the epilogue through a
//   shared-memory accumulator tile and go on with the main loop of the next one.
// * Epilogue: accumulator tile -> coalesced fp32 stores through an arbitrary (n,t,h,w)-strided
//   output view (channel-slice "concat in place", strided dgrad scatter), optional accumulate, and per-tile
//   per-channel (sum, sum^2) partials for train-mode BatchNorm ([2][cout][m_tiles]).
#include <algorithm>
#include <cstdint>
#include <cstdio>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "runtime.h"

namespace sfb {

constexpr int BLOCK_M = 128;
constexpr int MAX_STAGES = 8;
constexpr int EPI_WARPS = 8;                     // two per 32-row quarter of the tile: the pair splits the tile's 16-column chunks
constexpr int EPI_STAGE_FLOATS = 64;             // per epilogue warp: 32 row offsets (int64)
constexpr int MMA_WARPS = 8;                     // two warpgroups of 64 tile rows
constexpr int PRODUCER_WARP = MMA_WARPS;
constexpr int EPI_WARP0 = MMA_WARPS + 1;
constexpr int CONV_THREADS = 32 * (MMA_WARPS + 1 + EPI_WARPS);
constexpr int BN_MAX = 128;                      // accumulator columns per tile: 64 registers per MMA thread
constexpr int BLOCK_K = 64;                      // K columns per k-block (pipeline stage)
constexpr int KSTEPS = BLOCK_K / 16;             // wgmma k16 steps per k-block

struct ConvParams {
  CUtensorMap tmA[2];
  CUtensorMap tmB[2];
  int M, oq, op, oz, nb;
  int sw, sh, sd;
  int lw, lh, ld;
  int kw, kh, kd;
  int dw, dh, dd;
  int CK, cpt, n_chunks, cps, k_blocks;
  int Ntot, BN, n_tiles, m_tiles;
  int ksplit;  // CTAs sharing one output tile, each over a contiguous slice of the k-blocks (1 = no split-K)
  int stages;
  int a_tiled;  // tap-free stride-1 conv: A is the plain [M][C] matrix, loaded with tiled (not im2col) TMA
  uint32_t stage_bytes, chunk_bytes, b_bytes, a_total_bytes, a_plane_bytes;
  uint32_t a_layout, a_sbo, a_lbo;
  uint32_t a_kstep[KSTEPS];  // start of k-step ks's A columns in the stage, in 16-byte units
  uint32_t acc_pitch;  // floats per row of the shared-memory accumulator tile
  uint32_t off_acc, off_staging, off_red, off_bars;
  float* out;
  long long os_n, os_z, os_p, os_q;
  int accumulate;
  int epi_coalesced;
  float* stats;
};

// First k-block of slice `kpart` of p.ksplit (balanced; every slice is non-empty because ksplit <= k_blocks).
__device__ __forceinline__ int k_block_begin(const ConvParams& p, int kpart) {
  return kpart * p.k_blocks / p.ksplit;
}

// csrc/conv_direct.cu: fp32 SIMT body for narrow layers (C_in <= 8); returns 1 when it handled the call
int conv_direct_try(const sfb_conv_desc* d, cudaStream_t stream, int* rc_out);

template <int NSPLIT, int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv_igemm_kernel(const __grid_constant__ ConvParams p) {
  static_assert(BN % 16 == 0 && BN <= BN_MAX, "tile width: a multiple of 16 up to BN_MAX");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + MAX_STAGES;
  uint64_t* tfull = empty + MAX_STAGES;
  uint64_t* tempty = tfull + 1;
  float* acc_tile = reinterpret_cast<float*>(smem + p.off_acc);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 32 * MMA_WARPS);
    }
    mbar_init(tfull, 32 * MMA_WARPS);
    mbar_init(tempty, EPI_WARPS);
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  // A work unit is one output tile and one of its p.ksplit slices of k-blocks; a tile's slices are consecutive units.
  const int total_units = p.m_tiles * p.n_tiles * p.ksplit;

  if (warp == PRODUCER_WARP) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&p.tmA[0]);
      tma_prefetch_desc(&p.tmB[0]);
      if (NSPLIT == 3) {
        tma_prefetch_desc(&p.tmA[1]);
        tma_prefetch_desc(&p.tmB[1]);
      }
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
      const int tile = unit / p.ksplit, kpart = unit - tile * p.ksplit;
      const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
      const int kb0 = k_block_begin(p, kpart), kb1 = k_block_begin(p, kpart + 1);
      int t = mt * BLOCK_M;
      const int q0 = t % p.oq;
      t /= p.oq;
      const int p0 = t % p.op;
      t /= p.op;
      const int z0 = t % p.oz;
      const int n0 = t / p.oz;
      const int cw = p.lw + q0 * p.sw, ch = p.lh + p0 * p.sh, cd = p.ld + z0 * p.sd;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          const int chunk0 = kb * p.cps;
          const uint32_t bytes = (uint32_t(p.cps) * p.chunk_bytes + p.b_bytes) * (NSPLIT == 3 ? 2u : 1u);
          mbar_expect_tx(&full[stage], bytes);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          for (int j = 0; j < p.cps; ++j) {
            const int idx = chunk0 + j;
            int nn = p.nb, c0 = 0;  // out-of-range batch index => the unit writes a zero chunk
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
            if (p.a_tiled) {
              // 1x1x1 / stride 1 / no padding: output position == input position, so the A tile is a plain 2-D box
              // of the [M][C] activation matrix.  Tiled TMA streams it at full rate; im2col mode is limited by the
              // number of per-pixel requests it keeps in flight (~2 TB/s at 128-byte rows, far less below).
              // (a zero pad chunk = a box past the last row: out-of-bounds rows are zero-filled)
              const int row0 = idx < p.n_chunks ? mt * BLOCK_M : p.m_tiles * BLOCK_M;
              tma_load_2d(st + j * p.chunk_bytes, &p.tmA[0], &full[stage], c0, row0);
              if (NSPLIT == 3) tma_load_2d(st + p.a_plane_bytes + j * p.chunk_bytes, &p.tmA[1], &full[stage], c0, row0);
              continue;
            }
            tma_load_im2col_5d(st + j * p.chunk_bytes, &p.tmA[0], &full[stage], c0, cw, ch, cd, nn, ow, oh, od);
            if (NSPLIT == 3)
              tma_load_im2col_5d(st + p.a_plane_bytes + j * p.chunk_bytes, &p.tmA[1], &full[stage], c0, cw, ch, cd,
                                 nn, ow, oh, od);
          }
          tma_load_2d(st + p.a_total_bytes, &p.tmB[0], &full[stage], kb * 64, nt * BN);
          if (NSPLIT == 3)
            tma_load_2d(st + p.a_total_bytes + p.b_bytes, &p.tmB[1], &full[stage], kb * 64, nt * BN);
        }
        __syncwarp();
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp < MMA_WARPS) {
    // ------------------------------------------------------------------ MMA warpgroups
    // Every k-block is KSTEPS k16 steps (the producer pads the last one with zero chunks) and the tile width is the
    // template's BN, so the k-block's 3 x KSTEPS wgmmas are straight-line code issued back to back.
    const int g = warp >> 2;  // tile rows 64g .. 64g+63: 8 core-matrix row groups (SBO apart) further into the A tile
    const uint32_t a_row_off = uint32_t(g) * 8u * p.a_sbo;
    float d[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x, ++it) {
      const int kpart = unit % p.ksplit;
      const int kb0 = k_block_begin(p, kpart), kb1 = k_block_begin(p, kpart + 1);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int held = -1;  // stage whose MMAs may still be reading shared memory
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        // descriptors of k-step 0; a later k-step adds its offset to the start-address field (16-byte units)
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + a_row_off;
        const uint32_t b_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + p.a_total_bytes;
        const uint64_t a_hi0 = make_smem_desc(a_base, p.a_lbo, p.a_sbo, p.a_layout);
        const uint64_t b_hi0 = make_smem_desc(b_base, 16, 1024, 2);
#pragma unroll
        for (int ks = 0; ks < KSTEPS; ++ks) {
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
        wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage can be refilled
        if (held >= 0) mbar_arrive(&empty[held]);
        held = stage;
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      mbar_arrive(&empty[held]);
      mbar_wait(tempty, (it & 1) ^ 1);  // the epilogue has read the previous tile
      acc_store<BN>(d, BN, acc_tile + size_t(g) * 64 * p.acc_pitch, int(p.acc_pitch));
      mbar_arrive(tfull);
    }
  } else {
    // ------------------------------------------------------------------ epilogue (8 warps: 2 per 32-row quarter)
    // The two warps of a quarter take the even / odd 16-column chunks of the tile.  Per chunk: 8 rows x 64 bytes per store
    // instruction (full 32-byte sectors) read straight from the accumulator tile, and the BatchNorm column sums come out
    // of the same reads.  accumulate = 2 adds with red.global.add (one add per element, no dependent load).
    const int ew = warp - EPI_WARP0;
    const int q = ew & 3;
    const int half = ew >> 2;
    long long* roff_s = reinterpret_cast<long long*>(reinterpret_cast<float*>(smem + p.off_staging) + ew * EPI_STAGE_FLOATS);
    float* red = reinterpret_cast<float*>(smem + p.off_red);  // [2][4][BN][2]
    const int sub = lane >> 2, cq = lane & 3;   // row within a group of 8, 16-byte piece of the chunk's 64-byte row
    constexpr int nchunks = BN >> 4;
    const float* qtile = acc_tile + size_t(q) * 32 * p.acc_pitch;
    int it = 0;
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x, ++it) {
      const int tile = unit / p.ksplit;
      const int acc = it & 1;
      const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
      const int ncol0 = nt * BN;
      const int row = mt * BLOCK_M + q * 32 + lane;
      const bool rvalid = row < p.M;
      long long roff = 0;
      if (rvalid) {
        int t = row;
        const int oq_ = t % p.oq;
        t /= p.oq;
        const int op_ = t % p.op;
        t /= p.op;
        const int oz_ = t % p.oz;
        const int on_ = t / p.oz;
        roff = on_ * p.os_n + oz_ * p.os_z + op_ * p.os_p + oq_ * p.os_q;
      }
      const uint32_t rmask = __ballot_sync(0xffffffffu, rvalid);
      float* red_w = red + ((size_t(acc) * 4 + q) * BN) * 2;
      roff_s[lane] = roff;
      __syncwarp();
      long long ro[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) ro[k] = roff_s[k * 8 + sub];

      mbar_wait(tfull, it & 1);
      for (int ch = half; ch < nchunks; ch += 2) {
        const int c0 = ch * 16;
        const int limit = min(BN, p.Ntot - ncol0) - c0;      // valid columns of this chunk (a multiple of 4)
        const bool cvalid = cq * 4 < limit;
        float s4[4] = {0.f, 0.f, 0.f, 0.f}, q4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int r = k * 8 + sub;
          const float4 y = *reinterpret_cast<const float4*>(qtile + size_t(r) * p.acc_pitch + c0 + cq * 4);
          s4[0] += y.x; s4[1] += y.y; s4[2] += y.z; s4[3] += y.w;
          q4[0] = fmaf(y.x, y.x, q4[0]); q4[1] = fmaf(y.y, y.y, q4[1]);
          q4[2] = fmaf(y.z, y.z, q4[2]); q4[3] = fmaf(y.w, y.w, q4[3]);
          if (((rmask >> r) & 1u) && cvalid) {
            float4* dst = reinterpret_cast<float4*>(p.out + ro[k] + ncol0 + c0 + cq * 4);
            if (p.accumulate == 2) {
              asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(y.x), "f"(y.y), "f"(y.z), "f"(y.w)
                           : "memory");
            } else if (p.accumulate) {
              const float4 o = *dst;
              *dst = make_float4(y.x + o.x, y.y + o.y, y.z + o.z, y.w + o.w);
            } else {
              *dst = y;
            }
          }
        }
        if (p.stats != nullptr) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int o = 4; o <= 16; o <<= 1) {
              s4[i] += __shfl_xor_sync(0xffffffffu, s4[i], o);
              q4[i] += __shfl_xor_sync(0xffffffffu, q4[i], o);
            }
          }
          if (sub == 0) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int cl = c0 + cq * 4 + i;
              red_w[cl * 2 + 0] = s4[i];
              red_w[cl * 2 + 1] = q4[i];
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty);  // this warp is done with the accumulator tile
      if (p.stats != nullptr) {
        named_bar_sync(1, 32 * EPI_WARPS);
        // the four quarter partials of this tile are in red[acc]; spread the column reduction over the epilogue warps
        const float* rb = red + size_t(acc) * 4 * BN * 2;
        for (int cl = ew * 32 + lane; cl < BN; cl += 32 * EPI_WARPS) {
          const int col = ncol0 + cl;
          if (col < p.Ntot) {
            float s = 0.f, s2 = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              s += rb[(size_t(w) * BN + cl) * 2 + 0];
              s2 += rb[(size_t(w) * BN + cl) * 2 + 1];
            }
            // [2][cout][m_tiles]: tile axis contiguous for the finalize kernel's per-channel reduction
            p.stats[size_t(col) * p.m_tiles + mt] = s;
            p.stats[(size_t(p.Ntot) + col) * p.m_tiles + mt] = s2;
          }
        }
      }
    }
  }

}

static int pick_ck(int c) {
  if (c % 64 == 0) return 64;
  if (c % 32 == 0) return 32;
  if (c % 16 == 0) return 16;
  return 8;
}

// Tile grid of a launch: 128 x BN output tiles, K in 64-column k-blocks (the last one padded with zero chunks).
struct ConvGrid {
  int64_t M;
  int CK, cps, n_chunks, k_blocks, BN, m_tiles, n_tiles;
};
static ConvGrid conv_grid(const sfb_conv_desc* d) {
  ConvGrid g;
  g.M = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  g.CK = pick_ck(d->c);
  g.cps = BLOCK_K / g.CK;
  g.n_chunks = d->kt * d->kh * d->kw * (d->c / g.CK);
  g.k_blocks = (g.n_chunks + g.cps - 1) / g.cps;
  g.BN = std::min((d->cout + 15) / 16 * 16, BN_MAX);
  g.m_tiles = int((g.M + BLOCK_M - 1) / BLOCK_M);
  g.n_tiles = (d->cout + g.BN - 1) / g.BN;
  return g;
}

// The output view is a plain row matrix (rows n*t*h*w apart by os_w): it can be zero-filled with one 2-D memset and
// its BatchNorm statistics taken by sfb_bn_split_stats.
static bool rows_regular(const sfb_conv_desc* d) {
  return d->os_h == int64_t(d->out_w) * d->os_w && d->os_t == int64_t(d->out_h) * d->os_h &&
         d->os_n == int64_t(d->out_t) * d->os_t;
}

// Split-K for grids that leave much of their last wave idle: each tile's k-blocks are split over s CTAs whose partial
// tiles meet in the output with red.global.add.  s minimises the waves per tile, ceil(tiles * s / SMs) / s, with a 2 %
// charge per extra slice (zero fill, s partial-tile epilogues), and is taken only when that beats s = 1 by 10 %.
// Each slice keeps at least 4 k-blocks so that its pipeline fill is amortised.  Not split: grids under half a wave
// (short launches, where the zero fill and the statistics pass are fixed costs), narrow inputs (C_in <= 8 may take
// the SIMT body), overwrites of views that are not a row matrix, and statistics of accumulating launches or over
// channels that are not a multiple of 8 (sfb_bn_split_stats).
static int conv_ksplit(const sfb_conv_desc* d, const ConvGrid& g, int P, bool with_stats) {
  const int tiles = g.m_tiles * g.n_tiles;
  if (P <= 0 || d->c <= 8 || 2 * tiles < P) return 1;
  if ((d->accumulate == 0 || with_stats) && !rows_regular(d)) return 1;
  if (with_stats && (d->accumulate != 0 || d->cout % 8 != 0 || d->os_w % 4 != 0)) return 1;
  auto cost = [&](int s) { return double((int64_t(tiles) * s + P - 1) / P) / s * (1.0 + 0.02 * (s - 1)); };
  int best = 1;
  for (int s = 2; s <= 8 && 4 * s <= g.k_blocks; ++s)
    if (cost(s) < cost(best)) best = s;
  return cost(best) < 0.9 * cost(1) ? best : 1;
}

}  // namespace sfb

using namespace sfb;

extern "C" int64_t sfb_conv_m_tiles(const sfb_conv_desc* d) {
  const ConvGrid g = conv_grid(d);
  int sms = 0;
  if (device_limits(&sms, nullptr) == 0 && conv_ksplit(d, g, sms, true) > 1)
    return sfb_bn_split_stats_tiles(g.M, g.M, 1, d->cout);  // statistics from y after the split GEMM
  return g.m_tiles;
}

extern "C" int32_t sfb_conv_ksplit(const sfb_conv_desc* d) {
  int sms = 0;
  if (device_limits(&sms, nullptr)) return 1;
  return conv_ksplit(d, conv_grid(d), sms, d->stats != nullptr);
}

extern "C" int sfb_conv_igemm(const sfb_conv_desc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int num_sms = 0, smem_optin = 0;
  if (device_limits(&num_sms, &smem_optin)) return -1;
  if (d->nsplit != 1 && d->nsplit != 3) {
    set_error("sfb_conv_igemm: nsplit must be 1 or 3 (got %d)", d->nsplit);
    return -10;
  }
  if (d->c % 8 != 0 || d->c_pitch % 8 != 0 || d->c <= 0) {
    set_error("sfb_conv_igemm: channel count %d / pitch %lld must be positive multiples of 8", d->c,
              (long long)d->c_pitch);
    return -10;
  }
  if (!d->a_hi || !d->b_hi || !d->out || (d->nsplit == 3 && (!d->a_lo || !d->b_lo))) {
    set_error("sfb_conv_igemm: null operand pointer");
    return -10;
  }
  const int64_t M64 = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  if (M64 <= 0 || M64 > 0x7fffffffLL || d->cout <= 0) {
    set_error("sfb_conv_igemm: bad output extent M=%lld cout=%d", (long long)M64, d->cout);
    return -10;
  }

  {
    int rc_direct = 0;
    if (conv_direct_try(d, stream, &rc_direct)) return rc_direct;
  }
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.M = int(M64);
  p.oq = d->out_w;
  p.op = d->out_h;
  p.oz = d->out_t;
  p.nb = d->n;
  p.sw = d->str_w;
  p.sh = d->str_h;
  p.sd = d->str_t;
  p.lw = d->low_w;
  p.lh = d->low_h;
  p.ld = d->low_t;
  p.kw = d->kw;
  p.kh = d->kh;
  p.kd = d->kt;
  p.dw = d->dil_w;
  p.dh = d->dil_h;
  p.dd = d->dil_t;
  const ConvGrid g = conv_grid(d);
  const int taps = d->kt * d->kh * d->kw;
  p.CK = g.CK;
  p.cpt = d->c / p.CK;
  p.n_chunks = g.n_chunks;
  p.cps = g.cps;
  p.k_blocks = g.k_blocks;
  p.Ntot = d->cout;
  p.BN = g.BN;
  p.n_tiles = g.n_tiles;
  p.m_tiles = g.m_tiles;
  p.ksplit = conv_ksplit(d, g, num_sms, d->stats != nullptr);
  p.chunk_bytes = BLOCK_M * p.CK * 2;
  p.b_bytes = p.BN * 128;
  // one A plane holds the chunks of ONE k-block, 64 K-columns (zero chunks past the last filter tap)
  p.a_plane_bytes = (uint32_t(p.cps) * p.chunk_bytes + 1023u) / 1024u * 1024u;
  p.a_total_bytes = p.a_plane_bytes * (d->nsplit == 3 ? 2 : 1);
  p.stage_bytes = p.a_total_bytes + p.b_bytes * (d->nsplit == 3 ? 2 : 1);
  p.stage_bytes = (p.stage_bytes + 1023) / 1024 * 1024;
  switch (p.CK) {
    case 64: p.a_layout = 2; p.a_sbo = 1024; p.a_lbo = 16; break;
    case 32: p.a_layout = 4; p.a_sbo = 512; p.a_lbo = 16; break;
    case 16: p.a_layout = 6; p.a_sbo = 256; p.a_lbo = 16; break;
    default: p.a_layout = 0; p.a_sbo = 128; p.a_lbo = p.chunk_bytes; break;
  }
  for (int ks = 0; ks < KSTEPS; ++ks) {
    const int k0 = ks * 16;
    const uint32_t off = p.CK >= 16 ? uint32_t(k0 / p.CK) * p.chunk_bytes + uint32_t(k0 % p.CK) * 2u
                                    : uint32_t(ks * 2) * p.chunk_bytes;  // CK = 8: two chunks, LBO apart
    p.a_kstep[ks] = off >> 4;
  }
  p.acc_pitch = uint32_t(p.BN) + 4;  // 16-byte rows; the 4-float skew spreads the fragment stores over the banks
  const uint32_t acc_bytes = BLOCK_M * p.acc_pitch * 4;
  const uint32_t tail = acc_bytes + EPI_WARPS * EPI_STAGE_FLOATS * 4 + 2 * 4 * p.BN * 2 * 4 + 256;
  const uint32_t budget = uint32_t(smem_optin) - 1024 - tail;
  p.stages = std::min<int>(MAX_STAGES, budget / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, p.k_blocks * 4));
  const int ctas_per_sm = 1;  // 544 threads x up to 120 registers: one CTA fills the register file
  if (p.stages < 2) {
    set_error("sfb_conv_igemm: not enough shared memory for 2 pipeline stages (stage=%u B)", p.stage_bytes);
    return -11;
  }
  p.off_acc = p.stages * p.stage_bytes;
  p.off_staging = p.off_acc + acc_bytes;
  p.off_red = p.off_staging + EPI_WARPS * EPI_STAGE_FLOATS * 4;
  p.off_bars = p.off_red + 2 * 4 * p.BN * 2 * 4;
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  p.out = d->out;
  p.os_n = d->os_n;
  p.os_z = d->os_t;
  p.os_p = d->os_h;
  p.os_q = d->os_w;
  // split-K: the slices add into the output (zero-filled first by an overwrite) and the statistics come from y afterwards
  p.accumulate = p.ksplit > 1 ? 2 : d->accumulate;
  p.epi_coalesced = 1;
  p.stats = p.ksplit > 1 ? nullptr : d->stats;

  // ---- tensor maps
  const int lower[3] = {d->low_w, d->low_h, d->low_t};
  const int strd[3] = {d->str_w, d->str_h, d->str_t};
  const int upper[3] = {d->low_w + (d->out_w - 1) * d->str_w + 1 - d->w, d->low_h + (d->out_h - 1) * d->str_h + 1 - d->h,
                        d->low_t + (d->out_t - 1) * d->str_t + 1 - d->d};
  const SwizzleBytes aswz = p.CK == 64 ? SWZ_128 : p.CK == 32 ? SWZ_64 : p.CK == 16 ? SWZ_32 : SWZ_NONE;
  p.a_tiled = (taps == 1 && d->str_w == 1 && d->str_h == 1 && d->str_t == 1 && d->low_w == 0 && d->low_h == 0 &&
               d->low_t == 0 && d->out_w == d->w && d->out_h == d->h && d->out_t == d->d)
                  ? 1 : 0;
  int rc;
  if (p.a_tiled)
    rc = make_tmap_2d_bf16(&p.tmA[0], d->a_hi, uint64_t(p.M), uint64_t(d->c), uint64_t(d->c_pitch), BLOCK_M, p.CK, aswz);
  else
    rc = make_tmap_im2col_bf16(&p.tmA[0], d->a_hi, d->n, d->d, d->h, d->w, d->c, d->c_pitch, lower, upper, strd, p.CK,
                               BLOCK_M, aswz);
  if (rc) return rc;
  const uint64_t ktot = uint64_t(taps) * d->c;
  rc = make_tmap_2d_bf16(&p.tmB[0], d->b_hi, d->cout, ktot, ktot, p.BN, 64, SWZ_128);
  if (rc) return rc;
  if (d->nsplit == 3) {
    if (p.a_tiled)
      rc = make_tmap_2d_bf16(&p.tmA[1], d->a_lo, uint64_t(p.M), uint64_t(d->c), uint64_t(d->c_pitch), BLOCK_M, p.CK, aswz);
    else
      rc = make_tmap_im2col_bf16(&p.tmA[1], d->a_lo, d->n, d->d, d->h, d->w, d->c, d->c_pitch, lower, upper, strd,
                                 p.CK, BLOCK_M, aswz);
    if (rc) return rc;
    rc = make_tmap_2d_bf16(&p.tmB[1], d->b_lo, d->cout, ktot, ktot, p.BN, 64, SWZ_128);
    if (rc) return rc;
  }

  if (p.ksplit > 1 && d->accumulate == 0) {
    // the epilogue writes whole float4 groups: columns [cout, cout rounded up to 4) take zeros too
    const size_t width = size_t((d->cout + 3) & ~3) * sizeof(float);
    if (cudaMemset2DAsync(d->out, size_t(d->os_w) * sizeof(float), 0, width, size_t(p.M), stream) != cudaSuccess) {
      set_error("sfb_conv_igemm: zero fill of the split-K output failed: %s", cudaGetErrorString(cudaGetLastError()));
      return -20;
    }
  }
  const int units = p.m_tiles * p.n_tiles * p.ksplit;
  const int grid = std::min(units, num_sms * ctas_per_sm);
  {
    typedef void (*KernelFn)(const ConvParams);
#define SFB_CONV_FNS(S) {conv_igemm_kernel<S, 16>, conv_igemm_kernel<S, 32>, conv_igemm_kernel<S, 48>, \
                         conv_igemm_kernel<S, 64>, conv_igemm_kernel<S, 80>, conv_igemm_kernel<S, 96>, \
                         conv_igemm_kernel<S, 112>, conv_igemm_kernel<S, 128>}
    static const KernelFn fns[2][BN_MAX / 16] = {SFB_CONV_FNS(1), SFB_CONV_FNS(3)};
#undef SFB_CONV_FNS
    static bool attr[2][BN_MAX / 16] = {};
    const int a = d->nsplit == 3 ? 1 : 0, b = p.BN / 16 - 1;
    if (!attr[a][b]) {
      cudaFuncSetAttribute(fns[a][b], cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin);
      attr[a][b] = true;
    }
    fns[a][b]<<<grid, CONV_THREADS, smem_bytes, stream>>>(p);
  }
  if (int rc = launch_status("sfb_conv_igemm", "grid=%d smem=%u stages=%d BN=%d CK=%d ksplit=%d", grid, smem_bytes,
                             p.stages, p.BN, p.CK, p.ksplit))
    return rc;
  if (p.ksplit > 1 && d->stats != nullptr)  // [2][cout][sfb_conv_m_tiles(d)] partials of the finished output
    return sfb_bn_split_stats(d->out, d->os_w, p.M, d->cout, 1, p.M, d->stats, stream);
  return 0;
}
