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
// * Persistent ping-pong CTAs, warp-specialised: warpgroup 0 is the TMA producer (one elected lane issues the loads),
//   warpgroups 1 and 2 are consumers.  A consumer owns whole 128 x BN tiles (two m64 row blocks in its registers) and
//   the CTA's work units alternate between the two.  An ordered pair of named barriers lets one consumer issue its
//   main loop while the other runs its epilogue, so no shared-memory accumulator tile is needed and all of shared
//   memory but the BatchNorm scratch goes to the operand ring.
// * Epilogue from the wgmma fragments: each warp passes its rows through a 1 KB staging block (store_fragment), so every
//   fp32 store instruction writes whole 128-byte lines.  Stores go through an arbitrary (n,t,h,w)-strided output view
//   (channel-slice "concat in place", strided dgrad scatter), with optional accumulate, and per-tile per-channel
//   (sum, sum^2) partials for train-mode BatchNorm ([2][cout][m_tiles]).
#include <algorithm>
#include <cstdint>
#include <cstdio>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "runtime.h"

namespace sfb {

constexpr int BLOCK_M = 128;
constexpr int MAX_STAGES = 8;
constexpr int CONV_THREADS = 384;                // warpgroup 0: producer; warpgroups 1, 2: MMA + epilogue consumers
constexpr int PRODUCER_REGS = 40;                // 128 x (40 + 2 x 232) registers fit the 64 K register file
constexpr int CONSUMER_REGS = 232;
constexpr int BAR_ORDER = 1;                     // named barrier 1 + c: consumer c may issue its main loop
constexpr int BAR_EPI = 3;                       // named barrier 3 + c: consumer c's epilogue (row table, partials)
constexpr int BN_MAX = 128;                      // accumulator columns per tile: 128 registers per consumer thread
constexpr int BLOCK_K = 64;                      // K columns per k-block (pipeline stage)
constexpr int KSTEPS = BLOCK_K / 16;             // wgmma k16 steps per k-block
constexpr long long kNoRow = INT64_MIN;          // epilogue row table: tile row past M
// per consumer: the tile's row table, then 4 warps' 8 x 32 fp32 staging blocks, which the [4][BN][2] BatchNorm
// partials reuse once the tile is stored
constexpr uint32_t EPI_SCRATCH = BLOCK_M * 8 + 4 * 8 * 32 * 4;
static_assert(4 * BN_MAX * 2 * 4 <= 4 * 8 * 32 * 4, "BatchNorm partials fit the staging blocks");

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
  uint32_t off_epi, off_bars;
  float* out;
  long long os_n, os_z, os_p, os_q;
  int accumulate;
  float* stats;
};

// First k-block of slice `kpart` of p.ksplit (balanced; every slice is non-empty because ksplit <= k_blocks).
__device__ __forceinline__ int k_block_begin(const ConvParams& p, int kpart) {
  return kpart * p.k_blocks / p.ksplit;
}

// csrc/conv_direct.cu: fp32 SIMT body for narrow layers (C_in <= 8); returns 1 when it handled the call
int conv_direct_try(const sfb_conv_desc* d, cudaStream_t stream, int* rc_out);

// Stores a consumer's 128 x BN accumulator fragment (layout in the kernel's epilogue).  Each warp passes its rows through
// a 1 KB staging block, 8 rows x 32 columns at a time, so that every store instruction writes whole 128-byte lines:
// lane l writes float4 columns 4 (l % 8) .. +3 of rows l / 8 and l / 8 + 4.  The block's 8-column groups are XOR-swizzled
// by the row, so the fragment writes and the row reads are both conflict-free.  MODE 0 overwrites, 1 adds to the
// destination, 2 adds with red.global.add.  roff: the tile's row table (kNoRow: not stored); columns from ncols on are
// not stored.
template <int BN, int MODE>
__device__ __forceinline__ void store_fragment(const float (&d)[2][BN / 2], float* stage, const long long* roff,
                                               float* out, int ncols) {
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int g = lane >> 2, cq = 2 * (lane & 3);  // fragment: row g (+8 h), columns 8 jn + cq, +1
  const int rr = lane >> 3, c4 = 4 * (lane & 7);   // read-back: rows rr and rr + 4, columns c4 .. c4 + 3
#pragma unroll
  for (int rb = 0; rb < 2; ++rb) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int cg = 0; cg < (BN + 31) / 32; ++cg) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int jn = 4 * cg + jj;
          if (jn < BN / 8)
            *reinterpret_cast<float2*>(stage + g * 32 + ((8 * jj + cq) ^ (8 * (g & 3)))) =
                make_float2(d[rb][4 * jn + 2 * h], d[rb][4 * jn + 2 * h + 1]);
        }
        __syncwarp();
        float4 v[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) v[k] = *reinterpret_cast<const float4*>(stage + (rr + 4 * k) * 32 + (c4 ^ (8 * rr)));
        __syncwarp();
        const int col = 32 * cg + c4;
        if (col >= ncols) continue;
        float4* dst[2];
        bool ok[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const long long o = roff[64 * rb + 16 * warp + 8 * h + rr + 4 * k];
          ok[k] = o != kNoRow;
          dst[k] = reinterpret_cast<float4*>(out + (ok[k] ? o + col : 0));
        }
        if (MODE == 1) {
          float4 o[2];
#pragma unroll
          for (int k = 0; k < 2; ++k)
            if (ok[k]) o[k] = *dst[k];
#pragma unroll
          for (int k = 0; k < 2; ++k)
            if (ok[k]) *dst[k] = make_float4(v[k].x + o[k].x, v[k].y + o[k].y, v[k].z + o[k].z, v[k].w + o[k].w);
        } else {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            if (!ok[k]) continue;
            if (MODE == 2)
              asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst[k]), "f"(v[k].x), "f"(v[k].y),
                           "f"(v[k].z), "f"(v[k].w) : "memory");
            else
              *dst[k] = v[k];
          }
        }
      }
    }
  }
}

template <int NSPLIT, int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv_igemm_kernel(const __grid_constant__ ConvParams p) {
  static_assert(BN % 16 == 0 && BN <= BN_MAX, "tile width: a multiple of 16 up to BN_MAX");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + MAX_STAGES;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 128);  // the 128 threads of the consumer that read the stage
    }
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  // A work unit is one output tile and one of its p.ksplit slices of k-blocks; a tile's slices are consecutive units.
  const int total_units = p.m_tiles * p.n_tiles * p.ksplit;

  if (threadIdx.x < 128) {
    // ------------------------------------------------------------------ TMA producer (warp 0; warps 1..3 idle)
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x >= 32) return;
    if (threadIdx.x == 0) {
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
    return;
  }

  // -------------------------------------------------------------------- consumers (warpgroups 1, 2)
  // The CTA's j-th unit belongs to consumer j & 1.  Consumer c issues the main loop of unit j after the other consumer
  // has issued that of unit j - 1 (named barrier BAR_ORDER + c), so one consumer's epilogue overlaps the other's MMAs.
  // Every k-block is KSTEPS k16 steps (the producer pads the last one with zero chunks) and the tile width is the
  // template's BN, so the k-block's wgmmas are straight-line code issued back to back.
  setmaxnreg_inc<CONSUMER_REGS>();
  const int c = (threadIdx.x >> 7) - 1;
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  const uint32_t a_rb = (8u * p.a_sbo) >> 4;  // row block 1 = 8 core-matrix row groups (SBO apart) into the A tile
  float d[2][BN / 2];                         // rows 0..63 / 64..127 of the tile
  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0, unit = blockIdx.x; unit < total_units; ++j, unit += gridDim.x) {
    const int tile = unit / p.ksplit, kpart = unit - tile * p.ksplit;
    const int kb0 = k_block_begin(p, kpart), kb1 = k_block_begin(p, kpart + 1);
    if ((j & 1) != c) {  // the other consumer's unit: step over its stages
      for (int kb = kb0; kb < kb1; ++kb) {
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      continue;
    }
    if (j > 0) named_bar_sync(BAR_ORDER + c, 256);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[0][i] = d[1][i] = 0.f;
    int held = -1;  // stage whose MMAs may still be reading shared memory
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full[stage], phase);
      wgmma_fence();
      // descriptors of k-step 0; a later k-step adds its offset to the start-address field (16-byte units)
      const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes);
      const uint32_t b_base = a_base + p.a_total_bytes;
      const uint64_t a_hi0 = make_smem_desc(a_base, p.a_lbo, p.a_sbo, p.a_layout);
      const uint64_t b_hi0 = make_smem_desc(b_base, 16, 1024, 2);
#pragma unroll
      for (int ks = 0; ks < KSTEPS; ++ks) {
        const uint64_t a_hi = a_hi0 + p.a_kstep[ks];
        const uint64_t b_hi = b_hi0 + uint64_t(ks * 2);  // 32 bytes = 16 bf16 of the 128-byte swizzled rows
        // consecutive wgmmas alternate between the two row blocks' accumulators
        if (NSPLIT == 3) {
          const uint64_t a_lo = a_hi + (p.a_plane_bytes >> 4);
          const uint64_t b_lo = b_hi + (p.b_bytes >> 4);
          wgmma_m64n<BN>(d[0], a_lo, b_hi);
          wgmma_m64n<BN>(d[1], a_lo + a_rb, b_hi);
          wgmma_m64n<BN>(d[0], a_hi, b_lo);
          wgmma_m64n<BN>(d[1], a_hi + a_rb, b_lo);
        }
        wgmma_m64n<BN>(d[0], a_hi, b_hi);
        wgmma_m64n<BN>(d[1], a_hi + a_rb, b_hi);
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
    if (unit + int(gridDim.x) < total_units) named_bar_arrive(BAR_ORDER + (c ^ 1), 256);  // unit j + 1 may start

    // ------------------------------------------------------------------ epilogue
    // While the last MMAs run, each thread computes one row's offset through the (n,t,h,w) strides into the consumer's
    // row table (kNoRow: a row >= M; it holds zeros, as TMA zero-fills its A row, and is not stored).
    const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
    const int ncol0 = nt * BN;
    uint8_t* epi = smem + p.off_epi + size_t(c) * EPI_SCRATCH;  // row table, then staging blocks / BatchNorm partials
    long long* roff_s = reinterpret_cast<long long*>(epi);
    {
      int r = mt * BLOCK_M + t;
      long long off = kNoRow;
      if (r < p.M) {
        const int oq_ = r % p.oq;
        r /= p.oq;
        const int op_ = r % p.op;
        r /= p.op;
        const int oz_ = r % p.oz;
        const int on_ = r / p.oz;
        off = on_ * p.os_n + oz_ * p.os_z + op_ * p.os_p + oq_ * p.os_q;
      }
      roff_s[t] = off;
    }
    named_bar_sync(BAR_EPI + c, 128);
    // Thread (warp, lane) holds rows 16 warp + lane/4 (+8) of each row block and columns 8 jn + 2 (lane % 4) (+1):
    // d[rb][4 jn + 2 h + e] is row 64 rb + 8 h + 16 warp + lane/4, column 8 jn + 2 (lane % 4) + e.
    const int cq = 2 * (lane & 3);
    // whole groups of 4 columns up to cout are stored, as the split-K zero fill assumes
    const int ncols = min(BN, ((p.Ntot + 3) & ~3) - ncol0);
    float* stage_w = reinterpret_cast<float*>(epi + BLOCK_M * 8) + warp * 256;
    wgmma_wait<0>();
    mbar_arrive(&empty[held]);
    if (p.accumulate == 2) store_fragment<BN, 2>(d, stage_w, roff_s, p.out + ncol0, ncols);
    else if (p.accumulate == 1) store_fragment<BN, 1>(d, stage_w, roff_s, p.out + ncol0, ncols);
    else store_fragment<BN, 0>(d, stage_w, roff_s, p.out + ncol0, ncols);
    if (p.stats != nullptr) {
      // per-thread sums over its 4 rows, then over the 8 row lanes of the warp, then over the 4 warps in shared memory
      float* red = reinterpret_cast<float*>(epi + BLOCK_M * 8);  // [warp][BN][sum, sum^2], over the staging blocks
      named_bar_sync(BAR_EPI + c, 128);  // every warp is done with its staging block
#pragma unroll
      for (int jn = 0; jn < BN / 8; ++jn) {
        float s[2], q[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float a0 = d[0][4 * jn + e], a1 = d[0][4 * jn + 2 + e], a2 = d[1][4 * jn + e], a3 = d[1][4 * jn + 2 + e];
          s[e] = (a0 + a1) + (a2 + a3);
          q[e] = fmaf(a0, a0, fmaf(a1, a1, fmaf(a2, a2, a3 * a3)));
#pragma unroll
          for (int o = 4; o <= 16; o <<= 1) {
            s[e] += __shfl_xor_sync(0xffffffffu, s[e], o);
            q[e] += __shfl_xor_sync(0xffffffffu, q[e], o);
          }
        }
        if (lane < 4)
          *reinterpret_cast<float4*>(red + (size_t(warp) * BN + 8 * jn + cq) * 2) = make_float4(s[0], q[0], s[1], q[1]);
      }
      named_bar_sync(BAR_EPI + c, 128);
      const int col = ncol0 + t;
      if (t < BN && col < p.Ntot) {
        float s = 0.f, s2 = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          s += red[(size_t(w) * BN + t) * 2 + 0];
          s2 += red[(size_t(w) * BN + t) * 2 + 1];
        }
        // [2][cout][m_tiles]: tile axis contiguous for the finalize kernel's per-channel reduction
        p.stats[size_t(col) * p.m_tiles + mt] = s;
        p.stats[(size_t(p.Ntot) + col) * p.m_tiles + mt] = s2;
      }
      named_bar_sync(BAR_EPI + c, 128);  // the scratch is free for this consumer's next tile
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
  // all of shared memory but the barriers and the consumers' epilogue scratch goes to the operand ring
  const uint32_t epi_bytes = 2u * EPI_SCRATCH;
  const uint32_t budget = uint32_t(smem_optin) - 1024 - epi_bytes - 256;
  p.stages = std::min<int>(MAX_STAGES, budget / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, p.k_blocks * 4));
  const int ctas_per_sm = 1;  // 384 threads at 40 / 232 / 232 registers: one CTA fills the register file
  if (p.stages < 2) {
    set_error("sfb_conv_igemm: not enough shared memory for 2 pipeline stages (stage=%u B)", p.stage_bytes);
    return -11;
  }
  p.off_epi = p.stages * p.stage_bytes;
  p.off_bars = p.off_epi + epi_bytes;
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  p.out = d->out;
  p.os_n = d->os_n;
  p.os_z = d->os_t;
  p.os_p = d->os_h;
  p.os_q = d->os_w;
  // split-K: the slices add into the output (zero-filled first by an overwrite) and the statistics come from y afterwards
  p.accumulate = p.ksplit > 1 ? 2 : d->accumulate;
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
    // the epilogue writes whole groups of 4 columns: columns [cout, cout rounded up to 4) take zeros too
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
