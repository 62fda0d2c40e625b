// Convolution weight gradient (wgrad) as an implicit GEMM on wgmma:
//
//   dW[co, (tap, ci)] = sum_m dY[m, co] * X_im2col[m, (tap, ci)]        m over n*ot*oh*ow output positions
//
// GEMM view: D[M' = co (128 rows), N' = (tap, ci) columns] with the reduction over output positions.  Both
// operands are "MN-major" for the tensor core (the reduction index is the slow axis of the tiles as they sit in
// memory), which wgmma reads natively through MN-major shared-memory descriptors:
//   * A' = dY tile  : tiled TMA box [64 positions][64 co]  (two boxes for the 128 co rows)
//   * B' = X tile   : one TMA im2col load per (tap, channel chunk): [64 positions][CK channels]; consecutive
//                     chunks form the N' extent of the MMA, so one dY tile is reused by up to 256 dW columns.
// The reduction is split across CTAs (split-K) and combined with vector fp32 reductions into dW, which the
// caller zero-fills.  Padding, the position tail and missing rows/columns are zero-filled by the TMA unit.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "tmap.h"

namespace sfb {

constexpr int WG_BLOCK_K = 64;  // output positions per pipeline stage
constexpr int WG_MAX_STAGES = 8;
constexpr int WG_MMA_WARPS = 8;   // two warpgroups: co rows 0..63 / 64..127 of the tile
constexpr int WG_THREADS = 32 * (WG_MMA_WARPS + 1);
constexpr int WG_BN_MAX = 128;

struct WgradParams {
  CUtensorMap tmX[2];
  CUtensorMap tmDy[2];
  int M, oq, op, oz, nb;
  int sw, sh, sd;
  int lw, lh, ld;
  int kw, kh, kd;
  int dw, dh, dd;
  int CK, cpt, n_chunks;
  int NG;  // chunks per N' tile
  int BN;  // NG * CK
  int n_tiles, co_tiles, cout, ktot;
  int x_tiled;  // tap-free stride-1 layer: X loaded with tiled TMA
  int k_blocks, splits, kb_per_split;
  int stages;
  uint32_t stage_bytes, x_chunk_bytes, x_plane_bytes, dy_plane_bytes;
  uint32_t b_layout, b_lbo, b_sbo, b_kstep_bytes;
  uint32_t acc_pitch;
  uint32_t off_acc, off_bars;
  float* dw_out;
};

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

template <int NSPLIT>
__global__ void __launch_bounds__(WG_THREADS, 1) conv_wgrad_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + WG_MAX_STAGES;
  float* acc_tile = reinterpret_cast<float*>(smem + p.off_acc);

  const int split = blockIdx.x % p.splits;
  const int tile = blockIdx.x / p.splits;
  const int co_tile = tile % p.co_tiles;
  const int n_tile = tile / p.co_tiles;
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(p.k_blocks, kb0 + p.kb_per_split);
  const int nkb = kb1 - kb0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 32 * WG_MMA_WARPS);
    }
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int chunk_base = n_tile * p.NG;  // first (tap, channel-chunk) of this N' tile

  if (nkb > 0) {
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
          const uint32_t bytes = (p.dy_plane_bytes + uint32_t(p.NG) * p.x_chunk_bytes) * (NSPLIT == 3 ? 2u : 1u);
          mbar_expect_tx(&full[stage], bytes);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          // dY: two [64 pos][64 co] boxes -> co rows 0..63 and 64..127 of the tile
          for (int hlf = 0; hlf < 2; ++hlf) {
            tma_load_2d(st + hlf * 8192, &p.tmDy[0], &full[stage], co_tile * 128 + hlf * 64, kb * WG_BLOCK_K);
            if (NSPLIT == 3)
              tma_load_2d(st + p.dy_plane_bytes + hlf * 8192, &p.tmDy[1], &full[stage], co_tile * 128 + hlf * 64,
                          kb * WG_BLOCK_K);
          }
          uint8_t* xb = st + p.dy_plane_bytes * (NSPLIT == 3 ? 2 : 1);
          for (int j = 0; j < p.NG; ++j) {
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
    } else {
      // ---------------------------------------------------------------- MMA warpgroups, then the epilogue
      const int g = warp >> 2;
      float d[WG_BN_MAX / 2];
      int stage = 0;
      uint32_t phase = 0;
      int held = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + uint32_t(g) * 8192u;
        const uint32_t b_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + p.dy_plane_bytes * (NSPLIT == 3 ? 2 : 1);
#pragma unroll
        for (int ks = 0; ks < WG_BLOCK_K / 16; ++ks) {
          // A' (dY): MN-major, 128B swizzle; co atoms 8192 B apart, 8-position groups 1024 B apart
          const uint64_t a_hi = make_smem_desc(a_base + ks * 2048, 8192, 1024, 2);
          const uint64_t b_hi = make_smem_desc(b_base + ks * p.b_kstep_bytes, p.b_lbo, p.b_sbo, p.b_layout);
          const uint32_t acc_flag = (kb != kb0 || ks != 0) ? 1u : 0u;
          if (NSPLIT == 3) {
            const uint64_t a_lo = make_smem_desc(a_base + p.dy_plane_bytes + ks * 2048, 8192, 1024, 2);
            const uint64_t b_lo =
                make_smem_desc(b_base + p.x_plane_bytes + ks * p.b_kstep_bytes, p.b_lbo, p.b_sbo, p.b_layout);
            wgmma_bf16<WG_BN_MAX, 1, 1>(d, p.BN, a_lo, b_hi, acc_flag);
            wgmma_bf16<WG_BN_MAX, 1, 1>(d, p.BN, a_hi, b_lo, 1u);
            wgmma_bf16<WG_BN_MAX, 1, 1>(d, p.BN, a_hi, b_hi, 1u);
          } else {
            wgmma_bf16<WG_BN_MAX, 1, 1>(d, p.BN, a_hi, b_hi, acc_flag);
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
      acc_store<WG_BN_MAX>(d, p.BN, acc_tile + size_t(g) * 64 * p.acc_pitch, int(p.acc_pitch));
      named_bar_sync(1, 32 * WG_MMA_WARPS);
      // epilogue: red.add into dW; warp w takes co rows 32 (w % 4) .. +31 and every other 16-column chunk
      const int q = warp & 3;
      const int co = co_tile * 128 + q * 32 + lane;
      const float* arow = acc_tile + size_t(q * 32 + lane) * p.acc_pitch;
      const int col_base = chunk_base * p.CK;
      for (int c0 = (warp >> 2) * 16; c0 < p.BN; c0 += 32) {
        uint32_t v[16];
        acc_ld_x16(arow + c0, v);
        if (co < p.cout) {
          float* dst = p.dw_out + size_t(co) * p.ktot + col_base + c0;
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            if (col_base + c0 + j < p.ktot)  // ktot is a multiple of 8, so 4-wide groups never straddle the edge
              red_add_v4(dst + j, __uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]),
                         __uint_as_float(v[j + 3]));
          }
        }
      }
    }
  }
}

static int wg_num_sms = 0, wg_smem_optin = 0;

}  // namespace sfb

using namespace sfb;

namespace sfb {
int wgrad_direct_try(const sfb_wgrad_desc* d, cudaStream_t stream, int* rc_out);
}

extern "C" int sfb_conv_wgrad(const sfb_wgrad_desc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!wg_num_sms) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
      set_error("cudaGetDevice failed: no CUDA device");
      return -1;
    }
    cudaDeviceGetAttribute(&wg_num_sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&wg_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  }
  if (d->nsplit != 1 && d->nsplit != 3) {
    set_error("sfb_conv_wgrad: nsplit must be 1 or 3");
    return -10;
  }
  if (d->c % 8 || d->c_pitch % 8 || d->cout % 8 || d->dy_pitch % 8) {
    set_error("sfb_conv_wgrad: c=%d c_pitch=%lld cout=%d dy_pitch=%lld must be multiples of 8", d->c,
              (long long)d->c_pitch, d->cout, (long long)d->dy_pitch);
    return -10;
  }
  if (!d->x_hi || !d->dy_hi || !d->dw || (d->nsplit == 3 && (!d->x_lo || !d->dy_lo))) {
    set_error("sfb_conv_wgrad: null operand pointer");
    return -10;
  }
  const int64_t M64 = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  if (M64 <= 0 || M64 > 0x7fffffffLL) {
    set_error("sfb_conv_wgrad: bad M=%lld", (long long)M64);
    return -10;
  }
  {
    // narrow layers with many positions: fp32 SIMT body (conv_wgrad_direct.cu), same operands and dW layout
    int rc_direct = 0;
    if (sfb::wgrad_direct_try(d, stream, &rc_direct)) return rc_direct;
  }
  WgradParams p;
  memset(&p, 0, sizeof(p));
  const int ns = d->nsplit == 3 ? 2 : 1;
  p.M = int(M64);
  p.oq = d->out_w; p.op = d->out_h; p.oz = d->out_t; p.nb = d->n;
  p.sw = d->str_w; p.sh = d->str_h; p.sd = d->str_t;
  p.lw = d->low_w; p.lh = d->low_h; p.ld = d->low_t;
  p.kw = d->kw; p.kh = d->kh; p.kd = d->kt;
  p.dw = d->dil_w; p.dh = d->dil_h; p.dd = d->dil_t;
  p.CK = d->c % 64 == 0 ? 64 : d->c % 32 == 0 ? 32 : d->c % 16 == 0 ? 16 : 8;
  p.cpt = d->c / p.CK;
  const int taps = d->kt * d->kh * d->kw;
  p.n_chunks = taps * p.cpt;
  p.ktot = taps * d->c;
  p.cout = d->cout;
  int ng = std::min(p.n_chunks, WG_BN_MAX / p.CK);
  if ((ng * p.CK) % 16) ng += 1;  // CK == 8 with an odd chunk count: pad with a zero chunk
  p.NG = ng;
  p.BN = ng * p.CK;
  p.n_tiles = (p.n_chunks + p.NG - 1) / p.NG;
  p.co_tiles = (d->cout + 127) / 128;
  p.k_blocks = (p.M + WG_BLOCK_K - 1) / WG_BLOCK_K;
  const int tiles = p.n_tiles * p.co_tiles;
  int splits = std::max(1, (2 * wg_num_sms) / tiles);
  splits = std::min(splits, std::max(1, p.k_blocks / 4));
  p.kb_per_split = (p.k_blocks + splits - 1) / splits;
  p.splits = (p.k_blocks + p.kb_per_split - 1) / p.kb_per_split;
  p.x_chunk_bytes = WG_BLOCK_K * p.CK * 2;
  p.x_plane_bytes = p.NG * p.x_chunk_bytes;
  p.dy_plane_bytes = 2 * 8192;
  p.stage_bytes = (p.dy_plane_bytes + p.x_plane_bytes) * ns;
  p.stage_bytes = (p.stage_bytes + 1023) / 1024 * 1024;
  switch (p.CK) {
    case 64: p.b_layout = 2; p.b_lbo = p.x_chunk_bytes; p.b_sbo = 1024; p.b_kstep_bytes = 16 * 128; break;
    case 32: p.b_layout = 4; p.b_lbo = p.x_chunk_bytes; p.b_sbo = 512; p.b_kstep_bytes = 16 * 64; break;
    case 16: p.b_layout = 6; p.b_lbo = p.x_chunk_bytes; p.b_sbo = 256; p.b_kstep_bytes = 16 * 32; break;
    default: p.b_layout = 0; p.b_lbo = 128; p.b_sbo = p.x_chunk_bytes; p.b_kstep_bytes = 16 * 16; break;
  }
  p.acc_pitch = uint32_t(p.BN) + 4;
  const uint32_t acc_bytes = 128u * p.acc_pitch * 4u;
  const uint32_t budget = uint32_t(wg_smem_optin) - 1024 - 256 - acc_bytes;
  p.stages = std::min<int>(WG_MAX_STAGES, budget / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, p.kb_per_split));
  if (p.stages < 2) {
    set_error("sfb_conv_wgrad: not enough shared memory (stage=%u B)", p.stage_bytes);
    return -11;
  }
  p.off_acc = p.stages * p.stage_bytes;
  p.off_bars = p.off_acc + acc_bytes;
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  p.dw_out = d->dw;

  const int lower[3] = {d->low_w, d->low_h, d->low_t};
  const int strd[3] = {d->str_w, d->str_h, d->str_t};
  const int upper[3] = {d->low_w + (d->out_w - 1) * d->str_w + 1 - d->w, d->low_h + (d->out_h - 1) * d->str_h + 1 - d->h,
                        d->low_t + (d->out_t - 1) * d->str_t + 1 - d->d};
  const SwizzleBytes xswz = p.CK == 64 ? SWZ_128 : p.CK == 32 ? SWZ_64 : p.CK == 16 ? SWZ_32 : SWZ_NONE;
  {
    const char* e = getenv("SFB_CONV_FORCE_IM2COL");
    const bool force = e && e[0] == '1';
    p.x_tiled = (taps == 1 && d->str_w == 1 && d->str_h == 1 && d->str_t == 1 && d->low_w == 0 && d->low_h == 0 &&
                 d->low_t == 0 && d->out_w == d->w && d->out_h == d->h && d->out_t == d->d && !force) ? 1 : 0;
  }
  int rc;
  for (int pl = 0; pl < ns; ++pl) {
    if (p.x_tiled)
      rc = make_tmap_2d_bf16(&p.tmX[pl], pl ? d->x_lo : d->x_hi, uint64_t(p.M), uint64_t(d->c), uint64_t(d->c_pitch),
                             WG_BLOCK_K, p.CK, xswz);
    else
      rc = make_tmap_im2col_bf16(&p.tmX[pl], pl ? d->x_lo : d->x_hi, d->n, d->d, d->h, d->w, d->c, d->c_pitch, lower,
                                 upper, strd, p.CK, WG_BLOCK_K, xswz);
    if (rc) return rc;
    rc = make_tmap_2d_bf16(&p.tmDy[pl], pl ? d->dy_lo : d->dy_hi, uint64_t(p.M), uint64_t(d->cout),
                           uint64_t(d->dy_pitch), WG_BLOCK_K, 64, SWZ_128);
    if (rc) return rc;
  }
  const int grid = tiles * p.splits;
  if (d->nsplit == 3) {
    static bool a3 = false;
    if (!a3) {
      cudaFuncSetAttribute(conv_wgrad_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_optin);
      a3 = true;
    }
    conv_wgrad_kernel<3><<<grid, WG_THREADS, smem_bytes, stream>>>(p);
  } else {
    static bool a1 = false;
    if (!a1) {
      cudaFuncSetAttribute(conv_wgrad_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_optin);
      a1 = true;
    }
    conv_wgrad_kernel<1><<<grid, WG_THREADS, smem_bytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_conv_wgrad launch failed: %s (grid=%d smem=%u)", cudaGetErrorString(e), grid, smem_bytes);
    return -20;
  }
  return 0;
}
