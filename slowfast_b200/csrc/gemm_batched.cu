// Batched GEMM on wgmma for the attention products of MViT's MultiScaleAttention (attention.py:355-379 and
// their autograd transposes):
//
//     D[b](m, n) (+)= alpha * sum_k A[b](m, k) * B[b](n, k)          b = batch * heads
//
// Either operand may be "K-major" (memory [b][rows][K], K contiguous) or "MN-major" (memory [b][K][rows], rows
// contiguous); all four attention products and their gradients are covered without any transpose copy:
//     S  = q k^T      A=q  (K)   B=k  (K)        dP = dO v^T   A=dO (K)   B=v  (K)
//     O  = P v        A=P  (K)   B=v  (MN)       dq = dS k     A=dS (K)   B=k  (MN)
//     dv = P^T dO     A=P  (MN)  B=dO (MN)       dk = dS^T q   A=dS (MN)  B=q  (MN)
// Operands are split-bf16 planes (nsplit 3) or bf16 (nsplit 1), staged by 3-D tiled TMA (128B swizzle; K / row /
// batch tails zero-filled by the unit), accumulated in registers (two warpgroups of 64 x BN x 16 wgmma), same persistent
// warp-specialised pipeline as conv_igemm.cu (two MMA warpgroups / producer warp / 4 epilogue warps reading a
// shared-memory accumulator tile).
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "../../include/slowfast_b200.h"
#include "ptx.cuh"
#include "tmap.h"

namespace sfb {

constexpr int BG_BLOCK_M = 128;
constexpr int BG_BLOCK_K = 64;
constexpr int BG_MAX_STAGES = 8;
constexpr int BG_MMA_WARPS = 8;
constexpr int BG_EPI_WARP0 = BG_MMA_WARPS + 1;
constexpr int BG_THREADS = 32 * (BG_MMA_WARPS + 1 + 4);
constexpr int BG_BN_MAX = 128;

struct BgemmParams {
  CUtensorMap tmA[2];
  CUtensorMap tmB[2];
  int M, N, K, batch;
  int a_mn, b_mn;
  int BN, n_atoms;  // BN = UMMA N; n_atoms = ceil(BN / 64) (MN-major B only)
  int m_tiles, n_tiles, k_blocks;
  int stages;
  uint32_t stage_bytes, a_plane_bytes, b_plane_bytes;
  uint32_t acc_pitch;
  uint32_t off_acc, off_bars;
  float* out;
  long long ldd, batch_stride_d;
  float alpha;
  int accumulate;
  // split-K (r2): work item = (tile, k-split); every split reduces its k-block range into the (pre-zeroed or accumulated)
  // output with float atomics.  Used when the tile count cannot fill the machine and K is long (dV / dK of the early MViT
  // blocks: 16 tiles, K = 25 089 queries).
  int k_splits, kb_per_split;
};

__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* tm, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

template <int NSPLIT>
__global__ void __launch_bounds__(BG_THREADS, 1) gemm_batched_kernel(const __grid_constant__ BgemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bars);
  uint64_t* empty = full + BG_MAX_STAGES;
  uint64_t* tfull = empty + BG_MAX_STAGES;
  uint64_t* tempty = tfull + 1;
  float* acc_tile = reinterpret_cast<float*>(smem + p.off_acc);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 32 * BG_MMA_WARPS);
    }
    mbar_init(tfull, 32 * BG_MMA_WARPS);
    mbar_init(tempty, 4);
    fence_mbar_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int tiles_per_batch = p.m_tiles * p.n_tiles;
  const int total_tiles = tiles_per_batch * p.batch;
  const int total_work = total_tiles * p.k_splits;
  constexpr uint32_t NP = NSPLIT == 3 ? 2u : 1u;

  if (warp == BG_MMA_WARPS) {
    // ------------------------------------------------------------------ TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
      const int tile = work / p.k_splits, ksp = work - tile * p.k_splits;
      const int b = tile / tiles_per_batch;
      const int r = tile - b * tiles_per_batch;
      const int mt = r / p.n_tiles, nt = r - mt * p.n_tiles;
      const int m0 = mt * BG_BLOCK_M, n0 = nt * p.BN;
      const int kb0 = ksp * p.kb_per_split, kb1 = min(p.k_blocks, kb0 + p.kb_per_split);
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full[stage], (p.a_plane_bytes + p.b_plane_bytes) * NP);
          uint8_t* st = smem + size_t(stage) * p.stage_bytes;
          const int k0 = kb * BG_BLOCK_K;
          for (uint32_t pl = 0; pl < NP; ++pl) {
            uint8_t* a_dst = st + pl * p.a_plane_bytes;
            if (p.a_mn) {  // [b][K][M]: two boxes of 64 (M) x 64 (K rows)
              tma_load_3d(a_dst, &p.tmA[pl], &full[stage], m0, k0, b);
              tma_load_3d(a_dst + 8192, &p.tmA[pl], &full[stage], m0 + 64, k0, b);
            } else {       // [b][M][K]: one box of 64 (K) x 128 (M rows)
              tma_load_3d(a_dst, &p.tmA[pl], &full[stage], k0, m0, b);
            }
            uint8_t* b_dst = st + NP * p.a_plane_bytes + pl * p.b_plane_bytes;
            if (p.b_mn) {
              for (int j = 0; j < p.n_atoms; ++j)
                tma_load_3d(b_dst + j * 8192, &p.tmB[pl], &full[stage], n0 + j * 64, k0, b);
            } else {
              tma_load_3d(b_dst, &p.tmB[pl], &full[stage], k0, n0, b);
            }
          }
        }
        __syncwarp();
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp < BG_MMA_WARPS) {
    // ------------------------------------------------------------------ MMA warpgroups (rows 64g .. 64g+63)
    // Both operand forms put the second 64 rows 8192 B further: the next 64-row MN atom, or 8 more 1024-byte row groups.
    const int g = warp >> 2;
    const int mode = p.a_mn * 2 + p.b_mn;
    float d[BG_BN_MAX / 2];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int work = blockIdx.x; work < total_work; work += gridDim.x, ++it) {
      const int ksp = work % p.k_splits;
      const int kb0 = ksp * p.kb_per_split, kb1 = min(p.k_blocks, kb0 + p.kb_per_split);
      int held = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t a_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + uint32_t(g) * 8192u;
        const uint32_t b_base = smem_u32(smem + size_t(stage) * p.stage_bytes) + NP * p.a_plane_bytes;
#pragma unroll
        for (int ks = 0; ks < BG_BLOCK_K / 16; ++ks) {
          uint64_t a_d[2], b_d[2];
          for (uint32_t pl = 0; pl < NP; ++pl) {
            const uint32_t aa = a_base + pl * p.a_plane_bytes, bb = b_base + pl * p.b_plane_bytes;
            a_d[pl] = p.a_mn ? make_smem_desc(aa + ks * 2048, 8192, 1024, 2) : make_smem_desc(aa + ks * 32, 16, 1024, 2);
            b_d[pl] = p.b_mn ? make_smem_desc(bb + ks * 2048, 8192, 1024, 2) : make_smem_desc(bb + ks * 32, 16, 1024, 2);
          }
          const uint32_t acc_flag = ((kb - kb0) | ks) != 0 ? 1u : 0u;
          const int nprod = NSPLIT == 3 ? 3 : 1;
          for (int pr = 0; pr < nprod; ++pr) {
            // split products: A_lo*B_hi + A_hi*B_lo + A_hi*B_hi
            const uint64_t ad = (NSPLIT == 3 && pr == 0) ? a_d[1] : a_d[0];
            const uint64_t bd = (NSPLIT == 3 && pr == 1) ? b_d[1] : b_d[0];
            const uint32_t af = pr == 0 ? acc_flag : 1u;
            switch (mode) {
              case 0: wgmma_bf16<BG_BN_MAX, 0, 0>(d, p.BN, ad, bd, af); break;
              case 1: wgmma_bf16<BG_BN_MAX, 0, 1>(d, p.BN, ad, bd, af); break;
              case 2: wgmma_bf16<BG_BN_MAX, 1, 0>(d, p.BN, ad, bd, af); break;
              default: wgmma_bf16<BG_BN_MAX, 1, 1>(d, p.BN, ad, bd, af); break;
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
      acc_store<BG_BN_MAX>(d, p.BN, acc_tile + size_t(g) * 64 * p.acc_pitch, int(p.acc_pitch));
      mbar_arrive(tfull);
    }
  } else {
    // ------------------------------------------------------------------ epilogue
    const int q = warp - BG_EPI_WARP0;
    const float* arow = acc_tile + size_t(q * 32 + lane) * p.acc_pitch;
    int it = 0;
    for (int work = blockIdx.x; work < total_work; work += gridDim.x, ++it) {
      const int tile = work / p.k_splits;
      const int b = tile / tiles_per_batch;
      const int r = tile - b * tiles_per_batch;
      const int mt = r / p.n_tiles, nt = r - mt * p.n_tiles;
      const int row0 = mt * BG_BLOCK_M + q * 32;
      const int ncol0 = nt * p.BN;
      float* obase = p.out + size_t(b) * p.batch_stride_d;
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
        float x[32];
#pragma unroll
        for (int j = 0; j < 16; ++j) x[j] = __uint_as_float(v0[j]) * p.alpha;
#pragma unroll
        for (int j = 0; j < 16; ++j) x[16 + j] = second ? __uint_as_float(v1[j]) * p.alpha : 0.f;
        const int row = row0 + lane;
        if (row < p.M) {
          float* orow = obase + size_t(row) * p.ldd + ncol0 + c0;  // ldd % 4 == 0 and ncol0 % 16 == 0: 16 B aligned
          const int nvalid = min(min(p.BN, p.N - ncol0) - c0, 32);  // valid columns in this 32-wide chunk
          if (p.k_splits > 1) {   // partial sums of this k-range: float atomics into the zeroed / accumulated output
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (j < nvalid) atomicAdd(orow + j, x[j]);
            continue;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (4 * j + 3 < nvalid) {
              float4* d4 = reinterpret_cast<float4*>(orow) + j;
              float4 o = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
              if (p.accumulate) {
                const float4 old = *d4;
                o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
              }
              *d4 = o;
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (4 * j + e < nvalid) orow[4 * j + e] = p.accumulate ? orow[4 * j + e] + x[4 * j + e] : x[4 * j + e];
            }
          }
        }
      }
    }
  }

}

typedef CUresult (*EncodeTiledFn3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 3-D map over bf16 [batch][rows][cols] (cols contiguous, row pitch ld, batch stride bs), box = [1][box_rows][64]
static int make_tmap_3d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t ld,
                        uint64_t bs, uint32_t box_rows) {
  static EncodeTiledFn3 fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeTiled entry point unavailable");
      return -1;
    }
    fn = reinterpret_cast<EncodeTiledFn3>(f);
  }
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {ld * 2, bs * 2};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(3d) failed (%d): cols=%llu rows=%llu batch=%llu ld=%llu bs=%llu box_rows=%u", (int)r,
              (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)batch, (unsigned long long)ld,
              (unsigned long long)bs, box_rows);
    return -2;
  }
  return 0;
}

static int bg_sms = 0, bg_smem = 0;

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_gemm_batched(const sfb_bgemm_desc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!bg_sms) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
      set_error("cudaGetDevice failed: no CUDA device");
      return -1;
    }
    cudaDeviceGetAttribute(&bg_sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&bg_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  }
  if (d->nsplit != 1 && d->nsplit != 3) {
    set_error("sfb_gemm_batched: nsplit must be 1 or 3");
    return -10;
  }
  if (d->m <= 0 || d->n <= 0 || d->k <= 0 || d->batch <= 0) {
    set_error("sfb_gemm_batched: bad extents m=%d n=%d k=%d batch=%d", d->m, d->n, d->k, d->batch);
    return -10;
  }
  if (d->ldd % 4 || d->batch_stride_d % 4) {
    set_error("sfb_gemm_batched: output pitch / batch stride must be multiples of 4 elements (16 B)");
    return -10;
  }
  if (d->lda % 8 || d->ldb % 8 || d->batch_stride_a % 8 || d->batch_stride_b % 8) {
    set_error("sfb_gemm_batched: operand pitches / batch strides must be multiples of 8 elements (16 B)");
    return -10;
  }
  if (!d->a_hi || !d->b_hi || !d->out || (d->nsplit == 3 && (!d->a_lo || !d->b_lo))) {
    set_error("sfb_gemm_batched: null operand pointer");
    return -10;
  }
  const int np = d->nsplit == 3 ? 2 : 1;
  BgemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = d->m; p.N = d->n; p.K = d->k; p.batch = d->batch;
  p.a_mn = d->a_mn_major ? 1 : 0;
  p.b_mn = d->b_mn_major ? 1 : 0;
  const int n16 = (d->n + 15) / 16 * 16;
  p.BN = std::min(n16, BG_BN_MAX);
  p.n_atoms = (p.BN + 63) / 64;
  p.m_tiles = (d->m + BG_BLOCK_M - 1) / BG_BLOCK_M;
  p.n_tiles = (d->n + p.BN - 1) / p.BN;
  p.k_blocks = (d->k + BG_BLOCK_K - 1) / BG_BLOCK_K;
  p.a_plane_bytes = 16384;
  p.b_plane_bytes = p.b_mn ? uint32_t(p.n_atoms) * 8192u : uint32_t((p.BN + 7) / 8 * 8) * 128u;
  p.b_plane_bytes = (p.b_plane_bytes + 1023) / 1024 * 1024;
  p.stage_bytes = (p.a_plane_bytes + p.b_plane_bytes) * np;
  p.acc_pitch = uint32_t(p.BN) + 4;
  const uint32_t acc_bytes = uint32_t(BG_BLOCK_M) * p.acc_pitch * 4u;
  const uint32_t tail = acc_bytes + 256;
  const uint32_t budget = uint32_t(bg_smem) - 1024 - tail;
  p.stages = std::min<int>(BG_MAX_STAGES, budget / p.stage_bytes);
  p.stages = std::min(p.stages, std::max(2, p.k_blocks * 4));
  if (p.stages < 2) {
    set_error("sfb_gemm_batched: not enough shared memory (stage=%u B)", p.stage_bytes);
    return -11;
  }
  p.off_acc = p.stages * p.stage_bytes;
  p.off_bars = p.off_acc + acc_bytes;
  const uint32_t smem_bytes = p.off_bars + 256 + 1024;
  p.out = d->out;
  p.ldd = d->ldd;
  p.batch_stride_d = d->batch_stride_d;
  p.alpha = d->alpha;
  p.accumulate = d->accumulate;

  int rc;
  for (int pl = 0; pl < np; ++pl) {
    const void* a = pl ? d->a_lo : d->a_hi;
    const void* b = pl ? d->b_lo : d->b_hi;
    rc = p.a_mn ? make_tmap_3d(&p.tmA[pl], a, d->m, d->k, d->batch, d->lda, d->batch_stride_a, 64)
                : make_tmap_3d(&p.tmA[pl], a, d->k, d->m, d->batch, d->lda, d->batch_stride_a, 128);
    if (rc) return rc;
    rc = p.b_mn ? make_tmap_3d(&p.tmB[pl], b, d->n, d->k, d->batch, d->ldb, d->batch_stride_b, 64)
                : make_tmap_3d(&p.tmB[pl], b, d->k, d->n, d->batch, d->ldb, d->batch_stride_b, uint32_t(p.BN));
    if (rc) return rc;
  }
  const int total_tiles = p.m_tiles * p.n_tiles * p.batch;
  // split-K when the tiles cannot fill half the machine, K is long, and the output is a dense [batch][M][N] block (it is
  // zeroed here unless the caller accumulates): at least 8 k-blocks (512 reduction elements) per split
  p.k_splits = 1;
  p.kb_per_split = p.k_blocks;
  static const bool splitk_on = [] { const char* e = getenv("SFB_BGEMM_SPLITK"); return e ? e[0] != '0' : true; }();
  if (splitk_on && total_tiles * 2 <= bg_sms && p.k_blocks >= 32 && d->ldd == d->n && d->batch_stride_d == int64_t(d->m) * d->ldd) {
    int want = std::min(bg_sms / total_tiles, p.k_blocks / 8);
    if (want > 1) {
      p.kb_per_split = (p.k_blocks + want - 1) / want;
      p.k_splits = (p.k_blocks + p.kb_per_split - 1) / p.kb_per_split;
      if (!d->accumulate)
        cudaMemsetAsync(d->out, 0, size_t(d->batch) * size_t(d->batch_stride_d) * sizeof(float), stream);
    }
  }
  const int grid = std::min(total_tiles * p.k_splits, bg_sms);
  if (d->nsplit == 3) {
    static bool a3 = false;
    if (!a3) {
      cudaFuncSetAttribute(gemm_batched_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, bg_smem);
      a3 = true;
    }
    gemm_batched_kernel<3><<<grid, BG_THREADS, smem_bytes, stream>>>(p);
  } else {
    static bool a1 = false;
    if (!a1) {
      cudaFuncSetAttribute(gemm_batched_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, bg_smem);
      a1 = true;
    }
    gemm_batched_kernel<1><<<grid, BG_THREADS, smem_bytes, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_gemm_batched launch failed: %s (grid=%d smem=%u stages=%d BN=%d)", cudaGetErrorString(e), grid,
              smem_bytes, p.stages, p.BN);
    return -20;
  }
  return 0;
}
