// HBM-bound companions of the tensor-core kernels: operand packing (fp32 -> split-bf16 planes, NCDHW -> NDHWC,
// filter matrices), train-mode BatchNorm (finalize / apply+residual+ReLU / backward), ReLU+MaxPool for the stems,
// and the classification head pieces.  All kernels view an activation as a [rows = n*t*h*w, C] matrix with a row
// pitch (so channel slices of a wider tensor - "concat in place" - need no copies) and move 8 channels per thread
// (16-byte bf16 / 32-byte fp32 vectors), grid-strided with a grid of a few waves of the
// device's SMs (runtime.h's kGridSms stands in when no device answers).
#include <cstdint>
#include <cstring>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "planes.cuh"
#include "runtime.h"

namespace sfb {

// SM count of the device; kGridSms when there is none (the launch that follows reports that)
static int ew_sms() {
  int sms = kGridSms;
  device_limits(&sms, nullptr);
  return sms;
}
static int ew_grid(int64_t items, int block) { return capped_grid(items, block, int64_t(ew_sms()) * 8); }
// grid of the row-lane kernels (RowLanes): every thread walks ~4 rows of its channel group, at most 8 blocks per SM
static int rowlane_grid(int64_t rows, int cg, int block) {
  const int lanes_c = cg < block ? cg : block;
  const int lanes_r = block / lanes_c;
  return capped_grid(rows, lanes_r * 4, int64_t(ew_sms()) * 8);
}

struct f32x8 {
  float4 a, b;
};

__device__ __forceinline__ void load8(const float* p, float (&x)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
  x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
}
__device__ __forceinline__ void store8(float* p, const float (&x)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(x[0], x[1], x[2], x[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(x[4], x[5], x[6], x[7]);
}
// ------------------------------------------------------------------------------------------- packing
__global__ void split_planes_kernel(const float* __restrict__ x, int64_t rows, int cg, int64_t x_pitch,
                                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int64_t o_pitch) {
  const int64_t items = rows * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cg;
    const int c = int(i - r * cg) * 8;
    float v[8];
    load8(x + r * x_pitch + c, v);
    store_split8(hi + r * o_pitch + c, lo ? lo + r * o_pitch + c : nullptr, v);
  }
}

// NCDHW fp32 -> NDHWC split planes with the channel count padded to c_pad (zeros)
__global__ void input_pack_kernel(const float* __restrict__ x, int n, int c, int64_t thw, int c_pad,
                                  __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int64_t items = int64_t(n) * thw * (c_pad / 8);
  const int cg = c_pad / 8;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int g = int(i % cg);
    const int64_t pos = i / cg;  // n*thw + s
    const int64_t b = pos / thw, s = pos - b * thw;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = g * 8 + j;
      v[j] = ch < c ? x[(b * c + ch) * thw + s] : 0.f;
    }
    store_split8(hi + pos * c_pad + g * 8, lo ? lo + pos * c_pad + g * 8 : nullptr, v);
  }
}

// Filter matrix for the implicit GEMM: out[r][j][cc] (bf16 planes), r < rows, j < ntaps, cc < cols_pad
//   transpose == 0 (fprop / wgrad layout): r = co, cc = ci   -> w[co][ci][tapmap[j]]
//   transpose == 1 (dgrad):                r = ci, cc = co   -> w[co][ci][tapmap[j]]
struct FilterPackParams {
  const float* w;
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
  int cout, cin, taps_total, ntaps, rows, cols, cols_pad, transpose;
  int16_t tapmap[256];
};
__global__ void filter_pack_kernel(const __grid_constant__ FilterPackParams p) {
  const int64_t items = int64_t(p.rows) * p.ntaps * p.cols_pad;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int cc = int(i % p.cols_pad);
    const int64_t t = i / p.cols_pad;
    const int j = int(t % p.ntaps);
    const int r = int(t / p.ntaps);
    float v = 0.f;
    if (cc < p.cols) {
      const int co = p.transpose ? cc : r;
      const int ci = p.transpose ? r : cc;
      v = p.w[(int64_t(co) * p.cin + ci) * p.taps_total + p.tapmap[j]];
    }
    put_split(p.hi, p.lo, i, v);
  }
}

// wgrad matrix [cout][taps][cin_pad] (fp32) -> parameter-gradient layout [cout][cin][taps]
__global__ void filter_unpack_grad_kernel(const float* __restrict__ dwm, float* __restrict__ dw, int cout, int cin,
                                          int taps, int cin_pad, int accumulate) {
  const int64_t items = int64_t(cout) * cin * taps;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int tap = int(i % taps);
    const int64_t t = i / taps;
    const int ci = int(t % cin);
    const int co = int(t / cin);
    const float v = dwm[(int64_t(co) * taps + tap) * cin_pad + ci];
    dw[i] = accumulate ? dw[i] + v : v;
  }
}

// ------------------------------------------------------------------------------------------- BatchNorm forward
// Merge the conv epilogue's per-tile (sum, sum^2) partials in fp64, produce the affine (scale, shift) the apply
// kernel uses, save (mean, invstd) for backward and update the running statistics exactly like
// torch.nn.BatchNorm3d in train mode (biased variance for normalisation, unbiased for running_var).
// affine_c: period of gamma / beta.  SubBatchNorm3d finalizes its S*C split_bn channels against ONE shared [C] affine.
__global__ void __launch_bounds__(256) bn_finalize_kernel(const float* __restrict__ partials, int m_tiles, int c,
                                                          int affine_c, double count, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float* __restrict__ running_mean,
                                                          float* __restrict__ running_var, float momentum, float eps,
                                                          int training, float* __restrict__ scale,
                                                          float* __restrict__ shift, float* __restrict__ save_mean,
                                                          float* __restrict__ save_invstd) {
  // one block per channel; partials are laid out [2][c][m_tiles] so that the tile axis is contiguous
  __shared__ double sm1[256], sm2[256];
  const int ch = blockIdx.x;
  float mean_f, invstd_f;
  if (training) {
    const float* p1 = partials + size_t(ch) * m_tiles;
    const float* p2 = partials + (size_t(c) + ch) * m_tiles;
    double s = 0.0, s2 = 0.0;
    for (int t = threadIdx.x; t < m_tiles; t += 256) {
      s += double(p1[t]);
      s2 += double(p2[t]);
    }
    sm1[threadIdx.x] = s;
    sm2[threadIdx.x] = s2;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        sm1[threadIdx.x] += sm1[threadIdx.x + o];
        sm2[threadIdx.x] += sm2[threadIdx.x + o];
      }
      __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const double mean = sm1[0] / count;
    double var = sm2[0] / count - mean * mean;
    if (var < 0.0) var = 0.0;
    mean_f = float(mean);
    invstd_f = float(1.0 / sqrt(var + double(eps)));
    if (running_mean) {
      const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
      running_mean[ch] = float((1.0 - momentum) * double(running_mean[ch]) + momentum * mean);
      running_var[ch] = float((1.0 - momentum) * double(running_var[ch]) + momentum * unbiased);
    }
  } else {
    if (threadIdx.x != 0) return;
    mean_f = running_mean[ch];
    invstd_f = float(1.0 / sqrt(double(running_var[ch]) + double(eps)));
  }
  const int ca = ch % affine_c;
  const float g = gamma ? gamma[ca] : 1.f, b = beta ? beta[ca] : 0.f;
  scale[ch] = g * invstd_f;
  shift[ch] = b - mean_f * g * invstd_f;
  if (save_mean) save_mean[ch] = mean_f;
  if (save_invstd) save_invstd[ch] = invstd_f;
}

// Training statistics of SubBatchNorm3d (batchnorm_helper.py:101-106, x.view(n // S, C*S, t, h, w)): clip k of the
// batch is in split s = k % S and its channel c is split_bn channel s*C + c.  Every block sums one chunk of rows of ONE
// clip, so no partial mixes splits (the conv epilogue's 128-row tiles cross clip boundaries); the partials are laid out
// [2][S*C][blocks_per_split] (column = (k / S) * chunks + chunk), so sfb_bn_finalize reduces them as S*C channels.
// Rows per block: 8 per row lane, at least 128 (the tile height of the conv epilogue's partials).  256 threads cover
// min(C/8, 256) channel groups, so a narrow layer has many row lanes: C = 8 (the fast stem) takes 2048-row chunks.
__host__ __device__ inline int64_t split_stats_chunk(int c) {
  const int cg = c / 8;
  const int lanes_r = 256 / (cg < 256 ? cg : 256);
  return lanes_r * 8 > 128 ? lanes_r * 8 : 128;
}
struct SplitStatsParams {
  const float* y; int64_t y_pitch;
  int64_t rows_per_clip; int64_t chunk_rows;
  int c, splits, chunks, blocks_per_split;
  float* partials;
};
__global__ void __launch_bounds__(256) bn_split_stats_kernel(const SplitStatsParams p) {
  extern __shared__ float sm[];  // [blockDim.x][16]
  const int cg = p.c / 8;
  const int lanes_c = cg < int(blockDim.x) ? cg : int(blockDim.x);
  const int lanes_r = blockDim.x / lanes_c;
  const int lc = threadIdx.x % lanes_c;
  const int lr = threadIdx.x / lanes_c;
  const int64_t clip = blockIdx.x / p.chunks;
  const int j = int(blockIdx.x % p.chunks);
  const int s = int(clip % p.splits);
  const int col = int(clip / p.splits) * p.chunks + j;
  const int64_t r0 = clip * p.rows_per_clip + j * p.chunk_rows;
  const int64_t r1 = min(r0 + p.chunk_rows, (clip + 1) * p.rows_per_clip);
  const int64_t sq = int64_t(p.splits) * p.c * p.blocks_per_split;  // start of the sum-of-squares half
  for (int g0 = 0; g0 < cg; g0 += lanes_c) {
    const int g = g0 + lc;
    float s1[8], s2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s1[k] = s2[k] = 0.f;
    if (g < cg && lr < lanes_r) {
      for (int64_t r = r0 + lr; r < r1; r += lanes_r) {
        float v[8];
        load8(p.y + r * p.y_pitch + g * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          s1[k] += v[k];
          s2[k] = fmaf(v[k], v[k], s2[k]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      sm[threadIdx.x * 16 + k] = s1[k];
      sm[threadIdx.x * 16 + 8 + k] = s2[k];
    }
    __syncthreads();
    if (lr == 0 && g < cg) {
      for (int q = 1; q < lanes_r; ++q) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          s1[k] += sm[(q * lanes_c + lc) * 16 + k];
          s2[k] += sm[(q * lanes_c + lc) * 16 + 8 + k];
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int64_t ch = int64_t(s) * p.c + g * 8 + k;
        p.partials[ch * p.blocks_per_split + col] = s1[k];
        p.partials[sq + ch * p.blocks_per_split + col] = s2[k];
      }
    }
    __syncthreads();
  }
}

// out = act( y*scale + shift  [+ y2*scale2 + shift2]  [+ (r_hi + r_lo)] ), written as split planes
// splits > 1 (SubBatchNorm3d in training): the coefficient vectors are [splits][c] tables and row r uses row
// (r / rows_per_clip) % splits of them.
struct BnApplyParams {
  const float* y; int64_t y_pitch;
  const float* scale; const float* shift;
  const float* y2; int64_t y2_pitch;
  const float* scale2; const float* shift2;
  const __nv_bfloat16* r_hi; const __nv_bfloat16* r_lo; int64_t r_pitch;
  __nv_bfloat16* o_hi; __nv_bfloat16* o_lo; int64_t o_pitch;
  int64_t rows; int c; int relu;
  int splits; int64_t rows_per_clip;
};
__device__ __forceinline__ int split_of_row(int64_t r, int64_t rows_per_clip, int splits) {
  return int((r / rows_per_clip) % splits);
}
// Thread mapping of the BatchNorm elementwise passes: a thread owns ONE 8-channel group (its per-channel coefficients are
// loaded once, outside the row loop - ncu r2c showed the L1 at 71 % busy re-reading five coefficient vectors per item) and
// walks rows; consecutive lanes = consecutive channel groups (contiguous 32-byte pieces of a row), remaining lanes = rows.
struct RowLanes {
  int lanes_c, lanes_r, lc, lr;
  __device__ __forceinline__ RowLanes(int cg) {
    lanes_c = cg < int(blockDim.x) ? cg : int(blockDim.x);
    lanes_r = blockDim.x / lanes_c;
    lc = threadIdx.x % lanes_c;
    lr = threadIdx.x / lanes_c;
  }
};
__global__ void __launch_bounds__(256) bn_apply_kernel(const BnApplyParams p) {
  const int cg = p.c / 8;
  const RowLanes L(cg);
  if (L.lr >= L.lanes_r) return;
  for (int g = L.lc; g < cg; g += L.lanes_c) {
    const int c = g * 8;
    float sc[8], sh[8], sc2[8], sh2[8];
    load8(p.scale + c, sc);
    load8(p.shift + c, sh);
    if (p.y2) {
      load8(p.scale2 + c, sc2);
      load8(p.shift2 + c, sh2);
    }
    int cur = 0;  // coefficient row held in registers
    for (int64_t r = int64_t(blockIdx.x) * L.lanes_r + L.lr; r < p.rows; r += int64_t(gridDim.x) * L.lanes_r) {
      if (p.splits > 1) {
        const int s = split_of_row(r, p.rows_per_clip, p.splits);
        if (s != cur) {
          cur = s;
          const int64_t o = int64_t(s) * p.c + c;
          load8(p.scale + o, sc);
          load8(p.shift + o, sh);
          if (p.y2) {
            load8(p.scale2 + o, sc2);
            load8(p.shift2 + o, sh2);
          }
        }
      }
      float v[8];
      load8(p.y + r * p.y_pitch + c, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], sc[j], sh[j]);
      if (p.y2) {
        float w[8];
        load8(p.y2 + r * p.y2_pitch + c, w);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += fmaf(w[j], sc2[j], sh2[j]);
      }
      if (p.r_hi) {
        float w[8];
        load_planes8(p.r_hi + r * p.r_pitch + c, p.r_lo ? p.r_lo + r * p.r_pitch + c : nullptr, w);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += w[j];
      }
      if (p.relu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
      }
      store_split8(p.o_hi + r * p.o_pitch + c, p.o_lo ? p.o_lo + r * p.o_pitch + c : nullptr, v);
    }
  }
}

// ------------------------------------------------------------------------------------------- BatchNorm backward
// pass 1: per-channel  S1 = sum dz,  S2 = sum dz * xhat   with dz = dout * (mask > 0)   (mask = post-ReLU plane)
// Each block owns a contiguous slab of rows and writes one partial row; the finalize kernel merges them in fp64.
struct BnBwdReduceParams {
  const float* dout; int64_t dout_pitch;
  const __nv_bfloat16* mask; int64_t mask_pitch;   // may be null (no ReLU after this BN)
  const float* y; int64_t y_pitch;
  const float* mean; const float* invstd;
  int64_t rows; int c;
  float* partials;  // [gridDim.x][2][c]
  const float* mask_scale; const float* mask_shift;  // alternative ReLU mask: y*scale + shift > 0 (no planes kept)
  // splits > 1: mean / invstd / mask_scale / mask_shift are [splits][c] tables and every block reduces a slab of ONE
  // clip (blocks_per_clip slabs per clip), so its partial row belongs to split (blockIdx.x / blocks_per_clip) % splits
  int splits; int64_t rows_per_clip; int blocks_per_clip;
};
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const BnBwdReduceParams p) {
  extern __shared__ float sm[];  // [blockDim.x][16]
  const int cg = p.c / 8;
  // channel groups are covered in passes of min(cg, blockDim.x) lanes; rows are split over row-lanes and blocks
  const int lanes_c = cg < int(blockDim.x) ? cg : int(blockDim.x);
  const int lanes_r = blockDim.x / lanes_c;
  const int lc = threadIdx.x % lanes_c;
  const int lr = threadIdx.x / lanes_c;
  int64_t r0, r1, coff = 0;
  if (p.splits > 1) {
    const int64_t clip = blockIdx.x / p.blocks_per_clip;
    const int64_t rpb = (p.rows_per_clip + p.blocks_per_clip - 1) / p.blocks_per_clip;
    r0 = clip * p.rows_per_clip + (blockIdx.x % p.blocks_per_clip) * rpb;
    r1 = min(r0 + rpb, (clip + 1) * p.rows_per_clip);
    coff = (clip % p.splits) * p.c;
  } else {
    const int64_t rows_per_block = (p.rows + gridDim.x - 1) / gridDim.x;
    r0 = blockIdx.x * rows_per_block;
    r1 = (r0 + rows_per_block < p.rows) ? r0 + rows_per_block : p.rows;
  }
  for (int g0 = 0; g0 < cg; g0 += lanes_c) {
    const int g = g0 + lc;
    float s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s1[j] = s2[j] = 0.f;
    if (g < cg && lr < lanes_r) {
      const int c = g * 8;
      float mu[8], is[8], msc[8], msh[8];
      load8(p.mean + coff + c, mu);
      load8(p.invstd + coff + c, is);
      if (p.mask_scale) {
        load8(p.mask_scale + coff + c, msc);
        load8(p.mask_shift + coff + c, msh);
      }
      for (int64_t r = r0 + lr; r < r1; r += lanes_r) {
        float d[8], yv[8];
        load8(p.dout + r * p.dout_pitch + c, d);
        load8(p.y + r * p.y_pitch + c, yv);
        if (p.mask) {
          float m[8];
          load_planes8(p.mask + r * p.mask_pitch + c, nullptr, m);
#pragma unroll
          for (int j = 0; j < 8; ++j) d[j] = m[j] > 0.f ? d[j] : 0.f;
        } else if (p.mask_scale) {
#pragma unroll
          for (int j = 0; j < 8; ++j) d[j] = fmaf(yv[j], msc[j], msh[j]) > 0.f ? d[j] : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1[j] += d[j];
          s2[j] = fmaf(d[j], (yv[j] - mu[j]) * is[j], s2[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sm[threadIdx.x * 16 + j] = s1[j];
      sm[threadIdx.x * 16 + 8 + j] = s2[j];
    }
    __syncthreads();
    if (lr == 0 && g < cg) {
      for (int k = 1; k < lanes_r; ++k) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1[j] += sm[(k * lanes_c + lc) * 16 + j];
          s2[j] += sm[(k * lanes_c + lc) * 16 + 8 + j];
        }
      }
      float* out = p.partials + size_t(blockIdx.x) * 2 * p.c;
      store8(out + g * 8, s1);
      store8(out + p.c + g * 8, s2);
    }
    __syncthreads();
  }
}

// merge partials -> dgamma (+=), dbeta (+=) and the two per-channel coefficients of pass 2:
//   dy = a * dz - b - xhat * cc     with a = gamma*invstd, b = a*S1/M, cc = a*S2/M
// In eval mode (training == 0) the statistics are constants: dy = a * dz.
// splits > 1: the sums are taken per (split, channel) over that split's blocks (see bn_bwd_reduce_kernel), the
// coefficients become [3][splits][c] and count is the rows of one split; gamma is shared, so dgamma / dbeta are the sums
// over all splits.
__global__ void __launch_bounds__(64) bn_bwd_finalize_kernel(const float* __restrict__ partials, int nblocks, int c,
                                                             double count, const float* __restrict__ gamma,
                                                             const float* __restrict__ invstd,
                                                             float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                             int accumulate, int training,
                                                             float* __restrict__ coef /* [3][splits][c] */, int c_valid,
                                                             int splits, int blocks_per_clip) {
  // one 64-thread block per channel: the row-slab partials are merged in fp64 with a fixed (deterministic) tree
  __shared__ double sm1[64], sm2[64];
  const int ch = blockIdx.x;
  const int sc = splits * c;
  if (ch >= c_valid) {  // padding channel: its activations and gradients are exact zeros
    if (threadIdx.x == 0)
      for (int s = 0; s < splits; ++s) coef[s * c + ch] = coef[sc + s * c + ch] = coef[2 * sc + s * c + ch] = 0.f;
    return;
  }
  const int nb_split = nblocks / splits;
  double t1 = 0.0, t2 = 0.0;
  for (int s = 0; s < splits; ++s) {
    double s1 = 0.0, s2 = 0.0;
    for (int i = threadIdx.x; i < nb_split; i += 64) {
      const int b = splits > 1 ? ((i / blocks_per_clip) * splits + s) * blocks_per_clip + i % blocks_per_clip : i;
      s1 += double(partials[size_t(b) * 2 * c + ch]);
      s2 += double(partials[size_t(b) * 2 * c + c + ch]);
    }
    sm1[threadIdx.x] = s1;
    sm2[threadIdx.x] = s2;
    __syncthreads();
    for (int o = 32; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        sm1[threadIdx.x] += sm1[threadIdx.x + o];
        sm2[threadIdx.x] += sm2[threadIdx.x + o];
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      s1 = sm1[0];
      s2 = sm2[0];
      t1 += s1;
      t2 += s2;
      const double a = double(gamma ? gamma[ch] : 1.f) * double(invstd[s * c + ch]);
      coef[s * c + ch] = float(a);
      coef[sc + s * c + ch] = training ? float(a * s1 / count) : 0.f;
      coef[2 * sc + s * c + ch] = training ? float(a * s2 / count) : 0.f;
    }
    __syncthreads();  // sm1 / sm2 are refilled by the next split
  }
  if (threadIdx.x != 0) return;
  if (dgamma) dgamma[ch] = accumulate ? dgamma[ch] + float(t2) : float(t2);
  if (dbeta) dbeta[ch] = accumulate ? dbeta[ch] + float(t1) : float(t1);
}

// pass 2: dy = a*dz - b - xhat*cc  -> split planes for the dgrad / wgrad GEMMs; optionally also emits
// dz itself (fp32) as the gradient flowing into an identity shortcut (dres, either stored or accumulated).
struct BnBwdApplyParams {
  const float* dout; int64_t dout_pitch;
  const __nv_bfloat16* mask; int64_t mask_pitch;
  const float* y; int64_t y_pitch;
  const float* mean; const float* invstd; const float* coef;
  __nv_bfloat16* dy_hi; __nv_bfloat16* dy_lo; int64_t dy_pitch;
  float* dres; int64_t dres_pitch; int dres_accumulate;
  int64_t rows; int c;
  const float* mask_scale; const float* mask_shift;
  int splits; int64_t rows_per_clip;  // splits > 1: [splits][c] statistics / mask tables, [3][splits][c] coefficients
};
struct BnBwdCoef {
  float mu[8], ca[8], cb[8], k1[8], msc[8], msh[8];
  // dy = ca*dz - cb - (y - mu)*is*cc  =  ca*dz - (y - mu)*k1 - cb   with k1 = is*cc
  __device__ __forceinline__ void load(const BnBwdApplyParams& p, int s, int c) {
    const int64_t o = int64_t(s) * p.c + c, sc = int64_t(p.splits > 1 ? p.splits : 1) * p.c;
    float is[8], cc[8];
    load8(p.mean + o, mu);
    load8(p.invstd + o, is);
    load8(p.coef + o, ca);
    load8(p.coef + sc + o, cb);
    load8(p.coef + 2 * sc + o, cc);
#pragma unroll
    for (int j = 0; j < 8; ++j) k1[j] = is[j] * cc[j];
    if (p.mask_scale) {
      load8(p.mask_scale + o, msc);
      load8(p.mask_shift + o, msh);
    }
  }
};
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const BnBwdApplyParams p) {
  const int cg = p.c / 8;
  const RowLanes L(cg);
  if (L.lr >= L.lanes_r) return;
  for (int g = L.lc; g < cg; g += L.lanes_c) {
    const int c = g * 8;
    BnBwdCoef k;  // per-channel coefficients, loaded once per split change
    k.load(p, 0, c);
    float (&mu)[8] = k.mu, (&ca)[8] = k.ca, (&cb)[8] = k.cb, (&k1)[8] = k.k1, (&msc)[8] = k.msc, (&msh)[8] = k.msh;
    int cur = 0;
    for (int64_t r = int64_t(blockIdx.x) * L.lanes_r + L.lr; r < p.rows; r += int64_t(gridDim.x) * L.lanes_r) {
      if (p.splits > 1) {
        const int s = split_of_row(r, p.rows_per_clip, p.splits);
        if (s != cur) {
          cur = s;
          k.load(p, s, c);
        }
      }
      float d[8], yv[8];
      load8(p.dout + r * p.dout_pitch + c, d);
      load8(p.y + r * p.y_pitch + c, yv);
      if (p.mask) {
        float m[8];
        load_planes8(p.mask + r * p.mask_pitch + c, nullptr, m);
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = m[j] > 0.f ? d[j] : 0.f;
      } else if (p.mask_scale) {
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = fmaf(yv[j], msc[j], msh[j]) > 0.f ? d[j] : 0.f;
      }
      if (p.dres) {
        float* dr = p.dres + r * p.dres_pitch + c;
        if (p.dres_accumulate) {
          float o[8];
          load8(dr, o);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += d[j];
          store8(dr, o);
        } else {
          store8(dr, d);
        }
      }
      float gq[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) gq[j] = ca[j] * d[j] - cb[j] - (yv[j] - mu[j]) * k1[j];
      store_split8(p.dy_hi + r * p.dy_pitch + c, p.dy_lo ? p.dy_lo + r * p.dy_pitch + c : nullptr, gq);
    }
  }
}

// ------------------------------------------------------------------------------------------- stem: BN+ReLU+MaxPool
// out = maxpool_{1 x kh x kw, stride (1,sh,sw), pad (0,ph,pw)}( relu(y*scale+shift) ), first-maximum semantics
// (ties -> lowest (h,w) scan index, as torch).  argmax (uint8 window index, 255 = "max is not positive": the
// gradient dies in the ReLU) is saved for backward.
struct PoolParams {
  const float* y; const float* scale; const float* shift;
  int n, t, h, w, c; int oh, ow; int kh, kw, sh, sw, ph, pw;
  __nv_bfloat16* o_hi; __nv_bfloat16* o_lo; int64_t o_pitch;
  uint8_t* argmax;
  // backward
  const float* dout; int64_t dout_pitch; float* dz;
  int splits;  // > 1: scale / shift are [splits][c] tables, clip n uses row n % splits
};
// (4 blocks of 256 per SM, the occupancy this memory-bound pass had before the split index was added: <= 64 registers)
__global__ void __launch_bounds__(256, 4) bn_relu_maxpool_fwd_kernel(const PoolParams p) {
  const int cg = p.c / 8;
  const int64_t items = int64_t(p.n) * p.t * p.oh * p.ow * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int g = int(i % cg);
    int64_t pos = i / cg;
    const int ox = int(pos % p.ow);
    int64_t t2 = pos / p.ow;
    const int oy = int(t2 % p.oh);
    const int64_t nt = t2 / p.oh;  // n*t + tt
    const int c = g * 8;
    float sc[8], sh[8], best[8];
    uint8_t arg[8];
    const int64_t co = p.splits > 1 ? int64_t((nt / p.t) % p.splits) * p.c + c : c;
    load8(p.scale + co, sc);
    load8(p.shift + co, sh);
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = 255; }
    for (int ky = 0; ky < p.kh; ++ky) {
      const int iy = oy * p.sh - p.ph + ky;
      if (iy < 0 || iy >= p.h) continue;
      for (int kx = 0; kx < p.kw; ++kx) {
        const int ix = ox * p.sw - p.pw + kx;
        if (ix < 0 || ix >= p.w) continue;
        float v[8];
        load8(p.y + ((nt * p.h + iy) * p.w + ix) * int64_t(p.c) + c, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float z = fmaxf(fmaf(v[j], sc[j], sh[j]), 0.f);
          if (z > best[j]) { best[j] = z; arg[j] = uint8_t(ky * p.kw + kx); }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) if (!(best[j] > 0.f)) arg[j] = 255;
    store_split8(p.o_hi + pos * p.o_pitch + c, p.o_lo ? p.o_lo + pos * p.o_pitch + c : nullptr, best);
    *reinterpret_cast<uint2*>(p.argmax + pos * p.c + c) =
        make_uint2(arg[0] | (arg[1] << 8) | (arg[2] << 16) | (uint32_t(arg[3]) << 24),
                   arg[4] | (arg[5] << 8) | (arg[6] << 16) | (uint32_t(arg[7]) << 24));
  }
}
// dz[n,t,iy,ix,c] = sum over pooled outputs whose saved argmax points at (iy,ix) of dout   (gather form, no atomics)
__global__ void bn_relu_maxpool_bwd_kernel(const PoolParams p) {
  const int cg = p.c / 8;
  const int64_t items = int64_t(p.n) * p.t * p.h * p.w * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int g = int(i % cg);
    int64_t pos = i / cg;
    const int ix = int(pos % p.w);
    int64_t t2 = pos / p.w;
    const int iy = int(t2 % p.h);
    const int64_t nt = t2 / p.h;
    const int c = g * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // outputs oy with oy*sh - ph <= iy <= oy*sh - ph + kh - 1
    const int oy_lo = max(0, (iy + p.ph - p.kh + p.sh) / p.sh), oy_hi = min(p.oh - 1, (iy + p.ph) / p.sh);
    const int ox_lo = max(0, (ix + p.pw - p.kw + p.sw) / p.sw), ox_hi = min(p.ow - 1, (ix + p.pw) / p.sw);
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      const int ky = iy - (oy * p.sh - p.ph);
      if (ky < 0 || ky >= p.kh) continue;
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const int kx = ix - (ox * p.sw - p.pw);
        if (kx < 0 || kx >= p.kw) continue;
        const int64_t opos = (nt * p.oh + oy) * p.ow + ox;
        const uint2 am = *reinterpret_cast<const uint2*>(p.argmax + opos * p.c + c);
        float d[8];
        load8(p.dout + opos * p.dout_pitch + c, d);
        const uint32_t want = uint32_t(ky * p.kw + kx);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t a = ((j < 4 ? am.x : am.y) >> (8 * (j & 3))) & 0xffu;
          if (a == want) acc[j] += d[j];
        }
      }
    }
    store8(p.dz + pos * p.c + c, acc);
  }
}

}  // namespace sfb

using namespace sfb;
typedef __nv_bfloat16 bf16;

extern "C" int sfb_split_planes(const float* x, int64_t rows, int32_t c, int64_t x_pitch, void* hi, void* lo,
                                int64_t o_pitch, void* stream) {
  if (c % 8 || x_pitch % 4 || o_pitch % 8) {
    set_error("sfb_split_planes: c=%d must be a multiple of 8 (pitches 16-byte aligned)", c);
    return -10;
  }
  const int64_t items = rows * (c / 8);
  if (items == 0) return 0;
  split_planes_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(x, rows, c / 8, x_pitch, (bf16*)hi,
                                                                            (bf16*)lo, o_pitch);
  return launch_status("sfb_split_planes");
}

extern "C" int sfb_input_pack(const float* x, int32_t n, int32_t c, int32_t t, int32_t h, int32_t w, int32_t c_pad,
                              void* hi, void* lo, void* stream) {
  if (c_pad % 8 || c_pad < c) {
    set_error("sfb_input_pack: c_pad=%d must be a multiple of 8 and >= c=%d", c_pad, c);
    return -10;
  }
  const int64_t thw = int64_t(t) * h * w;
  const int64_t items = int64_t(n) * thw * (c_pad / 8);
  input_pack_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(x, n, c, thw, c_pad, (bf16*)hi, (bf16*)lo);
  return launch_status("sfb_input_pack");
}

extern "C" int sfb_filter_pack(const float* w, int32_t cout, int32_t cin, int32_t taps_total, const int32_t* tapmap,
                               int32_t ntaps, int32_t transpose, int32_t cols_pad, void* hi, void* lo, void* stream) {
  if (ntaps < 1 || ntaps > 256) {
    set_error("sfb_filter_pack: ntaps=%d outside [1,256]", ntaps);
    return -10;
  }
  FilterPackParams p;
  memset(&p, 0, sizeof(p));
  p.w = w; p.hi = (bf16*)hi; p.lo = (bf16*)lo;
  p.cout = cout; p.cin = cin; p.taps_total = taps_total; p.ntaps = ntaps;
  p.transpose = transpose;
  p.rows = transpose ? cin : cout;
  p.cols = transpose ? cout : cin;
  p.cols_pad = cols_pad;
  if (cols_pad < p.cols) {
    set_error("sfb_filter_pack: cols_pad=%d < cols=%d", cols_pad, p.cols);
    return -10;
  }
  for (int j = 0; j < ntaps; ++j) {
    const int tm = tapmap ? tapmap[j] : j;
    if (tm < 0 || tm >= taps_total) {
      set_error("sfb_filter_pack: tapmap[%d]=%d outside [0,%d)", j, tm, taps_total);
      return -10;
    }
    p.tapmap[j] = int16_t(tm);
  }
  const int64_t items = int64_t(p.rows) * ntaps * cols_pad;
  filter_pack_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_filter_pack");
}

extern "C" int sfb_filter_unpack_grad(const float* dwm, float* dw, int32_t cout, int32_t cin, int32_t taps,
                                      int32_t cin_pad, int32_t accumulate, void* stream) {
  const int64_t items = int64_t(cout) * cin * taps;
  filter_unpack_grad_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dwm, dw, cout, cin, taps, cin_pad,
                                                                                  accumulate);
  return launch_status("sfb_filter_unpack_grad");
}

extern "C" int sfb_bn_finalize(const float* partials, int32_t m_tiles, int32_t c, int64_t count, const float* gamma,
                               const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                               int32_t training, float* scale, float* shift, float* save_mean, float* save_invstd,
                               int32_t affine_c, void* stream) {
  if (!training && (!running_mean || !running_var)) {
    set_error("sfb_bn_finalize: eval mode needs running statistics");
    return -10;
  }
  if (affine_c <= 0) affine_c = c;
  if (c % affine_c) {
    set_error("sfb_bn_finalize: affine period %d does not divide c=%d", affine_c, c);
    return -10;
  }
  bn_finalize_kernel<<<c, 256, 0, (cudaStream_t)stream>>>(partials, m_tiles, c, affine_c, double(count), gamma,
                                                                       beta, running_mean, running_var, momentum, eps,
                                                                       training, scale, shift, save_mean, save_invstd);
  return launch_status("sfb_bn_finalize");
}

static int split_geometry_ok(const char* who, int64_t rows, int32_t splits, int64_t rows_per_clip) {
  if (splits <= 1) return 1;
  if (rows_per_clip <= 0 || rows % rows_per_clip || (rows / rows_per_clip) % splits) {
    set_error("%s: %lld rows are not whole clips of %lld rows in a multiple of %d splits", who, (long long)rows,
              (long long)rows_per_clip, splits);
    return 0;
  }
  return 1;
}

extern "C" int32_t sfb_bn_split_stats_tiles(int64_t rows, int64_t rows_per_clip, int32_t splits, int32_t c) {
  if (rows_per_clip <= 0 || splits <= 0 || c < 8) return 0;
  const int64_t chunk = split_stats_chunk(c);
  const int64_t chunks = (rows_per_clip + chunk - 1) / chunk;
  return int32_t(rows / rows_per_clip / splits * chunks);
}

extern "C" int sfb_bn_split_stats(const float* y, int64_t y_pitch, int64_t rows, int32_t c, int32_t splits,
                                  int64_t rows_per_clip, float* partials, void* stream) {
  if (c % 8 || y_pitch % 4 || splits < 1 || rows_per_clip <= 0 || rows % rows_per_clip ||
      (rows / rows_per_clip) % splits) {
    set_error("sfb_bn_split_stats: c=%d (a multiple of 8), %lld rows in clips of %lld rows, %d splits", c,
              (long long)rows, (long long)rows_per_clip, splits);
    return -10;
  }
  SplitStatsParams p;
  p.y = y; p.y_pitch = y_pitch; p.rows_per_clip = rows_per_clip; p.chunk_rows = split_stats_chunk(c);
  p.c = c; p.splits = splits;
  p.chunks = int((rows_per_clip + p.chunk_rows - 1) / p.chunk_rows);
  p.blocks_per_split = sfb_bn_split_stats_tiles(rows, rows_per_clip, splits, c);
  p.partials = partials;
  const int64_t blocks = rows / rows_per_clip * p.chunks;
  if (blocks == 0) return 0;
  bn_split_stats_kernel<<<unsigned(blocks), 256, 256 * 16 * sizeof(float), (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bn_split_stats");
}

extern "C" int sfb_bn_apply(const sfb_bn_apply_desc* d, void* stream) {
  if (d->c % 8) {
    set_error("sfb_bn_apply: c=%d must be a multiple of 8", d->c);
    return -10;
  }
  if (!split_geometry_ok("sfb_bn_apply", d->rows, d->splits, d->rows_per_clip)) return -10;
  BnApplyParams p;
  p.y = d->y; p.y_pitch = d->y_pitch; p.scale = d->scale; p.shift = d->shift;
  p.y2 = d->y2; p.y2_pitch = d->y2_pitch; p.scale2 = d->scale2; p.shift2 = d->shift2;
  p.r_hi = (const bf16*)d->res_hi; p.r_lo = (const bf16*)d->res_lo; p.r_pitch = d->res_pitch;
  p.o_hi = (bf16*)d->out_hi; p.o_lo = (bf16*)d->out_lo; p.o_pitch = d->out_pitch;
  p.rows = d->rows; p.c = d->c; p.relu = d->relu;
  p.splits = d->splits > 1 ? d->splits : 1; p.rows_per_clip = d->rows_per_clip;
  const int64_t items = d->rows * (d->c / 8);
  if (items == 0) return 0;
  bn_apply_kernel<<<rowlane_grid(d->rows, d->c / 8, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bn_apply");
}

static int64_t bn_bwd_slabs(int64_t rows) {
  // enough row slabs to fill the machine; at least 16 rows per slab (ncu r2c: 64-row slabs gave 196 blocks = 16 % active
  // warps on a 12.5 k-row layer)
  int64_t b = (rows + 15) / 16;
  const int64_t cap = int64_t(ew_sms()) * 4;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return b;
}

// slabs per clip of the split reduce: about as many blocks in all as the unsplit reduce, none straddling a clip
static int32_t bn_bwd_blocks_per_clip(int64_t rows, int64_t rows_per_clip) {
  const int64_t clips = rows / rows_per_clip;
  int64_t per = (bn_bwd_slabs(rows) + clips - 1) / clips;
  const int64_t most = (rows_per_clip + 15) / 16;
  if (per > most) per = most;
  return int32_t(per < 1 ? 1 : per);
}

extern "C" int32_t sfb_bn_bwd_blocks(int64_t rows, int32_t c, int32_t splits, int64_t rows_per_clip) {
  (void)c;
  if (splits > 1 && rows_per_clip > 0)
    return int32_t(rows / rows_per_clip * bn_bwd_blocks_per_clip(rows, rows_per_clip));
  return int32_t(bn_bwd_slabs(rows));
}

extern "C" int sfb_bn_bwd(const sfb_bn_bwd_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (d->c % 8) {
    set_error("sfb_bn_bwd: c=%d must be a multiple of 8", d->c);
    return -10;
  }
  if (!split_geometry_ok("sfb_bn_bwd", d->rows, d->splits, d->rows_per_clip)) return -10;
  const int splits = d->splits > 1 ? d->splits : 1;
  const int nblocks = sfb_bn_bwd_blocks(d->rows, d->c, splits, d->rows_per_clip);
  const int bpc = splits > 1 ? bn_bwd_blocks_per_clip(d->rows, d->rows_per_clip) : 1;
  BnBwdReduceParams r;
  r.dout = d->dout; r.dout_pitch = d->dout_pitch;
  r.mask = (const bf16*)d->mask_hi; r.mask_pitch = d->mask_pitch;
  r.mask_scale = d->mask_scale; r.mask_shift = d->mask_shift;
  r.y = d->y; r.y_pitch = d->y_pitch; r.mean = d->mean; r.invstd = d->invstd;
  r.rows = d->rows; r.c = d->c; r.partials = d->partials;
  r.splits = splits; r.rows_per_clip = d->rows_per_clip; r.blocks_per_clip = bpc;
  bn_bwd_reduce_kernel<<<nblocks, 256, 256 * 16 * sizeof(float), stream>>>(r);
  if (int rc = launch_status("sfb_bn_bwd(reduce)")) return rc;
  bn_bwd_finalize_kernel<<<d->c, 64, 0, stream>>>(d->partials, nblocks, d->c, double(d->rows / splits), d->gamma,
                                                                 d->invstd, d->dgamma, d->dbeta, d->accumulate_param_grads,
                                                                 d->training, d->coef,
                                                                 d->c_valid > 0 ? d->c_valid : d->c, splits, bpc);
  if (int rc = launch_status("sfb_bn_bwd(finalize)")) return rc;
  BnBwdApplyParams a;
  a.dout = d->dout; a.dout_pitch = d->dout_pitch;
  a.mask = (const bf16*)d->mask_hi; a.mask_pitch = d->mask_pitch;
  a.mask_scale = d->mask_scale; a.mask_shift = d->mask_shift;
  a.y = d->y; a.y_pitch = d->y_pitch; a.mean = d->mean; a.invstd = d->invstd; a.coef = d->coef;
  a.dy_hi = (bf16*)d->dy_hi; a.dy_lo = (bf16*)d->dy_lo; a.dy_pitch = d->dy_pitch;
  a.dres = d->dres; a.dres_pitch = d->dres_pitch; a.dres_accumulate = d->dres_accumulate;
  a.rows = d->rows; a.c = d->c;
  a.splits = splits; a.rows_per_clip = d->rows_per_clip;
  const int64_t items = d->rows * (d->c / 8);
  bn_bwd_apply_kernel<<<rowlane_grid(d->rows, d->c / 8, 256), 256, 0, stream>>>(a);
  return launch_status("sfb_bn_bwd(apply)");
}

extern "C" int sfb_bn_relu_maxpool_fwd(const sfb_pool_desc* d, void* stream) {
  if (d->c % 8 || d->kh * d->kw > 254) {
    set_error("sfb_bn_relu_maxpool_fwd: c=%d must be a multiple of 8 and the window < 255 taps", d->c);
    return -10;
  }
  PoolParams p;
  memset(&p, 0, sizeof(p));
  p.y = d->y; p.scale = d->scale; p.shift = d->shift;
  p.n = d->n; p.t = d->t; p.h = d->h; p.w = d->w; p.c = d->c; p.oh = d->oh; p.ow = d->ow;
  p.kh = d->kh; p.kw = d->kw; p.sh = d->sh; p.sw = d->sw; p.ph = d->ph; p.pw = d->pw;
  p.o_hi = (bf16*)d->out_hi; p.o_lo = (bf16*)d->out_lo; p.o_pitch = d->out_pitch; p.argmax = d->argmax;
  p.splits = d->splits > 1 ? d->splits : 1;
  if (d->n % p.splits) {
    set_error("sfb_bn_relu_maxpool_fwd: batch %d is not a multiple of %d splits", d->n, p.splits);
    return -10;
  }
  const int64_t items = int64_t(d->n) * d->t * d->oh * d->ow * (d->c / 8);
  bn_relu_maxpool_fwd_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bn_relu_maxpool_fwd");
}

extern "C" int sfb_bn_relu_maxpool_bwd(const sfb_pool_desc* d, void* stream) {
  if (d->c % 8) {
    set_error("sfb_bn_relu_maxpool_bwd: c=%d must be a multiple of 8", d->c);
    return -10;
  }
  PoolParams p;
  memset(&p, 0, sizeof(p));
  p.n = d->n; p.t = d->t; p.h = d->h; p.w = d->w; p.c = d->c; p.oh = d->oh; p.ow = d->ow;
  p.kh = d->kh; p.kw = d->kw; p.sh = d->sh; p.sw = d->sw; p.ph = d->ph; p.pw = d->pw;
  p.argmax = d->argmax; p.dout = d->dout; p.dout_pitch = d->dout_pitch; p.dz = d->dz;
  const int64_t items = int64_t(d->n) * d->t * d->h * d->w * (d->c / 8);
  bn_relu_maxpool_bwd_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bn_relu_maxpool_bwd");
}

// ------------------------------------------------------------------------------------------- MaxPool3d on planes
// Generic MaxPool3d over a split-bf16 activation (pathway{p}_pool of the C2D / I3D archs, video_model_builder.py
// :543-549; MViT's pool_skip, attention.py:486): values are compared as hi+lo, first maximum wins (torch scan order),
// the window index is saved (uint8) and the backward is a gather over the windows that cover an input position.
namespace sfb {
struct Pool3dParams {
  const __nv_bfloat16* i_hi; const __nv_bfloat16* i_lo; int64_t i_pitch;
  __nv_bfloat16* o_hi; __nv_bfloat16* o_lo; int64_t o_pitch;
  uint8_t* argmax;
  int n, t, h, w, c, ot, oh, ow;
  int kt, kh, kw, st, sh, sw, pt, ph, pw;
  const float* dout; int64_t dout_pitch; float* din; int64_t din_pitch; int din_accumulate;
};
__global__ void maxpool3d_fwd_kernel(const Pool3dParams p) {
  const int cg = p.c / 8;
  const int64_t items = int64_t(p.n) * p.ot * p.oh * p.ow * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int g = int(i % cg);
    int64_t pos = i / cg;
    const int ox = int(pos % p.ow);
    int64_t r = pos / p.ow;
    const int oy = int(r % p.oh);
    r /= p.oh;
    const int oz = int(r % p.ot);
    const int64_t b = r / p.ot;
    const int c = g * 8;
    float best[8];
    uint8_t arg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = 0; }
    for (int kz = 0; kz < p.kt; ++kz) {
      const int iz = oz * p.st - p.pt + kz;
      if (iz < 0 || iz >= p.t) continue;
      for (int ky = 0; ky < p.kh; ++ky) {
        const int iy = oy * p.sh - p.ph + ky;
        if (iy < 0 || iy >= p.h) continue;
        for (int kx = 0; kx < p.kw; ++kx) {
          const int ix = ox * p.sw - p.pw + kx;
          if (ix < 0 || ix >= p.w) continue;
          const int64_t ipos = ((b * p.t + iz) * p.h + iy) * p.w + ix;
          float v[8];
          load_planes8(p.i_hi + ipos * p.i_pitch + c, p.i_lo ? p.i_lo + ipos * p.i_pitch + c : nullptr, v);
          const uint8_t idx = uint8_t((kz * p.kh + ky) * p.kw + kx);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (v[j] > best[j]) { best[j] = v[j]; arg[j] = idx; }
        }
      }
    }
    store_split8(p.o_hi + pos * p.o_pitch + c, p.o_lo ? p.o_lo + pos * p.o_pitch + c : nullptr, best);
    *reinterpret_cast<uint2*>(p.argmax + pos * p.c + c) =
        make_uint2(arg[0] | (arg[1] << 8) | (arg[2] << 16) | (uint32_t(arg[3]) << 24),
                   arg[4] | (arg[5] << 8) | (arg[6] << 16) | (uint32_t(arg[7]) << 24));
  }
}
__global__ void maxpool3d_bwd_kernel(const Pool3dParams p) {
  const int cg = p.c / 8;
  const int64_t items = int64_t(p.n) * p.t * p.h * p.w * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int g = int(i % cg);
    int64_t pos = i / cg;
    const int ix = int(pos % p.w);
    int64_t r = pos / p.w;
    const int iy = int(r % p.h);
    r /= p.h;
    const int iz = int(r % p.t);
    const int64_t b = r / p.t;
    const int c = g * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const int oz_lo = max(0, (iz + p.pt - p.kt + p.st) / p.st), oz_hi = min(p.ot - 1, (iz + p.pt) / p.st);
    const int oy_lo = max(0, (iy + p.ph - p.kh + p.sh) / p.sh), oy_hi = min(p.oh - 1, (iy + p.ph) / p.sh);
    const int ox_lo = max(0, (ix + p.pw - p.kw + p.sw) / p.sw), ox_hi = min(p.ow - 1, (ix + p.pw) / p.sw);
    for (int oz = oz_lo; oz <= oz_hi; ++oz) {
      const int kz = iz - (oz * p.st - p.pt);
      if (kz < 0 || kz >= p.kt) continue;
      for (int oy = oy_lo; oy <= oy_hi; ++oy) {
        const int ky = iy - (oy * p.sh - p.ph);
        if (ky < 0 || ky >= p.kh) continue;
        for (int ox = ox_lo; ox <= ox_hi; ++ox) {
          const int kx = ix - (ox * p.sw - p.pw);
          if (kx < 0 || kx >= p.kw) continue;
          const int64_t opos = ((b * p.ot + oz) * p.oh + oy) * p.ow + ox;
          const uint2 am = *reinterpret_cast<const uint2*>(p.argmax + opos * p.c + c);
          float d[8];
          load8(p.dout + opos * p.dout_pitch + c, d);
          const uint32_t want = uint32_t((kz * p.kh + ky) * p.kw + kx);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const uint32_t a = ((j < 4 ? am.x : am.y) >> (8 * (j & 3))) & 0xffu;
            if (a == want) acc[j] += d[j];
          }
        }
      }
    }
    float* dst = p.din + pos * p.din_pitch + c;
    if (p.din_accumulate) {
      float o[8];
      load8(dst, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += o[j];
    }
    store8(dst, acc);
  }
}
}  // namespace sfb

extern "C" int sfb_maxpool3d_fwd(const sfb_pool3d_desc* d, void* stream) {
  if (d->c % 8 || d->kt * d->kh * d->kw > 255) {
    set_error("sfb_maxpool3d_fwd: c=%d must be a multiple of 8 and the window <= 255 taps", d->c);
    return -10;
  }
  sfb::Pool3dParams p;
  memset(&p, 0, sizeof(p));
  p.i_hi = (const bf16*)d->in_hi; p.i_lo = (const bf16*)d->in_lo; p.i_pitch = d->in_pitch;
  p.o_hi = (bf16*)d->out_hi; p.o_lo = (bf16*)d->out_lo; p.o_pitch = d->out_pitch; p.argmax = d->argmax;
  p.n = d->n; p.t = d->t; p.h = d->h; p.w = d->w; p.c = d->c; p.ot = d->ot; p.oh = d->oh; p.ow = d->ow;
  p.kt = d->kt; p.kh = d->kh; p.kw = d->kw; p.st = d->st; p.sh = d->sh; p.sw = d->sw; p.pt = d->pt; p.ph = d->ph; p.pw = d->pw;
  const int64_t items = int64_t(d->n) * d->ot * d->oh * d->ow * (d->c / 8);
  sfb::maxpool3d_fwd_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_maxpool3d_fwd");
}
extern "C" int sfb_maxpool3d_bwd(const sfb_pool3d_desc* d, void* stream) {
  if (d->c % 8) {
    set_error("sfb_maxpool3d_bwd: c=%d must be a multiple of 8", d->c);
    return -10;
  }
  sfb::Pool3dParams p;
  memset(&p, 0, sizeof(p));
  p.argmax = d->argmax;
  p.n = d->n; p.t = d->t; p.h = d->h; p.w = d->w; p.c = d->c; p.ot = d->ot; p.oh = d->oh; p.ow = d->ow;
  p.kt = d->kt; p.kh = d->kh; p.kw = d->kw; p.st = d->st; p.sh = d->sh; p.sw = d->sw; p.pt = d->pt; p.ph = d->ph; p.pw = d->pw;
  p.dout = d->dout; p.dout_pitch = d->dout_pitch; p.din = d->din; p.din_pitch = d->din_pitch;
  p.din_accumulate = d->din_accumulate;
  const int64_t items = int64_t(d->n) * d->t * d->h * d->w * (d->c / 8);
  sfb::maxpool3d_bwd_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_maxpool3d_bwd");
}

// dst[rows, c] += src[rows, c] (fp32 views with row pitches): the second and later contributions to an activation
// gradient are produced by a plain-store GEMM epilogue into scratch and merged here with fully coalesced traffic
// (a read-modify-write epilogue touches 32 different 128-byte lines per instruction).
namespace sfb {
__global__ void add_f32_2d_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t rows, int cg,
                                  int64_t dst_pitch, int64_t src_pitch) {
  const int64_t items = rows * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cg;
    const int c = int(i - r * cg) * 8;
    float a[8], b[8];
    load8(dst + r * dst_pitch + c, a);
    load8(src + r * src_pitch + c, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    store8(dst + r * dst_pitch + c, a);
  }
}
}  // namespace sfb
extern "C" int sfb_add_f32_2d(float* dst, const float* src, int64_t rows, int32_t c, int64_t dst_pitch,
                              int64_t src_pitch, void* stream) {
  if (c % 8 || dst_pitch % 4 || src_pitch % 4) {
    set_error("sfb_add_f32_2d: c=%d must be a multiple of 8 and pitches 16-byte aligned", c);
    return -10;
  }
  const int64_t items = rows * (c / 8);
  if (items == 0) return 0;
  sfb::add_f32_2d_kernel<<<ew_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dst, src, rows, c / 8, dst_pitch,
                                                                               src_pitch);
  return launch_status("sfb_add_f32_2d");
}
