// MAE pre-training kernels (slowfast/models/masked.py: _mae_random_masking :283, _mae_forward_encoder :319,
// _mae_forward_decoder :394, _get_pixel_label_3d :212):
//   * per-clip random masking from the noise: stable argsort ranks -> ids_keep / ids_restore / mask and the list of
//     removed tokens in ascending position
//   * encoder token assembly from the kept patches only (cls + separable positions gathered by ids_keep) and its
//     backward scatter onto the dense token grid
//   * the decoder's un-shuffle: decoder_embed rows or the mask token at every position, + the joint position table; its
//     backward with fixed-order sums for the table and the mask token
//   * row gather / scatter of the removed tokens for the prediction head, and the normalised-pixel targets
// Every reduction here is a fixed-order sum (no float atomics): the MAE step is bitwise reproducible.
#include <cstdint>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "runtime.h"

namespace sfb {

constexpr int kMaeMaxTokens = 4096;  // noise row of one clip held in shared memory
constexpr int kMaskThreads = 1024;
constexpr int kMaskPer = kMaeMaxTokens / kMaskThreads;

static int mae_grid(int64_t items, int block) { return capped_grid(items, block, int64_t(kGridSms) * 8); }

// ------------------------------------------------------------------------------------------- masking
// One CTA per clip.  rank[i] = #{j : noise[j] < noise[i] or (noise[j] == noise[i] and j < i)} is the position of token i
// in torch.argsort(noise, stable=True), so ids_restore = rank, ids_keep[rank] = i for rank < keep, mask = rank >= keep.
// Thread k owns the contiguous positions [k*per, k*per + per): an exclusive scan of the per-thread removed counts
// numbers the removed tokens in ascending position, and masked_rows lists them as rows of the [b, l+1] decoder sequence.
__global__ void __launch_bounds__(kMaskThreads, 1) mae_masking_kernel(const float* __restrict__ noise, int l, int keep,
                                                                   int* __restrict__ ids_keep,
                                                                   int* __restrict__ ids_restore,
                                                                   float* __restrict__ mask,
                                                                   int* __restrict__ masked_rows) {
  __shared__ float sn[kMaeMaxTokens];
  __shared__ int wsum[kMaskThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float* nz = noise + int64_t(b) * l;
  for (int i = tid; i < l; i += blockDim.x) sn[i] = nz[i];
  __syncthreads();
  const int per = (l + blockDim.x - 1) / blockDim.x;
  const int i0 = min(l, tid * per), i1 = min(l, i0 + per);
  int rank[kMaskPer];
  float v[kMaskPer];
#pragma unroll
  for (int k = 0; k < kMaskPer; ++k) {
    rank[k] = 0;
    v[k] = i0 + k < i1 ? sn[i0 + k] : 0.f;
  }
  for (int j = 0; j < l; ++j) {
    const float u = sn[j];
#pragma unroll
    for (int k = 0; k < kMaskPer; ++k) rank[k] += (u < v[k]) || (u == v[k] && j < i0 + k);
  }
  int removed = 0;
#pragma unroll
  for (int k = 0; k < kMaskPer; ++k) removed += (i0 + k < i1 && rank[k] >= keep);
  // block exclusive scan of `removed` in thread order
  int incl = removed;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) wsum[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const int nw = blockDim.x >> 5;
    int w = lane < nw ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < nw) wsum[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  int pos = incl - removed + (wid > 0 ? wsum[wid - 1] : 0);
  const int nrem = l - keep;
#pragma unroll
  for (int k = 0; k < kMaskPer; ++k) {
    const int i = i0 + k;
    if (i < i1) {
      const int r = rank[k];
      ids_restore[int64_t(b) * l + i] = r;
      mask[int64_t(b) * l + i] = r >= keep ? 1.f : 0.f;
      if (r < keep) {
        ids_keep[int64_t(b) * keep + r] = i;
      } else {
        masked_rows[int64_t(b) * nrem + pos] = b * (l + 1) + 1 + i;
        ++pos;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------- encoder tokens
// x[b,0] = cls + pc;  x[b,1+j] = (y[b,j] + bias) + (ps[m % hw] + pt[m / hw]),  m = ids_keep[b,j]   (masked.py:340-371)
__global__ void tokens_assemble_keep_kernel(const float* __restrict__ y, const float* __restrict__ bias,
                                            const float* __restrict__ cls, const float* __restrict__ ps,
                                            const float* __restrict__ pt, const float* __restrict__ pc,
                                            const int* __restrict__ keep_idx, int b, int nkeep, int hw, int c,
                                            float* __restrict__ x) {
  const int64_t items = int64_t(b) * (nkeep + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (nkeep + 1));
    const int64_t bb = t / (nkeep + 1);
    if (n == 0) {
      x[i] = cls[ch] + pc[ch];
    } else {
      const int j = n - 1;
      const int m = keep_idx[bb * nkeep + j];
      x[i] = (y[(bb * nkeep + j) * c + ch] + bias[ch]) + (ps[int64_t(m % hw) * c + ch] + pt[int64_t(m / hw) * c + ch]);
    }
  }
}
// dense[b,0] = dx[b,0];  dense[b,1+l] = r < nkeep ? dx[b,1+r] : 0,  r = ids_restore[b,l]
__global__ void tokens_scatter_keep_kernel(const float* __restrict__ dx, const int* __restrict__ ids_restore, int b,
                                           int nkeep, int l, int c, float* __restrict__ dense) {
  const int64_t items = int64_t(b) * (l + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (l + 1));
    const int64_t bb = t / (l + 1);
    float v = 0.f;
    if (n == 0) {
      v = dx[bb * (nkeep + 1) * c + ch];
    } else {
      const int r = ids_restore[bb * l + n - 1];
      if (r < nkeep) v = dx[(bb * (nkeep + 1) + 1 + r) * c + ch];
    }
    dense[i] = v;
  }
}

// ------------------------------------------------------------------------------------------- decoder tokens
// out[b,0] = (z[b,0] + bias) + pos[0];  out[b,1+l] = (r < nkeep ? z[b,1+r] + bias : mask_token) + pos[1+l]
// (masked.py:396-436: decoder_embed, mask tokens appended, un-shuffled by ids_restore, + decoder_pos_embed)
__global__ void decoder_assemble_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                                        const float* __restrict__ mask_token, const float* __restrict__ pos,
                                        const int* __restrict__ ids_restore, int b, int nkeep, int l, int c,
                                        float* __restrict__ out) {
  const int64_t items = int64_t(b) * (l + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (l + 1));
    const int64_t bb = t / (l + 1);
    const int r = n == 0 ? -1 : ids_restore[bb * l + n - 1];
    float v;
    if (r < nkeep)
      v = z[(bb * (nkeep + 1) + 1 + r) * c + ch] + bias[ch];  // r = -1: the cls row
    else
      v = mask_token[ch];
    out[i] = v + pos[int64_t(n) * c + ch];
  }
}
// dz[b,0] = dx[b,0];  dz[b,1+j] = dx[b,1+ids_keep[b,j]]
__global__ void decoder_gather_grad_kernel(const float* __restrict__ dx, const int* __restrict__ ids_keep, int b,
                                           int nkeep, int l, int c, float* __restrict__ dz) {
  const int64_t items = int64_t(b) * (nkeep + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (nkeep + 1));
    const int64_t bb = t / (nkeep + 1);
    const int src = n == 0 ? 0 : 1 + ids_keep[bb * nkeep + n - 1];
    dz[i] = dx[(bb * (l + 1) + src) * c + ch];
  }
}
// dpos[n] = sum_b dx[b,n]  (batch order)
__global__ void batch_sum_kernel(const float* __restrict__ dx, int b, int64_t n_items, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n_items; i += int64_t(gridDim.x) * blockDim.x) {
    float s = 0.f;
    for (int bb = 0; bb < b; ++bb) s += dx[bb * n_items + i];
    out[i] = s;
  }
}
// partials[slab][ch] = sum over the slab's rows r of src[rows[r] * c + ch] (row order); grid = slabs
__global__ void indexed_rowsum_partial_kernel(const float* __restrict__ src, const int* __restrict__ rows, int nrows,
                                              int c, float* __restrict__ partials) {
  const int slab = blockIdx.x, nslab = gridDim.x;
  const int rps = (nrows + nslab - 1) / nslab;
  const int r0 = slab * rps, r1 = min(nrows, r0 + rps);
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    float s = 0.f;
    for (int r = r0; r < r1; ++r) s += src[int64_t(rows[r]) * c + ch];
    partials[int64_t(slab) * c + ch] = s;
  }
}
// out[ch] = sum_slab partials[slab][ch]  (fp64, slab order)
__global__ void slab_merge_kernel(const float* __restrict__ partials, int nslab, int c, float* __restrict__ out) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double s = 0.0;
  for (int k = 0; k < nslab; ++k) s += double(partials[int64_t(k) * c + ch]);
  out[ch] = float(s);
}

// ------------------------------------------------------------------------------------------- head rows
// dst[r] = src[idx ? idx[r] : r] (+ bias)
__global__ void rows_gather_kernel(const float* __restrict__ src, int64_t src_pitch, const int* __restrict__ idx,
                                   int64_t rows, int c, const float* __restrict__ bias, float* __restrict__ dst) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t r = i / c;
    const int64_t s = idx ? int64_t(idx[r]) : r;
    const float v = src[s * src_pitch + ch];
    dst[i] = bias ? v + bias[ch] : v;
  }
}
// dst[idx[r]] = src[r]
__global__ void rows_scatter_kernel(const float* __restrict__ src, const int* __restrict__ idx, int64_t rows, int c,
                                    float* __restrict__ dst) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t r = i / c;
    dst[int64_t(idx[r]) * c + ch] = src[i];
  }
}

// ------------------------------------------------------------------------------------------- pixel targets
// One warp per selected row (decoder row index b*(l+1) + 1 + tok, tok = (tt, hh, ww) on the (t/t_stride, h/p, w/p)
// grid).  Column k = ((uu*p + py)*p + px)*ch + cc reads frame tt*t_stride + uu (u = 1 with TIME_STRIDE_LOSS, else
// t_stride): _patchify's "nctuhpwq->nthwupqc" order.  norm: (v - mean) / sqrt(var + 1e-6), var unbiased, two passes.
__global__ void __launch_bounds__(256) pixel_targets_kernel(const float* __restrict__ x, int b, int ch, int t, int h,
                                                            int w, int t_stride, int u, int p,
                                                            const int* __restrict__ rows, int nrows, int norm,
                                                            float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const int gh = h / p, gw = w / p, gt = t / t_stride;
  const int l = gt * gh * gw;
  const int D = u * p * p * ch;
  for (int64_t r = warp; r < nrows; r += nwarps) {
    const int row = rows[r];
    const int bb = row / (l + 1);
    const int tok = row % (l + 1) - 1;
    const int ww = tok % gw, hh = (tok / gw) % gh, tt = tok / (gw * gh);
    const float* base = x + ((int64_t(bb) * ch * t + int64_t(tt) * t_stride) * h + int64_t(hh) * p) * w + int64_t(ww) * p;
    auto at = [&](int k) {
      const int cc = k % ch;
      int q = k / ch;
      const int px = q % p;
      q /= p;
      const int py = q % p;
      const int uu = q / p;
      return base[((int64_t(cc) * t + uu) * h + py) * w + px];
    };
    float* o = out + r * int64_t(D);
    if (!norm) {
      for (int k = lane; k < D; k += 32) o[k] = at(k);
      continue;
    }
    float s = 0.f;
    for (int k = lane; k < D; k += 32) s += at(k);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    const float mean = s / float(D);
    float ss = 0.f;
    for (int k = lane; k < D; k += 32) {
      const float d = at(k) - mean;
      ss += d * d;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
    const float inv = 1.f / sqrtf(ss / float(D - 1) + 1e-6f);
    for (int k = lane; k < D; k += 32) o[k] = (at(k) - mean) * inv;
  }
}

}  // namespace sfb

using namespace sfb;

extern "C" int32_t sfb_mae_max_tokens(void) { return kMaeMaxTokens; }

extern "C" int sfb_mae_random_masking(const float* noise, int32_t b, int32_t l, int32_t keep, int32_t* ids_keep,
                                      int32_t* ids_restore, float* mask, int32_t* masked_rows, void* stream) {
  if (b < 1 || l < 2 || l > kMaeMaxTokens || keep < 1 || keep >= l || int64_t(b) * (l + 1) > INT32_MAX) {
    set_error("sfb_mae_random_masking: b=%d l=%d keep=%d (needs 1 <= keep < l <= %d)", b, l, keep, kMaeMaxTokens);
    return -10;
  }
  mae_masking_kernel<<<b, kMaskThreads, 0, (cudaStream_t)stream>>>(noise, l, keep, ids_keep, ids_restore, mask,
                                                                    masked_rows);
  return launch_status("sfb_mae_random_masking");
}

extern "C" int sfb_tokens_assemble_keep(const float* y, const float* bias, const float* cls, const float* pos_spatial,
                                        const float* pos_temporal, const float* pos_class, const int32_t* ids_keep,
                                        int32_t b, int32_t nkeep, int32_t l, int32_t hw, int32_t c, float* x,
                                        void* stream) {
  if (!pos_spatial || !pos_temporal || !pos_class || !ids_keep || hw < 1 || l % hw != 0 || nkeep < 1 || nkeep > l) {
    set_error("sfb_tokens_assemble_keep: needs the three position tables, ids_keep, hw=%d dividing l=%d, nkeep=%d",
              hw, l, nkeep);
    return -10;
  }
  const int64_t items = int64_t(b) * (nkeep + 1) * c;
  tokens_assemble_keep_kernel<<<mae_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(
      y, bias, cls, pos_spatial, pos_temporal, pos_class, ids_keep, b, nkeep, hw, c, x);
  return launch_status("sfb_tokens_assemble_keep");
}

extern "C" int sfb_tokens_scatter_keep(const float* dx, const int32_t* ids_restore, int32_t b, int32_t nkeep, int32_t l,
                                       int32_t c, float* dense, void* stream) {
  const int64_t items = int64_t(b) * (l + 1) * c;
  tokens_scatter_keep_kernel<<<mae_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dx, ids_restore, b, nkeep, l, c,
                                                                                      dense);
  return launch_status("sfb_tokens_scatter_keep");
}

extern "C" int sfb_decoder_assemble(const float* z, const float* bias, const float* mask_token, const float* pos,
                                    const int32_t* ids_restore, int32_t b, int32_t nkeep, int32_t l, int32_t c, float* out,
                                    void* stream) {
  const int64_t items = int64_t(b) * (l + 1) * c;
  decoder_assemble_kernel<<<mae_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(z, bias, mask_token, pos, ids_restore,
                                                                                   b, nkeep, l, c, out);
  return launch_status("sfb_decoder_assemble");
}

extern "C" int sfb_decoder_assemble_bwd(const float* dx, const int32_t* ids_keep, const int32_t* masked_rows, int32_t b,
                                        int32_t nkeep, int32_t l, int32_t c, float* dz, float* dpos, float* dmask_token,
                                        float* partials, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (b < 1 || nkeep < 1 || nkeep >= l || c < 1) {
    set_error("sfb_decoder_assemble_bwd: b=%d nkeep=%d l=%d c=%d", b, nkeep, l, c);
    return -10;
  }
  const int64_t items = int64_t(b) * (nkeep + 1) * c;
  decoder_gather_grad_kernel<<<mae_grid(items, 256), 256, 0, stream>>>(dx, ids_keep, b, nkeep, l, c, dz);
  if (int rc = launch_status("sfb_decoder_assemble_bwd(gather)")) return rc;
  const int64_t pitems = int64_t(l + 1) * c;
  batch_sum_kernel<<<mae_grid(pitems, 256), 256, 0, stream>>>(dx, b, pitems, dpos);
  if (int rc = launch_status("sfb_decoder_assemble_bwd(pos)")) return rc;
  const int nrows = b * (l - nkeep);
  const int nslab = sfb_segment_slabs(1, nrows);
  indexed_rowsum_partial_kernel<<<nslab, c < 256 ? (c + 31) / 32 * 32 : 256, 0, stream>>>(dx, masked_rows, nrows, c,
                                                                                          partials);
  if (int rc = launch_status("sfb_decoder_assemble_bwd(mask token)")) return rc;
  slab_merge_kernel<<<(c + 127) / 128, 128, 0, stream>>>(partials, nslab, c, dmask_token);
  return launch_status("sfb_decoder_assemble_bwd(mask token merge)");
}

extern "C" int sfb_rows_gather(const float* src, int64_t src_pitch, const int32_t* idx, int64_t rows, int32_t c,
                               const float* bias, float* dst, void* stream) {
  rows_gather_kernel<<<mae_grid(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(src, src_pitch, idx, rows, c, bias, dst);
  return launch_status("sfb_rows_gather");
}

extern "C" int sfb_rows_scatter(const float* src, const int32_t* idx, int64_t rows, int32_t c, float* dst, void* stream) {
  rows_scatter_kernel<<<mae_grid(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(src, idx, rows, c, dst);
  return launch_status("sfb_rows_scatter");
}

extern "C" int sfb_pixel_targets(const float* x, int32_t b, int32_t ch, int32_t t, int32_t h, int32_t w,
                                 int32_t t_stride, int32_t u, int32_t p, const int32_t* rows, int32_t nrows, int32_t norm,
                                 float* out, void* stream) {
  if (p < 1 || t_stride < 1 || (u != 1 && u != t_stride) || t % t_stride || h % p || w % p || u * p * p * ch < 2) {
    set_error("sfb_pixel_targets: %dx%dx%d clip, patch %d, time stride %d, u=%d", t, h, w, p, t_stride, u);
    return -10;
  }
  if (nrows < 1) return 0;
  pixel_targets_kernel<<<mae_grid(int64_t(nrows) * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      x, b, ch, t, h, w, t_stride, u, p, rows, nrows, norm, out);
  return launch_status("sfb_pixel_targets");
}
