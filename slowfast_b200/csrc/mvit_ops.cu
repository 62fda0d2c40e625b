// Token-path kernels of the MViT blocks (attention.py: attention_pool :13, cal_rel_pos_* :64/:111,
// MultiScaleAttention.forward :293, MultiScaleBlock.forward :491; common.py Mlp :26) that are not GEMMs:
// LayerNorm, depthwise 3-D pooling convolutions on the token grid, the rel-pos-biased softmax, head split/merge with
// residual pooling, GELU, residual/bias combines, max-pool skip and the bias-gradient column sums.
// Tokens are [B, N = 1 + T*H*W, C] with the cls token first (kCls = 1), or [B, T*H*W, C] without one (kCls = 0: the
// image recipes with CLS_EMBED_ON False); the residual stream is fp32, GEMM operands are split-bf16 planes.  All kernels are HBM-bound elementwise / row kernels.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "planes.cuh"
#include "runtime.h"

namespace sfb {

static constexpr size_t kSoftmaxSmemMax = 160 * 1024;  // 8 warps x (keys + rel-pos bins) fp32 rows
static int mv_grid(int64_t items, int block, int waves = 8) {
  return capped_grid(items, block, int64_t(kGridSms) * waves);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------- LayerNorm
// One warp per row (C <= 1024).  y = (x - mean) * rstd * gamma + beta -> split planes and/or fp32.
constexpr int LN_MAX_PER_LANE = 40;  // C <= 1280 (ViT-H)
// NPL = elements per lane (c <= 32*NPL): instantiated for 3 / 6 / 12 / 24 / 32 / 40 so that narrow rows (c = 96: the first
// MViT stages, the per-head pooling norms) do not pay for 24 predicated-off iterations per row
template <int NPL>
__global__ void __launch_bounds__(256) ln_fwd_kernel(const float* __restrict__ x, int64_t x_pitch, int64_t rows, int c,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                                     float eps, __nv_bfloat16* __restrict__ o_hi,
                                                     __nv_bfloat16* __restrict__ o_lo, float* __restrict__ o_f32,
                                                     int64_t o_pitch, float* __restrict__ mean,
                                                     float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float* xr = x + r * x_pitch;
    float v[NPL];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int j = lane + 32 * i;
      v[i] = j < c ? xr[j] : 0.f;
      s += v[i];
    }
    const float mu = warp_sum(s) / float(c);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const float d = (lane + 32 * i) < c ? v[i] - mu : 0.f;
      q = fmaf(d, d, q);
    }
    const float rs = rsqrtf(warp_sum(q) / float(c) + eps);
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int j = lane + 32 * i;
      if (j < c) {
        const float y = (v[i] - mu) * rs * gamma[j] + beta[j];
        if (o_hi) put_split(o_hi, o_lo, r * o_pitch + j, y);
        if (o_f32) o_f32[r * o_pitch + j] = y;
      }
    }
    if (lane == 0 && mean) {
      mean[r] = mu;
      rstd[r] = rs;
    }
  }
}
// dx (=|+=) rstd * (g - mean_c(g) - xhat * mean_c(g * xhat)),  g = dy * gamma;   per-block dgamma/dbeta partials
template <int NPL>
__global__ void __launch_bounds__(256) ln_bwd_kernel(const float* __restrict__ dy, int64_t dy_pitch,
                                                     const float* __restrict__ x, int64_t x_pitch, int64_t rows, int c,
                                                     const float* __restrict__ gamma, const float* __restrict__ mean,
                                                     const float* __restrict__ rstd, float* __restrict__ dx,
                                                     int64_t dx_pitch, int dx_accumulate,
                                                     float* __restrict__ partials /* [grid][2][c] */) {
  extern __shared__ float sm[];  // [8 warps][2][c]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  float dg[NPL], db[NPL], gm[NPL];
#pragma unroll
  for (int i = 0; i < NPL; ++i) {
    dg[i] = db[i] = 0.f;
    gm[i] = (lane + 32 * i) < c ? gamma[lane + 32 * i] : 0.f;
  }
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float mu = mean[r], rs = rstd[r];
    float g[NPL], xh[NPL];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int j = lane + 32 * i;
      const bool ok = j < c;
      const float d = ok ? dy[r * dy_pitch + j] : 0.f;
      xh[i] = ok ? (x[r * x_pitch + j] - mu) * rs : 0.f;
      g[i] = d * gm[i];
      s1 += g[i];
      s2 = fmaf(g[i], xh[i], s2);
      dg[i] = fmaf(d, xh[i], dg[i]);
      db[i] += d;
    }
    s1 = warp_sum(s1) / float(c);
    s2 = warp_sum(s2) / float(c);
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int j = lane + 32 * i;
      if (j < c) {
        const float v = rs * (g[i] - s1 - xh[i] * s2);
        float* o = dx + r * dx_pitch + j;
        *o = dx_accumulate ? *o + v : v;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NPL; ++i) {
    const int j = lane + 32 * i;
    if (j < c) {
      sm[(wid * 2 + 0) * c + j] = dg[i];
      sm[(wid * 2 + 1) * c + j] = db[i];
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * c; j += blockDim.x) {
    const int which = j / c, ch = j - which * c;
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += sm[(w * 2 + which) * c + ch];
    partials[(size_t(blockIdx.x) * 2 + which) * c + ch] = s;
  }
}
// Rows wider than 768 (ViT-L 1024, MViTv2-L's last stage 1152, ViT-H 1280): the same arithmetic, but a row's dy / x are
// read twice from global memory (L1 / L2) instead of being held in registers, and the per-block dgamma / dbeta merge runs
// in 256-channel chunks, so the kernel keeps its registers (no spills) and 16 KB of static shared memory.
template <int NPL>
__global__ void __launch_bounds__(256) ln_bwd_wide_kernel(const float* __restrict__ dy, int64_t dy_pitch,
                                                          const float* __restrict__ x, int64_t x_pitch, int64_t rows,
                                                          int c, const float* __restrict__ gamma,
                                                          const float* __restrict__ mean, const float* __restrict__ rstd,
                                                          float* __restrict__ dx, int64_t dx_pitch, int dx_accumulate,
                                                          float* __restrict__ partials /* [grid][2][c] */) {
  static_assert(NPL % 8 == 0, "chunked merge: 8 lane slots = 256 channels per chunk");
  __shared__ float sm[8][2][256];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  float dg[NPL], db[NPL];
#pragma unroll
  for (int i = 0; i < NPL; ++i) dg[i] = db[i] = 0.f;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float mu = mean[r], rs = rstd[r];
    const float* dyr = dy + r * dy_pitch;
    const float* xr = x + r * x_pitch;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int j = lane + 32 * i;
      const bool ok = j < c;
      const float d = ok ? dyr[j] : 0.f;
      const float xh = ok ? (xr[j] - mu) * rs : 0.f;
      const float g = d * (ok ? gamma[j] : 0.f);
      s1 += g;
      s2 = fmaf(g, xh, s2);
      dg[i] = fmaf(d, xh, dg[i]);
      db[i] += d;
    }
    s1 = warp_sum(s1) / float(c);
    s2 = warp_sum(s2) / float(c);
#pragma unroll
    for (int i = 0; i < NPL; ++i) {
      const int j = lane + 32 * i;
      if (j < c) {
        const float xh = (xr[j] - mu) * rs;
        const float v = rs * (dyr[j] * gamma[j] - s1 - xh * s2);
        float* o = dx + r * dx_pitch + j;
        *o = dx_accumulate ? *o + v : v;
      }
    }
  }
#pragma unroll
  for (int i0 = 0; i0 < NPL; i0 += 8) {
    const int c0 = 32 * i0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      sm[wid][0][lane + 32 * i] = dg[i0 + i];
      sm[wid][1][lane + 32 * i] = db[i0 + i];
    }
    __syncthreads();
    for (int j = threadIdx.x; j < 2 * 256; j += blockDim.x) {
      const int which = j >> 8, ch = j & 255;
      if (c0 + ch < c) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += sm[w][which][ch];
        partials[(size_t(blockIdx.x) * 2 + which) * c + c0 + ch] = s;
      }
    }
    __syncthreads();
  }
}
// ------------------------------------------------------------------------------------------- column sums (bias grads)
// partials[block][c] = sum over the block's row slab of src[rows, c]
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ src, int64_t pitch, int64_t rows, int c,
                                                     float* __restrict__ partials) {
  const int64_t rpb = (rows + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = blockIdx.x * rpb, r1 = min(rows, r0 + rpb);
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;  // four independent chains: the loads of 4 rows are in flight together
    int64_t r = r0;
    for (; r + 3 < r1; r += 4) {
      s0 += src[r * pitch + ch];
      s1 += src[(r + 1) * pitch + ch];
      s2 += src[(r + 2) * pitch + ch];
      s3 += src[(r + 3) * pitch + ch];
    }
    for (; r < r1; ++r) s0 += src[r * pitch + ch];
    partials[size_t(blockIdx.x) * c + ch] = (s0 + s1) + (s2 + s3);
  }
}
// c % 4 == 0 and 16-byte aligned rows: thread = (4-column group, row lane); every thread streams float4s, so narrow
// matrices (c = 96: 24 groups x 10 row lanes) keep the whole block busy instead of 96 of 256 threads
__global__ void __launch_bounds__(256) colsum4_kernel(const float* __restrict__ src, int64_t pitch, int64_t rows, int c,
                                                      float* __restrict__ partials) {
  __shared__ float4 red[256];
  const int cq = c >> 2;
  const int QL = cq < 256 ? cq : 256;
  const int RL = 256 / QL;
  const int ql = threadIdx.x % QL, rl = threadIdx.x / QL;
  const int64_t rpb = (rows + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = blockIdx.x * rpb, r1 = min(rows, r0 + rpb);
  for (int q0 = 0; q0 < cq; q0 += QL) {
    const int q = q0 + ql;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (rl < RL && q < cq) {
      int64_t r = r0 + rl;
      for (; r + RL < r1; r += 2 * RL) {
        const float4 u = *reinterpret_cast<const float4*>(src + r * pitch + q * 4);
        const float4 v = *reinterpret_cast<const float4*>(src + (r + RL) * pitch + q * 4);
        a.x += u.x; a.y += u.y; a.z += u.z; a.w += u.w;
        b.x += v.x; b.y += v.y; b.z += v.z; b.w += v.w;
      }
      if (r < r1) {
        const float4 u = *reinterpret_cast<const float4*>(src + r * pitch + q * 4);
        a.x += u.x; a.y += u.y; a.z += u.z; a.w += u.w;
      }
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    __syncthreads();
    red[threadIdx.x] = a;
    __syncthreads();
    if (rl == 0 && q < cq) {
      for (int j = 1; j < RL; ++j) {
        const float4 v = red[j * QL + ql];
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
      *reinterpret_cast<float4*>(partials + size_t(blockIdx.x) * c + q * 4) = a;
    }
  }
}

// ------------------------------------------------------------------------------------------- token assembly
// x[b, 0, :] = cls;  x[b, 1 + l, :] = y[b, l, :] + bias      (patch embedding output -> token sequence)
// with separable absolute positions (ps != null): x[b, 0, :] = cls + pc;  x[b, 1 + t*hw + s, :] = (y + bias) + (ps[s] + pt[t]),
// the reference's order (the position table is summed first, then added: video_model_builder.py:1189-1199)
__global__ void tokens_assemble_kernel(const float* __restrict__ y, const float* __restrict__ bias,
                                       const float* __restrict__ cls, const float* __restrict__ ps,
                                       const float* __restrict__ pt, const float* __restrict__ pc, int b, int l, int hw,
                                       int c, float* __restrict__ x) {
  const int64_t items = int64_t(b) * (l + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (l + 1));
    const int64_t bb = t / (l + 1);
    if (!ps) {
      x[i] = n == 0 ? cls[ch] : y[(bb * l + n - 1) * c + ch] + bias[ch];
    } else if (n == 0) {
      x[i] = cls[ch] + pc[ch];
    } else {
      const int m = n - 1;
      x[i] = (y[(bb * l + m) * c + ch] + bias[ch]) + (ps[int64_t(m % hw) * c + ch] + pt[int64_t(m / hw) * c + ch]);
    }
  }
}
// joint position table (SEP_POS_EMBED False) and / or no cls row (cls == null):
//   x[b, 0, :] = cls + pos[0];  x[b, 1 + l, :] = (y[b, l, :] + bias) + pos[1 + l]      (cls != null)
//   x[b, l, :] = (y[b, l, :] + bias) + pos[l]                                           (cls == null)
// the reference's order (cat, then +=: video_model_builder.py:1180-1201); pos == null adds no position
__global__ void tokens_assemble_joint_kernel(const float* __restrict__ y, const float* __restrict__ bias,
                                             const float* __restrict__ cls, const float* __restrict__ pos, int b, int l,
                                             int c, float* __restrict__ x) {
  const int nc = cls ? 1 : 0;
  const int64_t items = int64_t(b) * (l + nc) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (l + nc));
    const int64_t bb = t / (l + nc);
    const float v = n < nc ? cls[ch] : y[(bb * l + n - nc) * c + ch] + bias[ch];
    x[i] = pos ? v + pos[int64_t(n) * c + ch] : v;
  }
}
// dpos[n, :] = sum_b dx[b, n, :]: one thread per output element, batch in order (no atomics, replay-exact)
__global__ void pos_joint_bwd_kernel(const float* __restrict__ dx, int b, int n, int c, float* __restrict__ dpos) {
  const int64_t items = int64_t(n) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    float acc = 0.f;
    for (int bb = 0; bb < b; ++bb) acc += dx[int64_t(bb) * items + i];
    dpos[i] = acc;
  }
}
// ------------------------------------------------------------------------------------------- separable position grads
// Deterministic: every output element is a fixed-order sum (no atomics), so CUDA-graph replay reproduces eager bitwise.
// dps[s, :] = sum_b sum_t dx[b, 1 + t*hw + s, :] and dpc[:] = sum_b dx[b, 0, :]: one thread per output element
__global__ void pos_sep_bwd_spatial_kernel(const float* __restrict__ dx, int b, int t, int hw, int c,
                                           float* __restrict__ dps, float* __restrict__ dpc) {
  const int64_t n = 1 + int64_t(t) * hw;
  const int64_t items = int64_t(hw + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int s = int(i / c);
    float acc = 0.f;
    if (s == hw) {
      for (int bb = 0; bb < b; ++bb) acc += dx[bb * n * c + ch];
      dpc[ch] = acc;
    } else {
      for (int bb = 0; bb < b; ++bb) {
        const float* p = dx + (bb * n + 1 + s) * c + ch;
        for (int tt = 0; tt < t; ++tt) acc += p[int64_t(tt) * hw * c];
      }
      dps[int64_t(s) * c + ch] = acc;
    }
  }
}
// Segmented row sums (the temporal position gradient and the mean-token readout):
//   partials[g][slab][ch] = sum_{o < n_outer} sum_{r in slab} src[(o * outer_stride + g * group_stride + r) * c + ch]
// grid (slabs, groups); fixed order inside a block, so the result depends on the shape only
__global__ void segment_rowsum_partial_kernel(const float* __restrict__ src, int c, int n_outer, int64_t outer_stride,
                                              int64_t group_stride, int seg_rows, float* __restrict__ partials) {
  const int g = blockIdx.y, slab = blockIdx.x, nslab = gridDim.x;
  const int rps = (seg_rows + nslab - 1) / nslab;
  const int r0 = slab * rps, r1 = min(seg_rows, r0 + rps);
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    float s0 = 0.f, s1 = 0.f;  // two independent chains
    for (int o = 0; o < n_outer; ++o) {
      const float* p = src + (o * outer_stride + g * group_stride) * c + ch;
      int r = r0;
      for (; r + 1 < r1; r += 2) {
        s0 += p[int64_t(r) * c];
        s1 += p[int64_t(r + 1) * c];
      }
      if (r < r1) s0 += p[int64_t(r) * c];
    }
    partials[(int64_t(g) * nslab + slab) * c + ch] = s0 + s1;
  }
}
// out[g][ch] = scale * sum_slab partials[g][slab][ch]   (fp64, slab order)
__global__ void segment_rowsum_merge_kernel(const float* __restrict__ partials, int nslab, int groups, int c, float scale,
                                            float* __restrict__ out) {
  const int64_t items = int64_t(groups) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t g = i / c;
    double s = 0.0;
    for (int k = 0; k < nslab; ++k) s += double(partials[(g * nslab + k) * c + ch]);
    out[i] = float(s) * scale;
  }
}
// mean readout backward: dx[b, 0, :] = 0;  dx[b, 1 + l, :] = dmean[b, :] * scale  (kCls = 0: every row gets the share)
template <int kCls>
__global__ void token_mean_bwd_kernel(const float* __restrict__ dmean, int b, int n, int c, float scale,
                                      float* __restrict__ dx) {
  const int64_t items = int64_t(b) * n * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int r = int(t % n);
    dx[i] = (kCls && r == 0) ? 0.f : dmean[(t / n) * c + ch] * scale;
  }
}
// ------------------------------------------------------------------------------------------- non-overlapping patches
// stride == kernel, no padding: NCTHW clip -> split rows [b * L, cin*kt*kh*kw], row (b, ot, oh, ow), column
// (ci, dt, dy, dx) in Conv3d's weight-flatten order, so the patch embedding is one plain [E, K] GEMM.
// kGather (MAE): only the kept patches, rows [b * nkeep], row (b, j) = patch keep[b * nkeep + j]
template <bool kGather>
__global__ void patchify_kernel(const float* __restrict__ x, int b, int cin, int T, int H, int W, int kt, int kh, int kw,
                                int ot, int oh, int ow, const int* __restrict__ keep, int nkeep, __nv_bfloat16* hi,
                                __nv_bfloat16* lo) {
  const int K = cin * kt * kh * kw;
  const int64_t L = kGather ? int64_t(nkeep) : int64_t(ot) * oh * ow;
  const int64_t items = int64_t(b) * L * K;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    int k = int(i % K);
    const int64_t row = i / K;
    const int dx_ = k % kw;
    k /= kw;
    const int dy_ = k % kh;
    k /= kh;
    const int dt_ = k % kt;
    const int ci = k / kt;
    int64_t l = kGather ? int64_t(keep[row]) : row % L;
    const int64_t bb = row / L;
    const int px = int(l % ow);
    l /= ow;
    const int py = int(l % oh);
    const int pz = int(l / oh);
    const float v = x[(((bb * cin + ci) * T + pz * kt + dt_) * int64_t(H) + py * kh + dy_) * W + px * kw + dx_];
    put_split(hi, lo, i, v);
  }
}
// backward: dy[b, l, :] planes = dx[b, 1 + l, :];  dcls partial / dbias via colsum on the caller side
__global__ void tokens_split_grad_kernel(const float* __restrict__ dx, int b, int l, int c, __nv_bfloat16* dy_hi,
                                         __nv_bfloat16* dy_lo, float* __restrict__ dy_f32) {
  const int64_t items = int64_t(b) * l * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % l);
    const int64_t bb = t / l;
    const float v = dx[(bb * (l + 1) + n + 1) * c + ch];
    put_split(dy_hi, dy_lo, i, v);
    if (dy_f32) dy_f32[i] = v;
  }
}

// ------------------------------------------------------------------------------------------- depthwise pooling conv
// attention_pool with a depthwise Conv3d (groups = head_dim, weight [hd, 1, kt, kh, kw] shared by all heads):
//   src  : qkv GEMM output [B, 1+L, pitch] fp32, this tensor's channels at src_c0 + h*hd + c, bias added on the fly
//          (to real tokens only: the zero padding of the conv stays zero)
//   out  : [B, H, 1+L', hd] fp32 (cls row passes through), to be LayerNorm-ed by ln_fwd_kernel
// kCls = 0: no cls row in src / out / dout / dsrc ([B, L, pitch] -> [B, H, L', hd]).
struct DwPoolParams {
  const float* src; int64_t src_pitch; int src_c0; const float* bias;
  const float* w;  // [hd][kt*kh*kw]
  float* dw;       // weight gradient (bwd_weight: atomically accumulated)
  float* out;
  int B, H, hd, T, Hh, W, oT, oH, oW;
  int kt, kh, kw, st, sh, sw, pt, ph, pw;
  // backward
  const float* dout; float* dsrc; float* wpartials; int has_pool;
};
template <int kCls>
__global__ void dwpool_fwd_kernel(const DwPoolParams p) {
  // one thread = 4 consecutive channels of one (b, head, output token): float4 traffic, taps unrolled
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int hq = p.hd / 4;
  const int taps = p.kt * p.kh * p.kw;
  const int64_t items = int64_t(p.B) * p.H * (Lo + kCls) * hq;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % hq) * 4;
    int64_t t = i / hq;
    const int n = int(t % (Lo + kCls));
    t /= (Lo + kCls);
    const int h = int(t % p.H);
    const int64_t b = t / p.H;
    const int ch = p.src_c0 + h * p.hd + c;
    const float4 bias = p.bias ? *reinterpret_cast<const float4*>(p.bias + ch) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float* sb = p.src + b * int64_t(L + kCls) * p.src_pitch + ch;
    float4 acc;
    if ((kCls && n == 0) || !p.has_pool) {
      const float4 v = *reinterpret_cast<const float4*>(sb + int64_t(n) * p.src_pitch);
      acc = make_float4(v.x + bias.x, v.y + bias.y, v.z + bias.z, v.w + bias.w);
    } else {
      int o = n - kCls;
      const int ox = o % p.oW;
      o /= p.oW;
      const int oy = o % p.oH;
      const int oz = o / p.oH;
      acc = make_float4(0.f, 0.f, 0.f, 0.f);
      const float* w0 = p.w + c * taps;
      for (int kz = 0; kz < p.kt; ++kz) {
        const int iz = oz * p.st - p.pt + kz;
        if (iz < 0 || iz >= p.T) continue;
        for (int ky = 0; ky < p.kh; ++ky) {
          const int iy = oy * p.sh - p.ph + ky;
          if (iy < 0 || iy >= p.Hh) continue;
          for (int kx = 0; kx < p.kw; ++kx) {
            const int ix = ox * p.sw - p.pw + kx;
            if (ix < 0 || ix >= p.W) continue;
            const int64_t pos = kCls + (int64_t(iz) * p.Hh + iy) * p.W + ix;
            const float4 v = *reinterpret_cast<const float4*>(sb + pos * p.src_pitch);
            const int k = (kz * p.kh + ky) * p.kw + kx;
            acc.x = fmaf(v.x + bias.x, w0[k], acc.x);
            acc.y = fmaf(v.y + bias.y, w0[taps + k], acc.y);
            acc.z = fmaf(v.z + bias.z, w0[2 * taps + k], acc.z);
            acc.w = fmaf(v.w + bias.w, w0[3 * taps + k], acc.w);
          }
        }
      }
    }
    *reinterpret_cast<float4*>(p.out + ((b * p.H + h) * int64_t(Lo + kCls) + n) * p.hd + c) = acc;
  }
}
// data gradient: dsrc[b, n, ch] += sum over outputs/taps of dout * w   (gather form; "+=" because q, k, v and the
// block's other consumers all write into the same qkv gradient tensor, which the caller zero-fills first)
template <int kCls>
__global__ void dwpool_bwd_data_kernel(const DwPoolParams p) {
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int hq = p.hd / 4;
  const int taps = p.kt * p.kh * p.kw;
  const int64_t items = int64_t(p.B) * p.H * (L + kCls) * hq;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % hq) * 4;
    int64_t t = i / hq;
    const int n = int(t % (L + kCls));
    t /= (L + kCls);
    const int h = int(t % p.H);
    const int64_t b = t / p.H;
    const float* db = p.dout + ((b * p.H + h) * int64_t(Lo + kCls)) * p.hd + c;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((kCls && n == 0) || !p.has_pool) {
      acc = *reinterpret_cast<const float4*>(db + int64_t(n) * p.hd);
    } else {
      int q = n - kCls;
      const int ix = q % p.W;
      q /= p.W;
      const int iy = q % p.Hh;
      const int iz = q / p.Hh;
      const float* w0 = p.w + c * taps;
      // outputs o with o*s - pad + k == i for some tap k in [0, K):  o in [ceil((i + pad - K + 1) / s), floor((i + pad) / s)]
      const int z_hi = min(p.oT - 1, (iz + p.pt) / p.st), z_lo = max(0, (iz + p.pt - p.kt + p.st) / p.st);
      const int y_hi = min(p.oH - 1, (iy + p.ph) / p.sh), y_lo = max(0, (iy + p.ph - p.kh + p.sh) / p.sh);
      const int x_hi = min(p.oW - 1, (ix + p.pw) / p.sw), x_lo = max(0, (ix + p.pw - p.kw + p.sw) / p.sw);
      for (int oz = z_lo; oz <= z_hi; ++oz) {
        const int kz = iz + p.pt - oz * p.st;
        for (int oy = y_lo; oy <= y_hi; ++oy) {
          const int ky = iy + p.ph - oy * p.sh;
          for (int ox = x_lo; ox <= x_hi; ++ox) {
            const int kx = ix + p.pw - ox * p.sw;
            const int64_t opos = kCls + (int64_t(oz) * p.oH + oy) * p.oW + ox;
            const float4 g = *reinterpret_cast<const float4*>(db + opos * p.hd);
            const int k = (kz * p.kh + ky) * p.kw + kx;
            acc.x = fmaf(g.x, w0[k], acc.x);
            acc.y = fmaf(g.y, w0[taps + k], acc.y);
            acc.z = fmaf(g.z, w0[2 * taps + k], acc.z);
            acc.w = fmaf(g.w, w0[3 * taps + k], acc.w);
          }
        }
      }
    }
    float4* d = reinterpret_cast<float4*>(p.dsrc + (b * int64_t(L + kCls) + n) * p.src_pitch + p.src_c0 + h * p.hd + c);
    float4 o = *d;
    o.x += acc.x; o.y += acc.y; o.z += acc.z; o.w += acc.w;
    *d = o;
  }
}
// data gradient, scatter form, for strongly strided pooling (the K/V pools: stride 8 / 4 with a 3x3x3 kernel): work
// is proportional to the (few) OUTPUT positions x 27 taps instead of scanning every input position for taps that
// almost never exist.  Windows of neighbouring output frames overlap in time, hence atomic adds.
template <int kCls>
__global__ void dwpool_bwd_data_scatter_kernel(const DwPoolParams p) {
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int hq = p.hd / 4;
  const int taps = p.kt * p.kh * p.kw;
  const int64_t items = int64_t(p.B) * p.H * (Lo + kCls) * hq;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % hq) * 4;
    int64_t t = i / hq;
    const int n = int(t % (Lo + kCls));
    t /= (Lo + kCls);
    const int h = int(t % p.H);
    const int64_t b = t / p.H;
    const float4 g = *reinterpret_cast<const float4*>(p.dout + ((b * p.H + h) * int64_t(Lo + kCls) + n) * p.hd + c);
    float* db = p.dsrc + b * int64_t(L + kCls) * p.src_pitch + p.src_c0 + h * p.hd + c;
    if (kCls && n == 0) {  // cls row passes through the pooling
      atomicAdd(db + 0, g.x); atomicAdd(db + 1, g.y); atomicAdd(db + 2, g.z); atomicAdd(db + 3, g.w);
      continue;
    }
    int o = n - kCls;
    const int ox = o % p.oW;
    o /= p.oW;
    const int oy = o % p.oH;
    const int oz = o / p.oH;
    const float* w0 = p.w + c * taps;
    for (int kz = 0; kz < p.kt; ++kz) {
      const int iz = oz * p.st - p.pt + kz;
      if (iz < 0 || iz >= p.T) continue;
      for (int ky = 0; ky < p.kh; ++ky) {
        const int iy = oy * p.sh - p.ph + ky;
        if (iy < 0 || iy >= p.Hh) continue;
        for (int kx = 0; kx < p.kw; ++kx) {
          const int ix = ox * p.sw - p.pw + kx;
          if (ix < 0 || ix >= p.W) continue;
          const int k = (kz * p.kh + ky) * p.kw + kx;
          float* d = db + (kCls + (int64_t(iz) * p.Hh + iy) * p.W + ix) * p.src_pitch;
          atomicAdd(d + 0, g.x * w0[k]);
          atomicAdd(d + 1, g.y * w0[taps + k]);
          atomicAdd(d + 2, g.z * w0[2 * taps + k]);
          atomicAdd(d + 3, g.w * w0[3 * taps + k]);
        }
      }
    }
  }
}
// weight gradient partials: wpartials[block][c][tap] = sum over the block's (b, h, out position) slab.
// blockDim = hd * PL threads (channel-fastest => coalesced), PL position lanes per block, smem reduce over the lanes.
template <int kCls>
__global__ void __launch_bounds__(512) dwpool_bwd_weight_kernel(const DwPoolParams p) {
  extern __shared__ float wsm[];  // [PL][hd][27]
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int taps = p.kt * p.kh * p.kw;
  const int PL = blockDim.x / p.hd;
  const int c = threadIdx.x % p.hd, pl = threadIdx.x / p.hd;
  const int64_t total = int64_t(p.B) * p.H * Lo;
  const int64_t per = (total + gridDim.x - 1) / gridDim.x;
  const int64_t i0 = blockIdx.x * per, i1 = min(total, i0 + per);
  float acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.f;
  if (pl < PL) {
    for (int64_t i = i0 + pl; i < i1; i += PL) {
      int o = int(i % Lo);
      const int64_t bh = i / Lo;
      const int h = int(bh % p.H);
      const int64_t b = bh / p.H;
      const int ch = p.src_c0 + h * p.hd + c;
      const float bias = p.bias ? p.bias[ch] : 0.f;
      const float g = p.dout[(bh * int64_t(Lo + kCls) + kCls + o) * p.hd + c];
      const float* sb = p.src + b * int64_t(L + kCls) * p.src_pitch + ch;
      const int ox = o % p.oW;
      o /= p.oW;
      const int oy = o % p.oH;
      const int oz = o / p.oH;
#pragma unroll
      for (int kz = 0; kz < 3; ++kz) {
        const int iz = oz * p.st - p.pt + kz;
        if (kz >= p.kt || iz < 0 || iz >= p.T) continue;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          const int iy = oy * p.sh - p.ph + ky;
          if (ky >= p.kh || iy < 0 || iy >= p.Hh) continue;
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const int ix = ox * p.sw - p.pw + kx;
            if (kx >= p.kw || ix < 0 || ix >= p.W) continue;
            const int64_t pos = kCls + (int64_t(iz) * p.Hh + iy) * p.W + ix;
            acc[(kz * 3 + ky) * 3 + kx] = fmaf(g, sb[pos * p.src_pitch] + bias, acc[(kz * 3 + ky) * 3 + kx]);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 27; ++k) wsm[(pl * p.hd + c) * 27 + k] = acc[k];
  }
  __syncthreads();
  // taps are indexed (kz*3+ky)*3+kx in the accumulators; the parameter layout is (kz*kh+ky)*kw+kx
  for (int j = threadIdx.x; j < p.hd * taps; j += blockDim.x) {
    const int cc = j / taps, k = j - cc * taps;
    const int kx = k % p.kw, ky = (k / p.kw) % p.kh, kz = k / (p.kw * p.kh);
    float sum = 0.f;
    for (int l = 0; l < PL; ++l) sum += wsm[(l * p.hd + cc) * 27 + (kz * 3 + ky) * 3 + kx];
    atomicAdd(p.dw + size_t(cc) * taps + k, sum);  // one atomic per (channel, tap) and block into the zeroed slot
  }
}

// ------------------------------------------------------------------------------------------- rel-pos softmax
// P[bh, q, k] = softmax_k( S[bh, q, k] + bias(q, k) ),  bias = RQ[q-1, ih(qh,kh)] + RQ[q-1, Lh + iw] + RQ[q-1, Lh+Lw + it]
// for q > 0 and k > 0 (cls row / column carry no bias); index = floor(i*max(nk/nq,1) - j*max(nq/nk,1) + (nk-1)*max(nq/nk,1)).
// kCls = 0: no cls row / column, the bias is on every query and key.  kRelT = false: spatial terms only (no Rt table,
// REL_POS_SPATIAL without REL_POS_TEMPORAL), RQ rows are [Rh | Rw].
struct SoftmaxParams {
  const float* S; int64_t s_pitch;          // [BH, Nq, s_pitch]
  const float* RQ; int64_t rq_pitch;        // [BH, Lq, rq_pitch]  (may be null: no rel-pos)
  __nv_bfloat16* p_hi; __nv_bfloat16* p_lo; int64_t p_pitch;  // [BH, Nq, p_pitch], pad columns zeroed
  int BH, Nq, Nk;
  int qt, qh, qw, kt, kh, kw;
  int Lh, Lw, Lt;
  float rh_q, rh_k, rw_q, rw_k, rt_q, rt_k;  // index ratios
  // backward
  const float* dP; int64_t dp_pitch;        // [BH, Nq, dp_pitch] fp32
  __nv_bfloat16* ds_hi; __nv_bfloat16* ds_lo; int64_t ds_pitch;
  float* dRQ;                                // [BH, Lq, rq_pitch] fp32
};
__device__ __forceinline__ int rel_index(int i, int j, float rq, float rk, int nk) {
  return int(floorf(float(i) * rq - float(j) * rk + float(nk - 1) * rk));
}
template <int kCls, bool kRelT>
__global__ void __launch_bounds__(256) softmax_relpos_fwd_kernel(const SoftmaxParams p) {
  // one warp per (bh, q) row; the biased scores are computed ONCE into a per-warp shared-memory row
  extern __shared__ float srow[];  // [8 warps][Nk]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float* buf = srow + size_t(wid) * p.Nk;
  const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const int64_t rows = int64_t(p.BH) * p.Nq;
  const int khw = p.kh * p.kw;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const int q = int(r % p.Nq);
    const int64_t bh = r / p.Nq;
    const float* s = p.S + r * p.s_pitch;
    const float* rq = (p.RQ && q >= kCls) ? p.RQ + (bh * (p.Nq - kCls) + (q - kCls)) * p.rq_pitch : nullptr;
    int qz = 0, qy = 0, qx = 0;
    if (q >= kCls) {
      int t = q - kCls;
      qx = t % p.qw;
      t /= p.qw;
      qy = t % p.qh;
      qz = t / p.qh;
    }
    const float bh0 = float(qy) * p.rh_q + float(p.kh - 1) * p.rh_k;
    const float bw0 = float(qx) * p.rw_q + float(p.kw - 1) * p.rw_k;
    const float bt0 = float(qz) * p.rt_q + float(p.kt - 1) * p.rt_k;
    float mx = -INFINITY;
    for (int k = lane; k < p.Nk; k += 32) {
      float v = s[k];
      if (rq && k >= kCls) {
        const int t = k - kCls;
        const int kz = t / khw;
        const int rem = t - kz * khw;
        const int ky = rem / p.kw;
        const int kx = rem - ky * p.kw;
        if (kRelT)
          v += rq[int(floorf(bh0 - float(ky) * p.rh_k))] + rq[p.Lh + int(floorf(bw0 - float(kx) * p.rw_k))] +
               rq[p.Lh + p.Lw + int(floorf(bt0 - float(kz) * p.rt_k))];
        else
          v += rq[int(floorf(bh0 - float(ky) * p.rh_k))] + rq[p.Lh + int(floorf(bw0 - float(kx) * p.rw_k))];
      }
      buf[k] = v;
      mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int k = lane; k < p.Nk; k += 32) {
      const float e = expf(buf[k] - mx);
      buf[k] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int k = lane; k < p.p_pitch; k += 32) put_split(p.p_hi, p.p_lo, r * p.p_pitch + k, k < p.Nk ? buf[k] * inv : 0.f);
    __syncwarp();
  }
}
// dS = P * (dP - sum_k P*dP) -> planes (pad columns zero);  dRQ[q-1, j] = sum over k with index j of dS[q, k]
template <int kCls, bool kRelT>
__global__ void __launch_bounds__(256) softmax_relpos_bwd_kernel(const SoftmaxParams p) {
  // one warp per row.  dS is staged in a per-warp shared row; the relative-position gradient is reduced per key AXIS
  // first (sum over the other two axes, one lane per axis coordinate) and only then scattered into the table bins,
  // which replaces 3*Nk heavily colliding shared atomics per row by kh+kw+kt of them.
  extern __shared__ float smem[];  // [8 warps][Nk + Lh + Lw + Lt]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int Ltot = p.Lh + p.Lw + p.Lt;
  float* buf = smem + size_t(wid) * (p.Nk + Ltot);
  float* bins = buf + p.Nk;
  const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const int64_t rows = int64_t(p.BH) * p.Nq;
  const int khw = p.kh * p.kw;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const int q = int(r % p.Nq);
    const int64_t bh = r / p.Nq;
    const float* dp = p.dP + r * p.dp_pitch;
    float dot = 0.f;
    for (int k = lane; k < p.Nk; k += 32) {
      const float pv = get_split(p.p_hi, p.p_lo, r * p.p_pitch + k);
      buf[k] = pv;
      dot = fmaf(pv, dp[k], dot);
    }
    dot = warp_sum(dot);
    const bool rel = p.dRQ != nullptr && q >= kCls;
    if (rel)
      for (int j = lane; j < Ltot; j += 32) bins[j] = 0.f;
    for (int k = lane; k < p.ds_pitch; k += 32) {
      float ds = 0.f;
      if (k < p.Nk) {
        ds = buf[k] * (dp[k] - dot);
        buf[k] = ds;
      }
      put_split(p.ds_hi, p.ds_lo, r * p.ds_pitch + k, ds);
    }
    __syncwarp();
    if (rel) {
      int t = q - kCls;
      const int qx = t % p.qw;
      t /= p.qw;
      const int qy = t % p.qh;
      const int qz = t / p.qh;
      const float* g = buf + kCls;  // key grid [kt][kh][kw] behind the cls column
      for (int a = lane; a < p.kh + p.kw + (kRelT ? p.kt : 0); a += 32) {
        float sum = 0.f;
        int bin;
        if (a < p.kh) {
          for (int kz = 0; kz < p.kt; ++kz)
            for (int kx = 0; kx < p.kw; ++kx) sum += g[kz * khw + a * p.kw + kx];
          bin = rel_index(qy, a, p.rh_q, p.rh_k, p.kh);
        } else if (a < p.kh + p.kw) {
          const int kx = a - p.kh;
          for (int kz = 0; kz < p.kt; ++kz)
            for (int ky = 0; ky < p.kh; ++ky) sum += g[kz * khw + ky * p.kw + kx];
          bin = p.Lh + rel_index(qx, kx, p.rw_q, p.rw_k, p.kw);
        } else {
          const int kz = a - p.kh - p.kw;
          for (int j = 0; j < khw; ++j) sum += g[kz * khw + j];
          bin = p.Lh + p.Lw + rel_index(qz, kz, p.rt_q, p.rt_k, p.kt);
        }
        atomicAdd(&bins[bin], sum);
      }
      __syncwarp();
      float* o = p.dRQ + (bh * (p.Nq - kCls) + (q - kCls)) * p.rq_pitch;
      for (int j = lane; j < p.rq_pitch; j += 32) o[j] = j < Ltot ? bins[j] : 0.f;
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------- head merge / split
// merged[b, n, h*hd + c] = O[b, h, n, c] + (n > 0 ? q[b, h, n, c] : 0)   -> planes (input of the proj Linear)
// (kCls = 0: the residual is added on every row)
template <int kCls>
__global__ void attn_merge_kernel(const float* __restrict__ O, const __nv_bfloat16* __restrict__ q_hi,
                                  const __nv_bfloat16* __restrict__ q_lo, int B, int H, int N, int hd, int residual,
                                  __nv_bfloat16* __restrict__ m_hi, __nv_bfloat16* __restrict__ m_lo) {
  const int64_t items = int64_t(B) * N * H * hd;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % hd);
    int64_t t = i / hd;
    const int h = int(t % H);
    t /= H;
    const int n = int(t % N);
    const int64_t b = t / N;
    const int64_t src = ((b * H + h) * N + n) * hd + c;
    float v = O[src];
    if (residual && n >= kCls) v += get_split(q_hi, q_lo, src);
    put_split(m_hi, m_lo, i, v);
  }
}
// backward of the merge: dO[b, h, n, c] = dM[b, n, h*hd + c] -> planes (operand of dP / dV GEMMs) and the
// residual-pooling gradient dq[b, h, n, c] (= dM for n > 0, 0 for the cls row) as fp32 initialisation of dq
template <int kCls>
__global__ void attn_split_grad_kernel(const float* __restrict__ dM, int B, int H, int N, int hd, int residual,
                                       __nv_bfloat16* __restrict__ do_hi, __nv_bfloat16* __restrict__ do_lo,
                                       float* __restrict__ dq) {
  const int64_t items = int64_t(B) * H * N * hd;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % hd);
    int64_t t = i / hd;
    const int n = int(t % N);
    t /= N;
    const int h = int(t % H);
    const int64_t b = t / H;
    const float v = dM[(b * N + n) * int64_t(H) * hd + h * hd + c];
    put_split(do_hi, do_lo, i, v);
    dq[i] = (residual && n >= kCls) ? v : 0.f;
  }
}

// ------------------------------------------------------------------------------------------- residual combines / GELU
// out = a [+ a_bias] + s * (y + y_bias)       fp32; s = per-sample stochastic-depth scale (null = 1)
__global__ void residual_add_kernel(const float* __restrict__ a, const float* __restrict__ a_bias,
                                    const float* __restrict__ y, const float* __restrict__ y_bias,
                                    const float* __restrict__ scale, int64_t rows, int c, int64_t rows_per_sample,
                                    float* __restrict__ out) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t r = i / c;
    float v = a[i] + (a_bias ? a_bias[ch] : 0.f);
    const float s = scale ? scale[r / rows_per_sample] : 1.f;
    v += s * (y[i] + (y_bias ? y_bias[ch] : 0.f));
    out[i] = v;
  }
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
  return 0.5f * (1.f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
}
// h = gelu(y + bias) -> planes
__global__ void bias_gelu_kernel(const float* __restrict__ y, const float* __restrict__ bias, int64_t rows, int c,
                                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x)
    put_split(hi, lo, i, gelu_erf(y[i] + bias[int(i % c)]));
}
// dpre = dh * gelu'(y + bias) -> planes + fp32 (for the bias-gradient column sum)
__global__ void bias_gelu_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ y,
                                     const float* __restrict__ bias, int64_t rows, int c,
                                     __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                     float* __restrict__ dpre) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const float v = dh[i] * gelu_erf_grad(y[i] + bias[int(i % c)]);
    put_split(hi, lo, i, v);
    dpre[i] = v;
  }
}
// scale[b] * src -> planes (+ fp32): gradient entering a residual branch (stochastic depth scale; null = 1)
__global__ void scale_split_kernel(const float* __restrict__ src, const float* __restrict__ scale, int64_t rows, int c,
                                   int64_t rows_per_sample, __nv_bfloat16* __restrict__ hi,
                                   __nv_bfloat16* __restrict__ lo, float* __restrict__ f32) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const float v = src[i] * (scale ? scale[(i / c) / rows_per_sample] : 1.f);
    put_split(hi, lo, i, v);
    if (f32) f32[i] = v;
  }
}

// ------------------------------------------------------------------------------------------- max-pool skip on tokens
// attention_pool(x, MaxPool3d) of MultiScaleBlock (attention.py:485-489, :496): cls passes through, first max wins
// (kCls = 0: no pass-through row)
struct TokPoolParams {
  const float* x; float* out; uint8_t* argmax;
  int B, C, T, Hh, W, oT, oH, oW, kt, kh, kw, st, sh, sw, pt, ph, pw;
  const float* dout; float* dx; int dx_accumulate;
};
template <int kCls>
__global__ void token_maxpool_fwd_kernel(const TokPoolParams p) {
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int64_t items = int64_t(p.B) * (Lo + kCls) * p.C;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % p.C);
    int64_t t = i / p.C;
    const int n = int(t % (Lo + kCls));
    const int64_t b = t / (Lo + kCls);
    const float* xb = p.x + b * int64_t(L + kCls) * p.C + c;
    if (kCls && n == 0) {
      p.out[i] = xb[0];
      p.argmax[i] = 0;
      continue;
    }
    int o = n - kCls;
    const int ox = o % p.oW;
    o /= p.oW;
    const int oy = o % p.oH;
    const int oz = o / p.oH;
    float best = -INFINITY;
    uint8_t arg = 0;
    for (int kz = 0; kz < p.kt; ++kz) {
      const int iz = oz * p.st - p.pt + kz;
      if (iz < 0 || iz >= p.T) continue;
      for (int ky = 0; ky < p.kh; ++ky) {
        const int iy = oy * p.sh - p.ph + ky;
        if (iy < 0 || iy >= p.Hh) continue;
        for (int kx = 0; kx < p.kw; ++kx) {
          const int ix = ox * p.sw - p.pw + kx;
          if (ix < 0 || ix >= p.W) continue;
          const float v = xb[(kCls + (int64_t(iz) * p.Hh + iy) * p.W + ix) * p.C];
          if (v > best) {
            best = v;
            arg = uint8_t((kz * p.kh + ky) * p.kw + kx);
          }
        }
      }
    }
    p.out[i] = best;
    p.argmax[i] = arg;
  }
}
template <int kCls>
__global__ void token_maxpool_bwd_kernel(const TokPoolParams p) {
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int64_t items = int64_t(p.B) * (L + kCls) * p.C;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % p.C);
    int64_t t = i / p.C;
    const int n = int(t % (L + kCls));
    const int64_t b = t / (L + kCls);
    const float* db = p.dout + b * int64_t(Lo + kCls) * p.C + c;
    const uint8_t* ab = p.argmax + b * int64_t(Lo + kCls) * p.C + c;
    float acc = 0.f;
    if (kCls && n == 0) {
      acc = db[0];
    } else {
      int q = n - kCls;
      const int ix = q % p.W;
      q /= p.W;
      const int iy = q % p.Hh;
      const int iz = q / p.Hh;
      // only the outputs whose window contains this input: o in [ceil((i + pad - K + 1) / s), floor((i + pad) / s)]
      const int z_hi = min(p.oT - 1, (iz + p.pt) / p.st), z_lo = max(0, (iz + p.pt - p.kt + p.st) / p.st);
      const int y_hi = min(p.oH - 1, (iy + p.ph) / p.sh), y_lo = max(0, (iy + p.ph - p.kh + p.sh) / p.sh);
      const int x_hi = min(p.oW - 1, (ix + p.pw) / p.sw), x_lo = max(0, (ix + p.pw - p.kw + p.sw) / p.sw);
      for (int oz = z_lo; oz <= z_hi; ++oz) {
        const int kz = iz + p.pt - oz * p.st;
        for (int oy = y_lo; oy <= y_hi; ++oy) {
          const int ky = iy + p.ph - oy * p.sh;
          for (int ox = x_lo; ox <= x_hi; ++ox) {
            const int kx = ix + p.pw - ox * p.sw;
            const int64_t opos = (kCls + (int64_t(oz) * p.oH + oy) * p.oW + ox) * p.C;
            if (ab[opos] == uint8_t((kz * p.kh + ky) * p.kw + kx)) acc += db[opos];
          }
        }
      }
    }
    p.dx[i] = p.dx_accumulate ? p.dx[i] + acc : acc;
  }
}

}  // namespace sfb

using namespace sfb;
typedef __nv_bfloat16 bf;

extern "C" int sfb_layernorm_fwd(const float* x, int64_t x_pitch, int64_t rows, int32_t c, const float* gamma,
                                 const float* beta, float eps, void* o_hi, void* o_lo, float* o_f32, int64_t o_pitch,
                                 float* mean, float* rstd, void* stream) {
  if (c > 32 * LN_MAX_PER_LANE) {
    set_error("sfb_layernorm_fwd: c=%d exceeds %d", c, 32 * LN_MAX_PER_LANE);
    return -10;
  }
  if (rows == 0) return 0;
  if (c <= 96) ln_fwd_kernel<3><<<mv_grid(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, rows, c, gamma, beta, eps, (bf*)o_hi,
                                                                         (bf*)o_lo, o_f32, o_pitch, mean, rstd);
  else if (c <= 192) ln_fwd_kernel<6><<<mv_grid(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, rows, c, gamma, beta, eps, (bf*)o_hi,
                                                                         (bf*)o_lo, o_f32, o_pitch, mean, rstd);
  else if (c <= 384) ln_fwd_kernel<12><<<mv_grid(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, rows, c, gamma, beta, eps, (bf*)o_hi,
                                                                         (bf*)o_lo, o_f32, o_pitch, mean, rstd);
  else if (c <= 768) ln_fwd_kernel<24><<<mv_grid(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, rows, c, gamma, beta, eps, (bf*)o_hi,
                                                                         (bf*)o_lo, o_f32, o_pitch, mean, rstd);
  else if (c <= 1024) ln_fwd_kernel<32><<<mv_grid(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, rows, c, gamma, beta, eps, (bf*)o_hi,
                                                                         (bf*)o_lo, o_f32, o_pitch, mean, rstd);
  else ln_fwd_kernel<40><<<mv_grid(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, rows, c, gamma, beta, eps, (bf*)o_hi,
                                                                         (bf*)o_lo, o_f32, o_pitch, mean, rstd);
  return launch_status("sfb_layernorm_fwd");
}
extern "C" int32_t sfb_rowslab_blocks(int64_t rows) {
  // one slab per 8 rows (= one row per warp of a 256-thread block) until the machine is full: the deep stages of MViT have
  // only ~1.6 k token rows, and 64-row slabs left 5/6 of the SMs idle there (ncu r2a: 25 blocks, 127 us for 14 MB)
  int64_t b = (rows + 7) / 8;
  if (b > kGridSms * 2) b = kGridSms * 2;   // (more slabs only move the time into the partial-merge kernel: ncu r2h)
  return int32_t(b < 1 ? 1 : b);
}
// out_k[ch] (=|+=) sum_b partials[b][k][ch]: fp64 merge of row-slab partials, one 64-thread block per (channel, k)
__global__ void partial_merge2_kernel(const float* __restrict__ partials, int nblocks, int K, int c, float* o0, float* o1,
                                      int accumulate) {
  __shared__ double sm[64];
  const int ch = blockIdx.x, k = blockIdx.y;
  double s = 0.0;
  for (int b = threadIdx.x; b < nblocks; b += 64) s += double(partials[(size_t(b) * K + k) * c + ch]);
  sm[threadIdx.x] = s;
  __syncthreads();
  for (int o = 32; o > 0; o >>= 1) {
    if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o];
    __syncthreads();
  }
  float* out = k == 0 ? o0 : o1;
  if (threadIdx.x == 0 && out) out[ch] = accumulate ? out[ch] + float(sm[0]) : float(sm[0]);
}
extern "C" int sfb_layernorm_bwd(const float* dy, int64_t dy_pitch, const float* x, int64_t x_pitch, int64_t rows,
                                 int32_t c, const float* gamma, const float* mean, const float* rstd, float* dx,
                                 int64_t dx_pitch, int32_t dx_accumulate, float* dgamma, float* dbeta,
                                 int32_t param_accumulate, float* partials, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (c > 32 * LN_MAX_PER_LANE) {
    set_error("sfb_layernorm_bwd: c=%d exceeds %d", c, 32 * LN_MAX_PER_LANE);
    return -10;
  }
  const int nb = sfb_rowslab_blocks(rows);
  if (c <= 96) ln_bwd_kernel<3><<<nb, 256, size_t(8) * 2 * c * sizeof(float), stream>>>(dy, dy_pitch, x, x_pitch, rows, c, gamma, mean,
                                                                        rstd, dx, dx_pitch, dx_accumulate, partials);
  else if (c <= 192) ln_bwd_kernel<6><<<nb, 256, size_t(8) * 2 * c * sizeof(float), stream>>>(dy, dy_pitch, x, x_pitch, rows, c, gamma, mean,
                                                                        rstd, dx, dx_pitch, dx_accumulate, partials);
  else if (c <= 384) ln_bwd_kernel<12><<<nb, 256, size_t(8) * 2 * c * sizeof(float), stream>>>(dy, dy_pitch, x, x_pitch, rows, c, gamma, mean,
                                                                        rstd, dx, dx_pitch, dx_accumulate, partials);
  else if (c <= 768) ln_bwd_kernel<24><<<nb, 256, size_t(8) * 2 * c * sizeof(float), stream>>>(dy, dy_pitch, x, x_pitch, rows, c, gamma, mean,
                                                                        rstd, dx, dx_pitch, dx_accumulate, partials);
  else if (c <= 1024) ln_bwd_wide_kernel<32><<<nb, 256, 0, stream>>>(dy, dy_pitch, x, x_pitch, rows, c, gamma, mean, rstd, dx,
                                                                    dx_pitch, dx_accumulate, partials);
  else ln_bwd_wide_kernel<40><<<nb, 256, 0, stream>>>(dy, dy_pitch, x, x_pitch, rows, c, gamma, mean, rstd, dx, dx_pitch,
                                                     dx_accumulate, partials);
  if (int rc = launch_status("sfb_layernorm_bwd")) return rc;
  partial_merge2_kernel<<<dim3(c, 2), 64, 0, stream>>>(partials, nb, 2, c, dgamma, dbeta, param_accumulate);
  return launch_status("sfb_layernorm_bwd(merge)");
}
extern "C" int sfb_colsum(const float* src, int64_t pitch, int64_t rows, int32_t c, float* out, int32_t accumulate,
                          float* partials, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int nb = sfb_rowslab_blocks(rows);
  if (c % 4 == 0 && pitch % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0)
    colsum4_kernel<<<nb, 256, 0, stream>>>(src, pitch, rows, c, partials);
  else
    colsum_kernel<<<nb, 256, 0, stream>>>(src, pitch, rows, c, partials);
  if (int rc = launch_status("sfb_colsum")) return rc;
  partial_merge2_kernel<<<dim3(c, 1), 64, 0, stream>>>(partials, nb, 1, c, out, nullptr, accumulate);
  return launch_status("sfb_colsum(merge)");
}
extern "C" int sfb_tokens_assemble(const float* y, const float* bias, const float* cls, const float* pos_spatial,
                                   const float* pos_temporal, const float* pos_class, int32_t b, int32_t l, int32_t hw,
                                   int32_t c, float* x, void* stream) {
  const bool any = pos_spatial || pos_temporal || pos_class;
  if (any && !(pos_spatial && pos_temporal && pos_class && hw > 0 && l % hw == 0)) {
    set_error("sfb_tokens_assemble: positions need all three tables and hw=%d dividing l=%d", hw, l);
    return -10;
  }
  const int64_t items = int64_t(b) * (l + 1) * c;
  tokens_assemble_kernel<<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(
      y, bias, cls, pos_spatial, pos_temporal, pos_class, b, l, any ? hw : 1, c, x);
  return launch_status("sfb_tokens_assemble");
}
extern "C" int32_t sfb_segment_slabs(int32_t groups, int32_t seg_rows) {
  // about two blocks per SM over all groups, and at least 8 rows per slab
  int32_t s = (296 + groups - 1) / std::max(groups, 1);
  s = std::min(s, (seg_rows + 7) / 8);
  return std::max(s, 1);
}
static int segment_rowsum(const float* src, int c, int n_outer, int64_t outer_stride, int64_t group_stride, int seg_rows,
                          int groups, float scale, float* out, float* partials, cudaStream_t stream) {
  const int nslab = sfb_segment_slabs(groups, seg_rows);
  const int threads = std::min(256, (c + 31) / 32 * 32);
  segment_rowsum_partial_kernel<<<dim3(nslab, groups), threads, 0, stream>>>(src, c, n_outer, outer_stride, group_stride,
                                                                             seg_rows, partials);
  if (int rc = launch_status("segment_rowsum")) return rc;
  segment_rowsum_merge_kernel<<<mv_grid(int64_t(groups) * c, 256), 256, 0, stream>>>(partials, nslab, groups, c, scale,
                                                                                    out);
  return launch_status("segment_rowsum(merge)");
}
extern "C" int sfb_pos_embed_sep_bwd(const float* dx, int32_t b, int32_t t, int32_t hw, int32_t c, float* dps, float* dpt,
                                     float* dpc, float* partials, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (b < 1 || t < 1 || hw < 1 || c < 1) {
    set_error("sfb_pos_embed_sep_bwd: b=%d t=%d hw=%d c=%d", b, t, hw, c);
    return -10;
  }
  pos_sep_bwd_spatial_kernel<<<mv_grid(int64_t(hw + 1) * c, 256), 256, 0, stream>>>(dx, b, t, hw, c, dps, dpc);
  if (int rc = launch_status("sfb_pos_embed_sep_bwd")) return rc;
  const int64_t n = 1 + int64_t(t) * hw;
  return segment_rowsum(dx + c, c, b, n, hw, hw, t, 1.f, dpt, partials, stream);
}
extern "C" int sfb_token_mean_fwd(const float* x, int32_t b, int32_t n, int32_t c, float* out, float* partials,
                                  void* stream) {
  if (b < 1 || n < 2 || c < 1) {
    set_error("sfb_token_mean_fwd: b=%d n=%d c=%d (needs a token besides cls)", b, n, c);
    return -10;
  }
  return segment_rowsum(x + c, c, 1, 0, n, n - 1, b, 1.f / float(n - 1), out, partials, (cudaStream_t)stream);
}
extern "C" int sfb_token_mean_bwd(const float* dmean, int32_t b, int32_t n, int32_t c, float* dx, void* stream) {
  if (b < 1 || n < 2 || c < 1) {
    set_error("sfb_token_mean_bwd: b=%d n=%d c=%d (needs a token besides cls)", b, n, c);
    return -10;
  }
  token_mean_bwd_kernel<1><<<mv_grid(int64_t(b) * n * c, 256), 256, 0, (cudaStream_t)stream>>>(dmean, b, n, c,
                                                                                              1.f / float(n - 1), dx);
  return launch_status("sfb_token_mean_bwd");
}
extern "C" int sfb_token_mean_all_fwd(const float* x, int32_t b, int32_t n, int32_t c, float* out, float* partials,
                                      void* stream) {
  if (b < 1 || n < 1 || c < 1) {
    set_error("sfb_token_mean_all_fwd: b=%d n=%d c=%d", b, n, c);
    return -10;
  }
  return segment_rowsum(x, c, 1, 0, n, n, b, 1.f / float(n), out, partials, (cudaStream_t)stream);
}
extern "C" int sfb_token_mean_all_bwd(const float* dmean, int32_t b, int32_t n, int32_t c, float* dx, void* stream) {
  if (b < 1 || n < 1 || c < 1) {
    set_error("sfb_token_mean_all_bwd: b=%d n=%d c=%d", b, n, c);
    return -10;
  }
  token_mean_bwd_kernel<0><<<mv_grid(int64_t(b) * n * c, 256), 256, 0, (cudaStream_t)stream>>>(dmean, b, n, c,
                                                                                              1.f / float(n), dx);
  return launch_status("sfb_token_mean_all_bwd");
}
extern "C" int sfb_tokens_assemble_joint(const float* y, const float* bias, const float* cls, const float* pos, int32_t b,
                                         int32_t l, int32_t c, float* x, void* stream) {
  if (b < 1 || l < 1 || c < 1) {
    set_error("sfb_tokens_assemble_joint: b=%d l=%d c=%d", b, l, c);
    return -10;
  }
  const int64_t items = int64_t(b) * (l + (cls ? 1 : 0)) * c;
  tokens_assemble_joint_kernel<<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(y, bias, cls, pos, b, l, c, x);
  return launch_status("sfb_tokens_assemble_joint");
}
extern "C" int sfb_pos_embed_joint_bwd(const float* dx, int32_t b, int32_t n, int32_t c, float* dpos, void* stream) {
  if (b < 1 || n < 1 || c < 1) {
    set_error("sfb_pos_embed_joint_bwd: b=%d n=%d c=%d", b, n, c);
    return -10;
  }
  pos_joint_bwd_kernel<<<mv_grid(int64_t(n) * c, 256), 256, 0, (cudaStream_t)stream>>>(dx, b, n, c, dpos);
  return launch_status("sfb_pos_embed_joint_bwd");
}
extern "C" int sfb_patchify(const float* x, int32_t b, int32_t cin, int32_t t, int32_t h, int32_t w, int32_t kt, int32_t kh,
                            int32_t kw, void* hi, void* lo, void* stream) {
  if (kt < 1 || kh < 1 || kw < 1 || t < kt || h < kh || w < kw || (cin * kt * kh * kw) % 8 != 0) {
    set_error("sfb_patchify: kernel %dx%dx%d over %dx%dx%d with %d channels (K must be a multiple of 8)", kt, kh, kw, t,
              h, w, cin);
    return -10;
  }
  const int ot = t / kt, oh = h / kh, ow = w / kw;
  const int64_t items = int64_t(b) * ot * oh * ow * cin * kt * kh * kw;
  patchify_kernel<false><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(x, b, cin, t, h, w, kt, kh, kw, ot, oh,
                                                                                ow, nullptr, 0, (bf*)hi, (bf*)lo);
  return launch_status("sfb_patchify");
}
extern "C" int sfb_patchify_gather(const float* x, int32_t b, int32_t cin, int32_t t, int32_t h, int32_t w, int32_t kt,
                                   int32_t kh, int32_t kw, const int32_t* keep, int32_t nkeep, void* hi, void* lo,
                                   void* stream) {
  if (!keep) return sfb_patchify(x, b, cin, t, h, w, kt, kh, kw, hi, lo, stream);
  if (kt < 1 || kh < 1 || kw < 1 || t < kt || h < kh || w < kw || (cin * kt * kh * kw) % 8 != 0 || nkeep < 1 ||
      int64_t(nkeep) > int64_t(t / kt) * (h / kh) * (w / kw)) {
    set_error("sfb_patchify_gather: kernel %dx%dx%d over %dx%dx%d with %d channels, %d kept patches", kt, kh, kw, t, h,
              w, cin, nkeep);
    return -10;
  }
  const int ot = t / kt, oh = h / kh, ow = w / kw;
  const int64_t items = int64_t(b) * nkeep * cin * kt * kh * kw;
  patchify_kernel<true><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(x, b, cin, t, h, w, kt, kh, kw, ot, oh,
                                                                               ow, keep, nkeep, (bf*)hi, (bf*)lo);
  return launch_status("sfb_patchify_gather");
}
extern "C" int sfb_tokens_split_grad(const float* dx, int32_t b, int32_t l, int32_t c, void* dy_hi, void* dy_lo,
                                     float* dy_f32, void* stream) {
  const int64_t items = int64_t(b) * l * c;
  tokens_split_grad_kernel<<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dx, b, l, c, (bf*)dy_hi, (bf*)dy_lo,
                                                                                  dy_f32);
  return launch_status("sfb_tokens_split_grad");
}

// ring kernels of x3d_ops.cu (shared-memory frame ring, every input byte crosses HBM once) for the stride-1 3x3x3 pools
namespace sfb {
int dw3_run_strided(int mode, const float* x, int64_t x_pitch, int64_t x_so, int64_t x_si, const float* in_shift, int64_t aff_si,
                    const float* w, int flip, float* y, int64_t y_pitch, int64_t y_so, int64_t y_si, int y_accumulate,
                    const float* dy, int64_t dy_pitch, int64_t dy_so, int64_t dy_si, float* dw, int n_outer, int n_inner,
                    int T, int H, int W, int C, cudaStream_t st);
}
static bool dwpool_ring_ok(const sfb_dwpool_desc* d) {
  return !d->no_cls && d->has_pool && d->kt == 3 && d->kh == 3 && d->kw == 3 && d->st == 1 && d->sh == 1 && d->sw == 1 &&
         d->t >= 2 && d->h % 7 == 0 && d->w_ % 7 == 0 && d->ot == d->t && d->oh == d->h && d->ow == d->w_ && d->hd % 4 == 0 &&
         d->src_pitch % 4 == 0 && d->src_c0 % 4 == 0;
}
// cls rows of the pooled tensors pass through the pooling: out[b,h,0,:] = src[b,0,ch] + bias ; dsrc[b,0,ch] += dout[b,h,0,:]
__global__ void dwpool_cls_kernel(const DwPoolParams p, int backward) {
  const int L = p.T * p.Hh * p.W, Lo = p.oT * p.oH * p.oW;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.B * p.H * p.hd) return;
  const int c = i % p.hd, h = (i / p.hd) % p.H, b = i / (p.hd * p.H);
  const int ch = p.src_c0 + h * p.hd + c;
  const int64_t so = int64_t(b) * (L + 1) * p.src_pitch + ch, oo = (int64_t(b) * p.H + h) * (Lo + 1) * p.hd + c;
  if (backward) p.dsrc[so] += p.dout[oo];
  else p.out[oo] = p.src[so] + (p.bias ? p.bias[ch] : 0.f);
}

static void fill_dw(DwPoolParams& p, const sfb_dwpool_desc* d) {
  memset(&p, 0, sizeof(p));
  p.src = d->src; p.src_pitch = d->src_pitch; p.src_c0 = d->src_c0; p.bias = d->bias; p.w = d->w; p.out = d->out;
  p.B = d->b; p.H = d->heads; p.hd = d->hd; p.T = d->t; p.Hh = d->h; p.W = d->w_; p.oT = d->ot; p.oH = d->oh; p.oW = d->ow;
  p.kt = d->kt; p.kh = d->kh; p.kw = d->kw; p.st = d->st; p.sh = d->sh; p.sw = d->sw; p.pt = d->kt / 2; p.ph = d->kh / 2;
  p.pw = d->kw / 2;
  p.dout = d->dout; p.dsrc = d->dsrc; p.wpartials = d->wpartials; p.has_pool = d->has_pool;
}
extern "C" int sfb_dwpool_fwd(const sfb_dwpool_desc* d, void* stream) {
  if (d->has_pool && d->kt * d->kh * d->kw > 27) {
    set_error("sfb_dwpool_fwd: pooling kernels larger than 27 taps are not supported");
    return -10;
  }
  DwPoolParams p;
  fill_dw(p, d);
  if (d->hd % 4 || d->src_pitch % 4 || d->src_c0 % 4) {
    set_error("sfb_dwpool_fwd: head_dim / pitch / channel offset must be multiples of 4");
    return -10;
  }
  if (dwpool_ring_ok(d)) {
    const int64_t L = int64_t(d->t) * d->h * d->w_;
    const int rc = dw3_run_strided(0, d->src + d->src_pitch + d->src_c0, d->src_pitch, (L + 1) * d->src_pitch, d->hd,
                                   d->bias ? d->bias + d->src_c0 : nullptr, d->hd, d->w, 0, d->out + d->hd, d->hd,
                                   int64_t(d->heads) * (L + 1) * d->hd, (L + 1) * d->hd, 0, nullptr, 0, 0, 0, nullptr, d->b,
                                   d->heads, d->t, d->h, d->w_, d->hd, (cudaStream_t)stream);
    if (rc != -100) {
      if (rc) return rc;
      const int n = d->b * d->heads * d->hd;
      dwpool_cls_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p, 0);
      return launch_status("sfb_dwpool_fwd(cls)");
    }
  }
  const int64_t items = int64_t(d->b) * d->heads * (int64_t(d->ot) * d->oh * d->ow + (d->no_cls ? 0 : 1)) * (d->hd / 4);
  if (d->no_cls)
    dwpool_fwd_kernel<0><<<mv_grid(items, 256, 16), 256, 0, (cudaStream_t)stream>>>(p);
  else
    dwpool_fwd_kernel<1><<<mv_grid(items, 256, 16), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_dwpool_fwd");
}
extern "C" int32_t sfb_dwpool_wgrad_blocks(const sfb_dwpool_desc* d) {
  int64_t total = int64_t(d->b) * d->heads * d->ot * d->oh * d->ow;
  int64_t nb = (total + 15) / 16;
  if (nb > kGridSms * 4) nb = kGridSms * 4;
  return int32_t(nb < 1 ? 1 : nb);
}
__global__ void dwpool_wmerge_kernel(const float* __restrict__ partials, int nblocks, int n, float* __restrict__ out,
                                     int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int b = 0; b < nblocks; ++b) s += double(partials[size_t(b) * n + i]);
  out[i] = accumulate ? out[i] + float(s) : float(s);
}
extern "C" int sfb_dwpool_bwd(const sfb_dwpool_desc* d, float* dw, int32_t dw_accumulate, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DwPoolParams p;
  fill_dw(p, d);
  if (dwpool_ring_ok(d)) {
    const int64_t L = int64_t(d->t) * d->h * d->w_;
    const int64_t o_so = int64_t(d->heads) * (L + 1) * d->hd, o_si = (L + 1) * d->hd;
    // data gradient: dsrc[token rows of this third] += conv(dout, mirrored filter)
    int rc = dw3_run_strided(0, d->dout + d->hd, d->hd, o_so, o_si, nullptr, 0, d->w, 1, d->dsrc + d->src_pitch + d->src_c0,
                             d->src_pitch, (L + 1) * d->src_pitch, d->hd, 1, nullptr, 0, 0, 0, nullptr, d->b, d->heads, d->t,
                             d->h, d->w_, d->hd, stream);
    if (rc != -100) {
      if (rc) return rc;
      const int n = d->b * d->heads * d->hd;
      dwpool_cls_kernel<<<(n + 255) / 256, 256, 0, stream>>>(p, 1);
      if (int rc = launch_status("sfb_dwpool_bwd(cls)")) return rc;
      if (dw) {
        if (!dw_accumulate) cudaMemsetAsync(dw, 0, size_t(d->hd) * 27 * sizeof(float), stream);
        rc = dw3_run_strided(1, d->src + d->src_pitch + d->src_c0, d->src_pitch, (L + 1) * d->src_pitch, d->hd,
                             d->bias ? d->bias + d->src_c0 : nullptr, d->hd, nullptr, 0, nullptr, 0, 0, 0, 0, d->dout + d->hd,
                             d->hd, o_so, o_si, dw, d->b, d->heads, d->t, d->h, d->w_, d->hd, stream);
        if (rc) return rc;
      }
      return 0;
    }
  }
  const int cls = d->no_cls ? 0 : 1;
  if (d->has_pool && d->sh >= d->kh && d->sw >= d->kw) {
    const int64_t items = int64_t(d->b) * d->heads * (int64_t(d->ot) * d->oh * d->ow + cls) * (d->hd / 4);
    if (cls)
      dwpool_bwd_data_scatter_kernel<1><<<mv_grid(items, 256, 16), 256, 0, stream>>>(p);
    else
      dwpool_bwd_data_scatter_kernel<0><<<mv_grid(items, 256, 16), 256, 0, stream>>>(p);
  } else {
    const int64_t items = int64_t(d->b) * d->heads * (int64_t(d->t) * d->h * d->w_ + cls) * (d->hd / 4);
    if (cls)
      dwpool_bwd_data_kernel<1><<<mv_grid(items, 256, 16), 256, 0, stream>>>(p);
    else
      dwpool_bwd_data_kernel<0><<<mv_grid(items, 256, 16), 256, 0, stream>>>(p);
  }
  if (int rc = launch_status("sfb_dwpool_bwd(data)")) return rc;
  if (d->has_pool && dw) {
    const int nb = sfb_dwpool_wgrad_blocks(d);
    if (d->hd > 256 || d->kt > 3 || d->kh > 3 || d->kw > 3) {
      set_error("sfb_dwpool_bwd: head_dim <= 256 and pooling kernels <= 3x3x3 are supported");
      return -10;
    }
    const int pl = std::max(1, std::min(4, 512 / d->hd));   // position lanes per block (<= 41 KB of shared memory at hd = 96)
    const int n = d->hd * d->kt * d->kh * d->kw;
    if (!dw_accumulate) cudaMemsetAsync(dw, 0, size_t(n) * sizeof(float), stream);
    p.dw = dw;
    if (cls)
      dwpool_bwd_weight_kernel<1><<<nb, pl * d->hd, size_t(pl) * d->hd * 27 * sizeof(float), stream>>>(p);
    else
      dwpool_bwd_weight_kernel<0><<<nb, pl * d->hd, size_t(pl) * d->hd * 27 * sizeof(float), stream>>>(p);
    if (int rc = launch_status("sfb_dwpool_bwd(weight)")) return rc;
  }
  return 0;
}

static void fill_sm(SoftmaxParams& p, const sfb_softmax_desc* d) {
  memset(&p, 0, sizeof(p));
  p.S = d->s; p.s_pitch = d->s_pitch; p.RQ = d->rq; p.rq_pitch = d->rq_pitch;
  p.p_hi = (bf*)d->p_hi; p.p_lo = (bf*)d->p_lo; p.p_pitch = d->p_pitch;
  p.BH = d->bh; p.Nq = d->nq; p.Nk = d->nk;
  p.qt = d->qt; p.qh = d->qh; p.qw = d->qw; p.kt = d->kt; p.kh = d->kh; p.kw = d->kw;
  p.Lh = 2 * (d->qh > d->kh ? d->qh : d->kh) - 1;
  p.Lw = 2 * (d->qw > d->kw ? d->qw : d->kw) - 1;
  p.Lt = d->spatial_only ? 0 : 2 * (d->qt > d->kt ? d->qt : d->kt) - 1;
  auto ratio = [](int a, int b) { float r = float(a) / float(b); return r > 1.f ? r : 1.f; };
  p.rh_q = ratio(d->kh, d->qh); p.rh_k = ratio(d->qh, d->kh);
  p.rw_q = ratio(d->kw, d->qw); p.rw_k = ratio(d->qw, d->kw);
  p.rt_q = ratio(d->kt, d->qt); p.rt_k = ratio(d->qt, d->kt);
  p.dP = d->dp; p.dp_pitch = d->dp_pitch;
  p.ds_hi = (bf*)d->ds_hi; p.ds_lo = (bf*)d->ds_lo; p.ds_pitch = d->ds_pitch; p.dRQ = d->drq;
}
template <bool kBwd, int kCls, bool kRelT>
static void softmax_launch(const SoftmaxParams& p, int64_t rows, size_t smem, cudaStream_t stream) {
  auto kernel = kBwd ? softmax_relpos_bwd_kernel<kCls, kRelT> : softmax_relpos_fwd_kernel<kCls, kRelT>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kSoftmaxSmemMax));
    attr_set = true;
  }
  kernel<<<mv_grid(rows * 32, 256, 16), 256, smem, stream>>>(p);
}
template <bool kBwd>
static void softmax_dispatch(const sfb_softmax_desc* d, const SoftmaxParams& p, int64_t rows, size_t smem,
                             cudaStream_t stream) {
  if (!d->no_cls && !d->spatial_only) softmax_launch<kBwd, 1, true>(p, rows, smem, stream);
  else if (!d->no_cls) softmax_launch<kBwd, 1, false>(p, rows, smem, stream);
  else if (!d->spatial_only) softmax_launch<kBwd, 0, true>(p, rows, smem, stream);
  else softmax_launch<kBwd, 0, false>(p, rows, smem, stream);
}
extern "C" int sfb_softmax_relpos_fwd(const sfb_softmax_desc* d, void* stream) {
  SoftmaxParams p;
  fill_sm(p, d);
  const int64_t rows = int64_t(d->bh) * d->nq;
  const size_t smem = size_t(8) * d->nk * sizeof(float);
  if (smem > kSoftmaxSmemMax) {
    set_error("sfb_softmax_relpos_fwd: %d keys exceed the shared-memory row buffer", d->nk);
    return -10;
  }
  softmax_dispatch<false>(d, p, rows, smem, (cudaStream_t)stream);
  return launch_status("sfb_softmax_relpos_fwd");
}
extern "C" int sfb_softmax_relpos_bwd(const sfb_softmax_desc* d, void* stream) {
  SoftmaxParams p;
  fill_sm(p, d);
  const int64_t rows = int64_t(d->bh) * d->nq;
  const size_t smem = size_t(8) * (p.Nk + p.Lh + p.Lw + p.Lt) * sizeof(float);
  if (smem > kSoftmaxSmemMax) {
    set_error("sfb_softmax_relpos_bwd: %d keys exceed the shared-memory row buffer", d->nk);
    return -10;
  }
  softmax_dispatch<true>(d, p, rows, smem, (cudaStream_t)stream);
  return launch_status("sfb_softmax_relpos_bwd");
}
extern "C" int sfb_attn_merge(const float* o, const void* q_hi, const void* q_lo, int32_t b, int32_t h, int32_t n,
                              int32_t hd, int32_t residual, void* m_hi, void* m_lo, void* stream) {
  const int64_t items = int64_t(b) * n * h * hd;
  attn_merge_kernel<1><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(o, (const bf*)q_hi, (const bf*)q_lo, b, h, n,
                                                                             hd, residual, (bf*)m_hi, (bf*)m_lo);
  return launch_status("sfb_attn_merge");
}
extern "C" int sfb_attn_merge_nocls(const float* o, const void* q_hi, const void* q_lo, int32_t b, int32_t h, int32_t n,
                                    int32_t hd, int32_t residual, void* m_hi, void* m_lo, void* stream) {
  const int64_t items = int64_t(b) * n * h * hd;
  attn_merge_kernel<0><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(o, (const bf*)q_hi, (const bf*)q_lo, b, h, n,
                                                                             hd, residual, (bf*)m_hi, (bf*)m_lo);
  return launch_status("sfb_attn_merge_nocls");
}
extern "C" int sfb_attn_split_grad(const float* dm, int32_t b, int32_t h, int32_t n, int32_t hd, int32_t residual,
                                   void* do_hi, void* do_lo, float* dq, void* stream) {
  const int64_t items = int64_t(b) * h * n * hd;
  attn_split_grad_kernel<1><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dm, b, h, n, hd, residual,
                                                                                   (bf*)do_hi, (bf*)do_lo, dq);
  return launch_status("sfb_attn_split_grad");
}
extern "C" int sfb_attn_split_grad_nocls(const float* dm, int32_t b, int32_t h, int32_t n, int32_t hd, int32_t residual,
                                         void* do_hi, void* do_lo, float* dq, void* stream) {
  const int64_t items = int64_t(b) * h * n * hd;
  attn_split_grad_kernel<0><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dm, b, h, n, hd, residual,
                                                                                   (bf*)do_hi, (bf*)do_lo, dq);
  return launch_status("sfb_attn_split_grad_nocls");
}
extern "C" int sfb_residual_add(const float* a, const float* a_bias, const float* y, const float* y_bias,
                                const float* scale, int64_t rows, int32_t c, int64_t rows_per_sample, float* out,
                                void* stream) {
  residual_add_kernel<<<mv_grid(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(a, a_bias, y, y_bias, scale, rows, c,
                                                                                rows_per_sample, out);
  return launch_status("sfb_residual_add");
}
extern "C" int sfb_bias_gelu(const float* y, const float* bias, int64_t rows, int32_t c, void* hi, void* lo,
                             void* stream) {
  bias_gelu_kernel<<<mv_grid(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(y, bias, rows, c, (bf*)hi, (bf*)lo);
  return launch_status("sfb_bias_gelu");
}
extern "C" int sfb_bias_gelu_bwd(const float* dh, const float* y, const float* bias, int64_t rows, int32_t c, void* hi,
                                 void* lo, float* dpre, void* stream) {
  bias_gelu_bwd_kernel<<<mv_grid(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(dh, y, bias, rows, c, (bf*)hi, (bf*)lo,
                                                                                 dpre);
  return launch_status("sfb_bias_gelu_bwd");
}
extern "C" int sfb_scale_split(const float* src, const float* scale, int64_t rows, int32_t c, int64_t rows_per_sample,
                               void* hi, void* lo, float* f32, void* stream) {
  scale_split_kernel<<<mv_grid(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(src, scale, rows, c, rows_per_sample,
                                                                               (bf*)hi, (bf*)lo, f32);
  return launch_status("sfb_scale_split");
}
static void fill_tp(TokPoolParams& p, const sfb_tokpool_desc* d) {
  memset(&p, 0, sizeof(p));
  p.x = d->x; p.out = d->out; p.argmax = d->argmax;
  p.B = d->b; p.C = d->c; p.T = d->t; p.Hh = d->h; p.W = d->w; p.oT = d->ot; p.oH = d->oh; p.oW = d->ow;
  p.kt = d->kt; p.kh = d->kh; p.kw = d->kw; p.st = d->st; p.sh = d->sh; p.sw = d->sw;
  p.pt = d->kt / 2; p.ph = d->kh / 2; p.pw = d->kw / 2;
  p.dout = d->dout; p.dx = d->dx; p.dx_accumulate = d->dx_accumulate;
}
extern "C" int sfb_token_maxpool_fwd(const sfb_tokpool_desc* d, void* stream) {
  TokPoolParams p;
  fill_tp(p, d);
  const int64_t items = int64_t(d->b) * (int64_t(d->ot) * d->oh * d->ow + (d->no_cls ? 0 : 1)) * d->c;
  if (d->no_cls)
    token_maxpool_fwd_kernel<0><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  else
    token_maxpool_fwd_kernel<1><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_token_maxpool_fwd");
}
extern "C" int sfb_token_maxpool_bwd(const sfb_tokpool_desc* d, void* stream) {
  TokPoolParams p;
  fill_tp(p, d);
  const int64_t items = int64_t(d->b) * (int64_t(d->t) * d->h * d->w + (d->no_cls ? 0 : 1)) * d->c;
  if (d->no_cls)
    token_maxpool_bwd_kernel<0><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  else
    token_maxpool_bwd_kernel<1><<<mv_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_token_maxpool_bwd");
}
