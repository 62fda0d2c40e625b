// MaskFeat wrapper kernels (SURVEY.md section 8 row a19; slowfast/models/masked.py):
//   * mask-token substitution on the patch-embedding output and its backward   (masked.py:551-561)
//   * nearest-neighbour upsampling of the loader's cube mask to the token grid (masked.py:556-559, F.interpolate)
//   * HOG targets: Sobel gradients with reflect padding, 9 unsigned-orientation bins weighted by magnitude, 8x8 cell
//     sums, L2 normalisation over the bins, regrouped to one 108-vector per output token
//     (operators.py:79-122 HOGLayerC.forward, masked.py:254-281 _get_hog_label_3d)
//   * the prediction head's row bookkeeping (drop the cls row, add the Linear bias; pad 108 -> 112 columns for the
//     tensor-core gradient kernels)                                             (head_helper.py:656-672)
#include <cstdint>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "planes.cuh"
#include "runtime.h"

namespace sfb {

using bf = __nv_bfloat16;

static int mf_grid(int64_t items, int block) { return capped_grid(items, block, int64_t(kGridSms) * 8); }

__global__ void mask_upsample_kernel(const float* __restrict__ mask, int b, int mt, int mh, int mw, int t, int h, int w,
                                     float* __restrict__ out) {
  const int64_t items = int64_t(b) * t * h * w;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int x = int(i % w);
    int64_t r = i / w;
    const int y = int(r % h);
    r /= h;
    const int z = int(r % t);
    const int64_t bb = r / t;
    // torch 'nearest': src = floor(dst * in / out) (exact in integers for these sizes)
    const int sx = min(int((int64_t(x) * mw) / w), mw - 1), sy = min(int((int64_t(y) * mh) / h), mh - 1),
              sz = min(int((int64_t(z) * mt) / t), mt - 1);
    out[i] = mask[((bb * mt + sz) * mh + sy) * mw + sx];
  }
}

__global__ void tokens_assemble_masked_kernel(const float* __restrict__ y, const float* __restrict__ bias,
                                              const float* __restrict__ cls, const float* __restrict__ mtok,
                                              const float* __restrict__ m, int b, int l, int c, float* __restrict__ x) {
  const int64_t items = int64_t(b) * (l + 1) * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % (l + 1));
    const int64_t bb = t / (l + 1);
    if (n == 0) {
      x[i] = cls[ch];
    } else {
      const float mm = m[bb * l + n - 1];
      x[i] = (y[(bb * l + n - 1) * c + ch] + bias[ch]) * (1.f - mm) + mtok[ch] * mm;
    }
  }
}
__global__ void tokens_split_grad_masked_kernel(const float* __restrict__ dx, const float* __restrict__ m, int b, int l,
                                                int c, bf* dy_hi, bf* dy_lo, float* __restrict__ dy_f32,
                                                float* __restrict__ dxm) {
  const int64_t items = int64_t(b) * l * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % l);
    const int64_t bb = t / l;
    const float g = dx[(bb * (l + 1) + n + 1) * c + ch];
    const float mm = m[bb * l + n];
    const float v = g * (1.f - mm);
    put_split(dy_hi, dy_lo, i, v);
    dy_f32[i] = v;
    dxm[i] = g * mm;
  }
}

__global__ void rows_unpad_bias_kernel(const float* __restrict__ y, int64_t ldy, const float* __restrict__ bias, int b,
                                       int l, int c, float* __restrict__ out) {
  const int64_t items = int64_t(b) * l * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t t = i / c;
    const int n = int(t % l);
    const int64_t bb = t / l;
    out[i] = y[(bb * (l + 1) + 1 + n) * ldy + ch] + bias[ch];
  }
}
__global__ void rows_pad_split_kernel(const float* __restrict__ d, int b, int l, int c, int cp, bf* hi, bf* lo) {
  const int64_t items = int64_t(b) * (l + 1) * cp;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % cp);
    const int64_t t = i / cp;
    const int n = int(t % (l + 1));
    const int64_t bb = t / (l + 1);
    const float v = (n > 0 && ch < c) ? d[(bb * l + n - 1) * c + ch] : 0.f;
    put_split(hi, lo, i, v);
  }
}

// one thread = one (frame, colour channel, cell): 9 register bins over cell x cell pixels
constexpr int HOG_MAX_BINS = 9;
__global__ void hog_targets_kernel(const float* __restrict__ x, int b, int ch, int t, int h, int w, int t_stride,
                                   int nbins, int cell, int fs, float* __restrict__ out) {
  const int tp = t / t_stride;  // frames that carry a label
  const int cy_n = h / cell, cx_n = w / cell;
  const int u = cy_n / fs;      // cells per output token along each axis (unfold size)
  const int feat = ch * nbins * u * u;
  const int64_t items = int64_t(b) * tp * ch * cy_n * cx_n;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int cx = int(i % cx_n);
    int64_t r = i / cx_n;
    const int cy = int(r % cy_n);
    r /= cy_n;
    const int c = int(r % ch);
    r /= ch;
    const int f = int(r % tp);
    const int64_t bb = r / tp;
    const float* img = x + ((bb * ch + c) * t + int64_t(f) * t_stride) * h * w;
    float bins[HOG_MAX_BINS];
#pragma unroll
    for (int k = 0; k < HOG_MAX_BINS; ++k) bins[k] = 0.f;
    for (int py = 0; py < cell; ++py) {
      const int yy = cy * cell + py;
      const int ym = yy == 0 ? 1 : yy - 1, yp = yy == h - 1 ? h - 2 : yy + 1;  // reflect padding of width 1
      for (int px = 0; px < cell; ++px) {
        const int xx = cx * cell + px;
        const int xm = xx == 0 ? 1 : xx - 1, xp = xx == w - 1 ? w - 2 : xx + 1;
        const float a00 = img[ym * w + xm], a01 = img[ym * w + xx], a02 = img[ym * w + xp];
        const float a10 = img[yy * w + xm], a12 = img[yy * w + xp];
        const float a20 = img[yp * w + xm], a21 = img[yp * w + xx], a22 = img[yp * w + xp];
        // cross-correlation with [[1,0,-1],[2,0,-2],[1,0,-1]] and its transpose (operators.py:85-87)
        const float gx = (a00 - a02) + 2.f * (a10 - a12) + (a20 - a22);
        const float gy = (a00 + 2.f * a01 + a02) - (a20 + 2.f * a21 + a22);
        const float mag = sqrtf(gx * gx + gy * gy);
        const float phase = atan2f(gx, gy) / 3.14159265358979323846f * float(nbins);
        int k = int(floorf(phase)) % nbins;
        if (k < 0) k += nbins;
#pragma unroll
        for (int q = 0; q < HOG_MAX_BINS; ++q)
          if (q == k) bins[q] += mag;
      }
    }
    float nrm = 0.f;
#pragma unroll
    for (int k = 0; k < HOG_MAX_BINS; ++k)
      if (k < nbins) nrm = fmaf(bins[k], bins[k], nrm);
    const float inv = 1.f / fmaxf(sqrtf(nrm), 1e-12f);  // F.normalize(p=2, dim=bins, eps=1e-12)
    const int ty = cy / u, wy = cy - ty * u, tx = cx / u, wx = cx - tx * u;
    float* o = out + (((bb * tp + f) * fs + ty) * fs + tx) * int64_t(feat);
#pragma unroll
    for (int k = 0; k < HOG_MAX_BINS; ++k)
      if (k < nbins) o[((c * nbins + k) * u + wy) * u + wx] = bins[k] * inv;
  }
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_mask_upsample(const float* mask, int32_t b, int32_t mt, int32_t mh, int32_t mw, int32_t t, int32_t h,
                                 int32_t w, float* out, void* stream) {
  mask_upsample_kernel<<<mf_grid(int64_t(b) * t * h * w, 256), 256, 0, (cudaStream_t)stream>>>(mask, b, mt, mh, mw, t,
                                                                                              h, w, out);
  return launch_status("sfb_mask_upsample");
}
extern "C" int sfb_tokens_assemble_masked(const float* y, const float* bias, const float* cls, const float* mask_token,
                                          const float* tokmask, int32_t b, int32_t l, int32_t c, float* x,
                                          void* stream) {
  tokens_assemble_masked_kernel<<<mf_grid(int64_t(b) * (l + 1) * c, 256), 256, 0, (cudaStream_t)stream>>>(
      y, bias, cls, mask_token, tokmask, b, l, c, x);
  return launch_status("sfb_tokens_assemble_masked");
}
extern "C" int sfb_tokens_split_grad_masked(const float* dx, const float* tokmask, int32_t b, int32_t l, int32_t c,
                                            void* dy_hi, void* dy_lo, float* dy_f32, float* dxm, void* stream) {
  tokens_split_grad_masked_kernel<<<mf_grid(int64_t(b) * l * c, 256), 256, 0, (cudaStream_t)stream>>>(
      dx, tokmask, b, l, c, (bf*)dy_hi, (bf*)dy_lo, dy_f32, dxm);
  return launch_status("sfb_tokens_split_grad_masked");
}
extern "C" int sfb_rows_unpad_bias(const float* y, int64_t ldy, const float* bias, int32_t b, int32_t l, int32_t c,
                                   float* out, void* stream) {
  rows_unpad_bias_kernel<<<mf_grid(int64_t(b) * l * c, 256), 256, 0, (cudaStream_t)stream>>>(y, ldy, bias, b, l, c, out);
  return launch_status("sfb_rows_unpad_bias");
}
extern "C" int sfb_rows_pad_split(const float* d, int32_t b, int32_t l, int32_t c, int32_t cp, void* hi, void* lo,
                                  void* stream) {
  rows_pad_split_kernel<<<mf_grid(int64_t(b) * (l + 1) * cp, 256), 256, 0, (cudaStream_t)stream>>>(d, b, l, c, cp,
                                                                                                  (bf*)hi, (bf*)lo);
  return launch_status("sfb_rows_pad_split");
}
extern "C" int sfb_hog_targets(const float* x, int32_t b, int32_t ch, int32_t t, int32_t h, int32_t w, int32_t t_stride,
                               int32_t nbins, int32_t cell, int32_t fs, float* out, void* stream) {
  if (nbins > HOG_MAX_BINS || nbins < 1 || h % cell || w % cell || h != w || (h / cell) % fs || t % t_stride || h < 2) {
    set_error("sfb_hog_targets: unsupported geometry (nbins=%d cell=%d h=%d w=%d fs=%d)", nbins, cell, h, w, fs);
    return -10;
  }
  const int64_t items = int64_t(b) * (t / t_stride) * ch * (h / cell) * (w / cell);
  hog_targets_kernel<<<mf_grid(items, 128), 128, 0, (cudaStream_t)stream>>>(x, b, ch, t, h, w, t_stride, nbins, cell, fs,
                                                                           out);
  return launch_status("sfb_hog_targets");
}
