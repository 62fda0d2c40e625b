// Classification-head pieces (head_helper.py:305-350 ResNetBasicHead / :547-563 TransformerBasicHead):
// global average pool over (T,H,W), dropout, the small Linear (M = batch rows) and the eval-mode softmax / sigmoid.
// These are tiny next to the backbone (a few MFLOP); they are plain SIMT kernels so that the whole model path
// stays inside this library and on the caller's stream.
#include <algorithm>
#include <cstdint>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "runtime.h"

namespace sfb {

// out[n, c] = mean_{s < spatial} (hi + lo)[n, s, c]; one block per (n, 32-channel strip), 8 row-lanes
__global__ void __launch_bounds__(256) global_avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ hi,
                                                                 const __nv_bfloat16* __restrict__ lo, int64_t pitch,
                                                                 int spatial, int c, float* __restrict__ out,
                                                                 int64_t out_pitch) {
  __shared__ float sm[8][32];
  const int n = blockIdx.y;
  const int ch = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  float acc = 0.f;
  if (ch < c) {
    const int64_t base = int64_t(n) * spatial * pitch + ch;
    for (int s = rl; s < spatial; s += 8) {
      float v = __bfloat162float(hi[base + s * pitch]);
      if (lo) v += __bfloat162float(lo[base + s * pitch]);
      acc += v;
    }
  }
  sm[rl][threadIdx.x & 31] = acc;
  __syncthreads();
  if (rl == 0 && ch < c) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += sm[k][threadIdx.x];
    out[int64_t(n) * out_pitch + ch] = s / float(spatial);
  }
}

// dx[n, s, c] = dpooled[n, c] / spatial  (fp32 gradient w.r.t. the pooled activation)
__global__ void global_avgpool_bwd_kernel(const float* __restrict__ dpooled, int64_t dp_pitch, int spatial, int c,
                                          int n, float* __restrict__ dx, int64_t dx_pitch) {
  const int64_t items = int64_t(n) * spatial * c;
  const float inv = 1.f / float(spatial);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    const int64_t r = i / c;
    const int64_t b = r / spatial;
    dx[r * dx_pitch + ch] = dpooled[b * dp_pitch + ch] * inv;
  }
}

// Fully-convolutional inference of ResNetBasicHead (head_helper.py:305-350): AvgPool3d(pool_size, stride=1) over a
// feature map larger than the train-time pool (TEST_CROP_SIZE 256 -> 8x8 map, 7x7 pool -> 2x2 windows).
// out[((n*ot+z)*oh+p)*ow+q, c] = mean over the kt x kh x kw window of (hi+lo); one thread per (window, channel).
__global__ void window_avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                                          int64_t pitch, int n, int t, int h, int w, int c, int kt, int kh, int kw,
                                          float* __restrict__ out, int64_t out_pitch) {
  const int ot = t - kt + 1, oh = h - kh + 1, ow = w - kw + 1;
  const int64_t items = int64_t(n) * ot * oh * ow * c;
  const float inv = 1.f / float(kt * kh * kw);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ch = int(i % c);
    int64_t r = i / c;
    const int q = int(r % ow); r /= ow;
    const int pp = int(r % oh); r /= oh;
    const int z = int(r % ot);
    const int b = int(r / ot);
    float acc = 0.f;
    for (int a = 0; a < kt; ++a)
      for (int y = 0; y < kh; ++y)
        for (int x = 0; x < kw; ++x) {
          const int64_t o = (((int64_t(b) * t + z + a) * h + pp + y) * w + q + x) * pitch + ch;
          float v = __bfloat162float(hi[o]);
          if (lo) v += __bfloat162float(lo[o]);
          acc += v;
        }
    out[(i / c) * out_pitch + ch] = acc * inv;
  }
}

// out[n, k] = mean over g consecutive rows of in[n*g + j, k]  (x_proj.mean([1,2,3]), head_helper.py:343)
__global__ void rows_group_mean_kernel(const float* __restrict__ in, float* __restrict__ out, int n, int g, int k) {
  const int64_t items = int64_t(n) * k;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int col = int(i % k);
    const int64_t b = i / k;
    float acc = 0.f;
    for (int j = 0; j < g; ++j) acc += in[(b * g + j) * k + col];
    out[i] = acc / float(g);
  }
}

__device__ __forceinline__ uint32_t mix32(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return uint32_t((z ^ (z >> 31)) >> 32);
}
// x *= keep/(1-p) with keep ~ Bernoulli(1-p) from a counter-based generator keyed by (seed, element index);
// the keep mask is saved (uint8) for backward.
__global__ void dropout_fwd_kernel(float* __restrict__ x, uint8_t* __restrict__ mask, int64_t nelem, float p,
                                   uint64_t seed, const uint64_t* __restrict__ step) {
  const float scale = 1.f / (1.f - p);
  if (step) seed = seed * 0x9E3779B97F4A7C15ull + *step;  // device-side step counter: CUDA-graph replays differ
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nelem; i += int64_t(gridDim.x) * blockDim.x) {
    const float u = float(mix32(seed * 0x100000001B3ull + uint64_t(i)) >> 8) * (1.f / 16777216.f);
    const uint8_t keep = u >= p ? 1 : 0;
    mask[i] = keep;
    x[i] = keep ? x[i] * scale : 0.f;
  }
}
__global__ void counter_inc_kernel(uint64_t* c) { *c += 1; }
__global__ void dropout_bwd_kernel(float* __restrict__ dx, const uint8_t* __restrict__ mask, int64_t nelem, float p) {
  const float scale = 1.f / (1.f - p);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nelem; i += int64_t(gridDim.x) * blockDim.x)
    dx[i] = mask[i] ? dx[i] * scale : 0.f;
}

// y[m, k] = sum_j x[m, j] * w[k, j] + b[k]     one warp per output, fp32 (fma order: lane-strided then butterfly)
// RELU: y = relu(...) (the hidden layers of MLPHead, head_helper.py:147-196)
template <bool RELU>
__global__ void small_linear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                        const float* __restrict__ b, float* __restrict__ y, int m, int k, int j) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= m * k) return;
  const int mi = warp / k, ki = warp - mi * k;
  const float* xr = x + int64_t(mi) * j;
  const float* wr = w + int64_t(ki) * j;
  float acc = 0.f;
  for (int t = lane; t < j; t += 32) acc = fmaf(xr[t], wr[t], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    const float v = acc + (b ? b[ki] : 0.f);
    y[warp] = RELU ? (v < 0.f ? 0.f : v) : v;
  }
}
// dw[k, j] (+)= sum_m dy[m, k] x[m, j];  db[k] (+)= sum_m dy[m, k]
__global__ void small_linear_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                          float* __restrict__ dw, float* __restrict__ db, int m, int k, int j,
                                          int accumulate) {
  const int64_t items = int64_t(k) * j;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ji = int(i % j);
    const int ki = int(i / j);
    float acc = 0.f;
    for (int mi = 0; mi < m; ++mi) acc = fmaf(dy[int64_t(mi) * k + ki], x[int64_t(mi) * j + ji], acc);
    dw[i] = accumulate ? dw[i] + acc : acc;
    if (ji == 0 && db) {
      float s = 0.f;
      for (int mi = 0; mi < m; ++mi) s += dy[int64_t(mi) * k + ki];
      db[ki] = accumulate ? db[ki] + s : s;
    }
  }
}
// dx[m, j] = sum_k dy[m, k] w[k, j]
// RELU_MASK: dx[m, j] = 0 where x[m, j] <= 0 - x is the output of the ReLU in front of this layer, so this is
// torch's threshold_backward(dx, x, 0) fused into the data gradient
template <bool RELU_MASK>
__global__ void small_linear_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w,
                                          float* __restrict__ dx, int m, int k, int j, const float* __restrict__ x) {
  const int64_t items = int64_t(m) * j;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int ji = int(i % j);
    const int mi = int(i / j);
    float acc = 0.f;
    for (int ki = 0; ki < k; ++ki) acc = fmaf(dy[int64_t(mi) * k + ki], w[int64_t(ki) * j + ji], acc);
    dx[i] = RELU_MASK ? (x[i] > 0.f ? acc : 0.f) : acc;
  }
}
// row softmax in place (eval-mode head activation), one warp per row
__global__ void row_softmax_kernel(float* __restrict__ x, int rows, int cols) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  float* r = x + int64_t(warp) * cols;
  float mx = -INFINITY;
  for (int t = lane; t < cols; t += 32) mx = fmaxf(mx, r[t]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float s = 0.f;
  for (int t = lane; t < cols; t += 32) s += expf(r[t] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float inv = 1.f / s;
  for (int t = lane; t < cols; t += 32) r[t] = expf(r[t] - mx) * inv;
}
// elementwise logistic sigmoid in place (eval-mode multi-label head activation); exp of -|x| only, so no overflow
// for large |x|: 1 / (1 + e^-x) for x >= 0, e^x / (1 + e^x) below
__global__ void row_sigmoid_kernel(float* __restrict__ x, int64_t nelem) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nelem; i += int64_t(gridDim.x) * blockDim.x) {
    const float v = x[i];
    const float e = expf(-fabsf(v));
    x[i] = v >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
  }
}

static int hd_grid(int64_t items, int block) { return capped_grid(items, block, int64_t(kGridSms) * 8); }

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_global_avgpool_fwd(const void* hi, const void* lo, int64_t pitch, int32_t n, int32_t spatial,
                                      int32_t c, float* out, int64_t out_pitch, void* stream) {
  dim3 grid((c + 31) / 32, n);
  global_avgpool_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)hi, (const __nv_bfloat16*)lo,
                                                                   pitch, spatial, c, out, out_pitch);
  return launch_status("sfb_global_avgpool_fwd");
}
extern "C" int sfb_global_avgpool_bwd(const float* dpooled, int64_t dp_pitch, int32_t n, int32_t spatial, int32_t c,
                                      float* dx, int64_t dx_pitch, void* stream) {
  const int64_t items = int64_t(n) * spatial * c;
  global_avgpool_bwd_kernel<<<hd_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(dpooled, dp_pitch, spatial, c, n, dx,
                                                                                  dx_pitch);
  return launch_status("sfb_global_avgpool_bwd");
}
extern "C" int sfb_window_avgpool_fwd(const void* hi, const void* lo, int64_t pitch, int32_t n, int32_t t, int32_t h,
                                      int32_t w, int32_t c, int32_t kt, int32_t kh, int32_t kw, float* out,
                                      int64_t out_pitch, void* stream) {
  if (kt > t || kh > h || kw > w || kt < 1 || kh < 1 || kw < 1) {
    sfb::set_error("sfb_window_avgpool_fwd: window %dx%dx%d does not fit the %dx%dx%d map", kt, kh, kw, t, h, w);
    return -1;
  }
  const int64_t items = int64_t(n) * (t - kt + 1) * (h - kh + 1) * (w - kw + 1) * c;
  if (items == 0) return 0;
  const int blocks = int(std::min<int64_t>((items + 255) / 256, kGridSms * 8));
  sfb::window_avgpool_fwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)hi, (const __nv_bfloat16*)lo, pitch, n, t, h, w, c, kt, kh, kw, out, out_pitch);
  return launch_status("window_avgpool_fwd");
}

extern "C" int sfb_rows_group_mean(const float* in, float* out, int32_t n, int32_t g, int32_t k, void* stream) {
  const int64_t items = int64_t(n) * k;
  if (items == 0) return 0;
  const int blocks = int(std::min<int64_t>((items + 255) / 256, kGridSms * 8));
  sfb::rows_group_mean_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(in, out, n, g, k);
  return launch_status("rows_group_mean");
}

extern "C" int sfb_dropout_fwd(float* x, uint8_t* mask, int64_t nelem, float p, uint64_t seed, uint64_t* step,
                               void* stream) {
  if (!(p >= 0.f && p < 1.f)) {
    set_error("sfb_dropout_fwd: p=%f outside [0,1)", p);
    return -10;
  }
  dropout_fwd_kernel<<<hd_grid(nelem, 256), 256, 0, (cudaStream_t)stream>>>(x, mask, nelem, p, seed, step);
  if (int rc = launch_status("sfb_dropout_fwd")) return rc;
  if (step) {
    counter_inc_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step);
    if (int rc = launch_status("sfb_dropout_fwd(counter)")) return rc;
  }
  return 0;
}
extern "C" int sfb_dropout_bwd(float* dx, const uint8_t* mask, int64_t nelem, float p, void* stream) {
  dropout_bwd_kernel<<<hd_grid(nelem, 256), 256, 0, (cudaStream_t)stream>>>(dx, mask, nelem, p);
  return launch_status("sfb_dropout_bwd");
}
template <bool RELU>
static int small_linear_fwd(const float* x, const float* w, const float* b, float* y, int32_t m, int32_t k, int32_t j,
                            void* stream, const char* name) {
  const int64_t threads = int64_t(m) * k * 32;
  small_linear_fwd_kernel<RELU><<<int((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, w, b, y, m, k, j);
  return launch_status(name);
}
template <bool RELU_MASK>
static int small_linear_bwd(const float* dy, const float* x, const float* w, float* dw, float* db, float* dx, int32_t m,
                            int32_t k, int32_t j, int32_t accumulate, void* stream) {
  if (dw) {
    small_linear_wgrad_kernel<<<hd_grid(int64_t(k) * j, 256), 256, 0, (cudaStream_t)stream>>>(dy, x, dw, db, m, k, j,
                                                                                             accumulate);
    if (int rc = launch_status("sfb_small_linear_bwd(wgrad)")) return rc;
  }
  if (dx) {
    small_linear_dgrad_kernel<RELU_MASK><<<hd_grid(int64_t(m) * j, 256), 256, 0, (cudaStream_t)stream>>>(dy, w, dx, m,
                                                                                                        k, j, x);
    if (int rc = launch_status("sfb_small_linear_bwd(dgrad)")) return rc;
  }
  return 0;
}
extern "C" int sfb_small_linear_fwd(const float* x, const float* w, const float* b, float* y, int32_t m, int32_t k,
                                    int32_t j, void* stream) {
  return small_linear_fwd<false>(x, w, b, y, m, k, j, stream, "sfb_small_linear_fwd");
}
extern "C" int sfb_small_linear_relu_fwd(const float* x, const float* w, const float* b, float* y, int32_t m, int32_t k,
                                         int32_t j, void* stream) {
  return small_linear_fwd<true>(x, w, b, y, m, k, j, stream, "sfb_small_linear_relu_fwd");
}
extern "C" int sfb_small_linear_bwd(const float* dy, const float* x, const float* w, float* dw, float* db, float* dx,
                                    int32_t m, int32_t k, int32_t j, int32_t accumulate, void* stream) {
  return small_linear_bwd<false>(dy, x, w, dw, db, dx, m, k, j, accumulate, stream);
}
extern "C" int sfb_small_linear_relu_bwd(const float* dy, const float* x, const float* w, float* dw, float* db,
                                         float* dx, int32_t m, int32_t k, int32_t j, int32_t accumulate, void* stream) {
  return small_linear_bwd<true>(dy, x, w, dw, db, dx, m, k, j, accumulate, stream);
}
extern "C" int sfb_row_softmax(float* x, int32_t rows, int32_t cols, void* stream) {
  row_softmax_kernel<<<(rows * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(x, rows, cols);
  return launch_status("sfb_row_softmax");
}
extern "C" int sfb_row_sigmoid(float* x, int32_t rows, int32_t cols, void* stream) {
  const int64_t nelem = int64_t(rows) * cols;
  if (nelem == 0) return 0;
  row_sigmoid_kernel<<<hd_grid(nelem, 256), 256, 0, (cudaStream_t)stream>>>(x, nelem);
  return launch_status("sfb_row_sigmoid");
}

// Stochastic-depth scales (common.py:46-59 drop_path): out[i*b + s] = floor(keep_i + U) / keep_i per sample, from the
// same counter-based generator as dropout (device step counter => fresh draws on CUDA-graph replays).
namespace sfb {
__global__ void droppath_scales_kernel(float* __restrict__ out, const float* __restrict__ rates, int n_rates, int b,
                                       uint64_t seed, const uint64_t* __restrict__ step) {
  if (step) seed = seed * 0x9E3779B97F4A7C15ull + *step;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rates * b) return;
  const float keep = 1.f - rates[i / b];
  const float u = float(mix32(seed * 0x100000001B3ull + 0xD1B54A32D192ED03ull + uint64_t(i)) >> 8) * (1.f / 16777216.f);
  out[i] = keep >= 1.f ? 1.f : (floorf(keep + u) / keep);
}
}  // namespace sfb
extern "C" int sfb_droppath_scales(float* out, const float* rates, int32_t n_rates, int32_t b, uint64_t seed,
                                   uint64_t* step, void* stream) {
  const int n = n_rates * b;
  sfb::droppath_scales_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(out, rates, n_rates, b, seed, step);
  if (int rc = launch_status("sfb_droppath_scales")) return rc;
  if (step) {
    sfb::counter_inc_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step);
    if (int rc = launch_status("sfb_droppath_scales(counter)")) return rc;
  }
  return 0;
}
