// Companion kernels of the Non-local block (slowfast/models/nonlocal_helper.py:103-144) on the engine.  The block's heavy
// work runs on the existing kernels (1x1x1 convs on conv_igemm / conv_wgrad, the pooling on maxpool3d, the affinity products
// on gemm_batched, the softmax on softmax_relpos with no bias); what is left is moving fp32 GEMM results into split-bf16
// operand planes with the conv bias added, and the BatchNorm behind conv_out, which - unlike every other BN of the ResNet
// family - follows a conv WITH a bias.
#include <cstdint>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "planes.cuh"
#include "runtime.h"

namespace sfb {

typedef __nv_bfloat16 nl_bf;

// 8 blocks per SM of the device (of kGridSms when there is none: the launch that follows reports it)
static int nl_grid(int64_t items, int block) {
  int sms = kGridSms;
  device_limits(&sms, nullptr);
  return capped_grid(items, block, int64_t(sms) * 8);
}

// out[r, j] = x[r, j] + bias[j] for j < c, 0 for c <= j < c_out; one thread per 8 output columns of a row
__global__ void bias_split_kernel(const float* __restrict__ x, int64_t rows, int c, int64_t x_pitch,
                                  const float* __restrict__ bias, nl_bf* __restrict__ hi, nl_bf* __restrict__ lo,
                                  int64_t o_pitch, int c_out) {
  const int cg = c_out / 8;
  const int64_t items = rows * cg;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cg;
    const int j0 = int(i - r * cg) * 8;
    const float* xr = x + r * x_pitch;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int j = j0 + e;
      const float v = j < c ? xr[j] + (bias ? bias[j] : 0.f) : 0.f;
      put_split(hi, lo, r * o_pitch + j, v);
    }
  }
}

// BatchNorm behind a biased conv, z = y + b with y the bias-free conv output the statistics were taken from:
//   train: the batch mean of z is mean(y) + b  -> running_mean += momentum * b (normalised output unchanged)
//   eval : (y + b - rm) * scale + beta         -> shift += scale * b, save_mean = rm - b (what the backward centres y by)
// splits > 1 (SubBatchNorm3d in training): running_mean is split_bn's [splits][c]; every split's mean moves by b.
__global__ void bn_conv_bias_kernel(const float* __restrict__ bias, int c, float momentum, int training,
                                    float* __restrict__ running_mean, const float* __restrict__ scale,
                                    float* __restrict__ shift, float* __restrict__ save_mean, int splits) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  const float b = bias[ch];
  if (training) {
    if (running_mean)
      for (int s = 0; s < splits; ++s) running_mean[s * c + ch] += momentum * b;
  } else {
    shift[ch] += scale[ch] * b;
    if (save_mean) save_mean[ch] -= b;
  }
}

__global__ void planes_to_f32_kernel(const nl_bf* __restrict__ hi, const nl_bf* __restrict__ lo, int64_t rows, int c,
                                     int64_t pitch, float* __restrict__ out, int64_t out_pitch) {
  const int64_t items = rows * c;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / c;
    const int j = int(i - r * c);
    float v = __bfloat162float(hi[r * pitch + j]);
    if (lo) v += __bfloat162float(lo[r * pitch + j]);
    out[r * out_pitch + j] = v;
  }
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_bias_split(const float* x, int64_t rows, int32_t c, int64_t x_pitch, const float* bias, void* hi,
                              void* lo, int64_t o_pitch, int32_t c_out, void* stream) {
  if (c_out % 8 || c > c_out || o_pitch % 8 || c_out > o_pitch || c <= 0) {
    set_error("sfb_bias_split: c=%d c_out=%d o_pitch=%lld (c <= c_out <= o_pitch, c_out and o_pitch multiples of 8)", c,
              c_out, (long long)o_pitch);
    return -10;
  }
  const int64_t items = rows * (c_out / 8);
  if (items == 0) return 0;
  bias_split_kernel<<<nl_grid(items, 256), 256, 0, (cudaStream_t)stream>>>(x, rows, c, x_pitch, bias, (nl_bf*)hi,
                                                                           (nl_bf*)lo, o_pitch, c_out);
  return launch_status("sfb_bias_split");
}

extern "C" int sfb_bn_conv_bias(const float* bias, int32_t c, float momentum, int32_t training, float* running_mean,
                                const float* scale, float* shift, float* save_mean, int32_t splits, void* stream) {
  if (!bias || (!training && (!scale || !shift))) {
    set_error("sfb_bn_conv_bias: null bias, or eval mode without scale / shift");
    return -10;
  }
  if (!training) splits = 1;  // eval uses the single BN's statistics
  bn_conv_bias_kernel<<<(c + 255) / 256, 256, 0, (cudaStream_t)stream>>>(bias, c, momentum, training, running_mean, scale,
                                                                         shift, save_mean, splits > 1 ? splits : 1);
  return launch_status("sfb_bn_conv_bias");
}

extern "C" int sfb_planes_to_f32(const void* hi, const void* lo, int64_t rows, int32_t c, int64_t pitch, float* out,
                                 int64_t out_pitch, void* stream) {
  const int64_t items = rows * c;
  if (items == 0) return 0;
  planes_to_f32_kernel<<<nl_grid(items, 256), 256, 0, (cudaStream_t)stream>>>((const nl_bf*)hi, (const nl_bf*)lo, rows, c,
                                                                               pitch, out, out_pitch);
  return launch_status("sfb_planes_to_f32");
}
