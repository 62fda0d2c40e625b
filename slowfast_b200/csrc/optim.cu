// Optimizer step and gradient norm / clipping on the engine's flat gradient bucket (SURVEY.md section 8f-1).
//
// Reference call sites replaced: torch.optim.SGD(nesterov) / AdamW built by slowfast/models/optimizer.py:105-136
// (one multi-tensor update per parameter group), get_grad_norm_ (:362-379) and clip_grad_norm_ (tools/train_net.py:154-172).
// In the reference these are ~3 ATen kernels per parameter tensor (or foreach launches over a list of 300-660 tensors)
// preceded by one gradient copy per parameter; here the gradients already sit in ONE contiguous fp32 bucket (the single
// all-reduce message), so the step is
//   1. sfb_flat_sumsq  : sum of squares of the bucket (pad slots are exact zeros) -> device scalar, fp64 merge;
//   2. sfb_flat_sgd / sfb_flat_adamw : one launch over a chunk table; every chunk = up to CHUNK contiguous elements of
//      one parameter: {param ptr, bucket offset, count, group}.  Optimizer state (momentum / exp_avg / exp_avg_sq) is a
//      bucket-shaped buffer, so state and gradient are read with the same offset; per-group hyper-parameters
//      (lr * layer_decay, weight_decay) come from a small device array; the clip coefficient is read from the device
//      scalar written by step 1 (no host synchronisation anywhere).
// Arithmetic follows torch.optim exactly (same operation order in fp32):
//   SGD   : g += wd*p; buf = first ? g : mom*buf + (1-damp)*g; g = nesterov ? g + mom*buf : buf; p -= lr*g
//   AdamW : p *= 1 - lr*wd; m = b1*m + (1-b1)*g; v = b2*v + (1-b2)*g*g; p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)
#include <algorithm>
#include <cstdint>

#include "../../include/slowfast_b200.h"
#include "runtime.h"

namespace sfb {

constexpr int OPT_THREADS = 256;

__global__ void __launch_bounds__(OPT_THREADS) flat_sumsq_partial_kernel(const float* __restrict__ g, int64_t n,
                                                                         double* __restrict__ partials) {
  double acc = 0.0;
  const int64_t n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n4; i += int64_t(gridDim.x) * blockDim.x) {
    const float4 v = g4[i];
    acc += double(v.x * v.x + v.y * v.y) + double(v.z * v.z + v.w * v.w);
  }
  for (int64_t i = (n4 << 2) + blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    acc += double(g[i]) * double(g[i]);
  __shared__ double sm[OPT_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < OPT_THREADS / 32; ++w) s += sm[w];
    partials[blockIdx.x] = s;
  }
}

// out[0] = ||g||_2 * inv_scale, out[1] = clip coefficient min(1, max_norm / (norm + 1e-6)) (1 when max_norm <= 0),
// out[2] = inv_scale * clip coefficient (what the update kernels multiply every gradient with)
__global__ void flat_sumsq_final_kernel(const double* __restrict__ partials, int nblocks, float max_norm,
                                        float inv_scale, float* __restrict__ out) {
  __shared__ double sm[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) acc += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < int(blockDim.x >> 5); ++w) s += sm[w];
    const float norm = float(sqrt(s)) * inv_scale;
    float coef = 1.f;
    if (max_norm > 0.f) coef = fminf(1.f, max_norm / (norm + 1e-6f));   // torch.nn.utils.clip_grad_norm_
    out[0] = norm;
    out[1] = coef;
    out[2] = coef * inv_scale;
  }
}

struct OptChunk {      // mirrors sfb_opt_chunk
  float* param;        // first element of this chunk inside its parameter tensor
  int64_t offset;      // element offset of the chunk in the flat bucket (gradient and state)
  int32_t count;       // elements in the chunk
  int32_t group;       // index into the per-group hyper-parameter arrays
};

template <bool ADAMW>
__global__ void __launch_bounds__(OPT_THREADS) flat_update_kernel(const OptChunk* __restrict__ chunks,
                                                                  const float* __restrict__ grad,
                                                                  float* __restrict__ state1, float* __restrict__ state2,
                                                                  const float* __restrict__ group_lr,
                                                                  const float* __restrict__ group_wd,
                                                                  const float* __restrict__ gscale,  // device scalar or null
                                                                  float momentum, float dampening, int nesterov,
                                                                  int first_step, float beta1, float beta2, float eps,
                                                                  float bc1, float bc2_sqrt) {
  const OptChunk c = chunks[blockIdx.x];
  const float lr = group_lr[c.group], wd = group_wd[c.group];
  const float gs = gscale ? gscale[2] : 1.f;
  const float* g = grad + c.offset;
  float* s1 = state1 + c.offset;
  float* s2 = ADAMW ? state2 + c.offset : nullptr;
  float* p = c.param;
  for (int i = threadIdx.x; i < c.count; i += OPT_THREADS) {
    float gi = g[i] * gs;
    float pi = p[i];
    if (ADAMW) {
      pi *= 1.f - lr * wd;
      const float m = beta1 * s1[i] + (1.f - beta1) * gi;
      const float v = beta2 * s2[i] + (1.f - beta2) * gi * gi;
      s1[i] = m;
      s2[i] = v;
      const float denom = sqrtf(v) / bc2_sqrt + eps;
      pi -= (lr / bc1) * (m / denom);
    } else {
      gi += wd * pi;
      float buf = first_step ? gi : momentum * s1[i] + (1.f - dampening) * gi;
      if (momentum != 0.f) {
        s1[i] = buf;
        gi = nesterov ? gi + momentum * buf : buf;
      }
      pi -= lr * gi;
    }
    p[i] = pi;
  }
}

struct MomentumChunk {  // mirrors sfb_momentum_chunk
  float* key;
  const float* query;
  int64_t count;
};

// key = fl(fl(q * c1) + fl(key * c2)): the explicit _rn intrinsics keep the compiler from contracting this into an FMA,
// which would round once instead of three times and differ from the reference's three ATen kernels in the last bit
__global__ void __launch_bounds__(OPT_THREADS) momentum_update_kernel(const MomentumChunk* __restrict__ chunks, float c1,
                                                                      float c2) {
  const MomentumChunk c = chunks[blockIdx.x];
  for (int64_t i = threadIdx.x; i < c.count; i += OPT_THREADS)
    c.key[i] = __fadd_rn(__fmul_rn(c.query[i], c1), __fmul_rn(c.key[i], c2));
}

}  // namespace sfb

extern "C" int32_t sfb_flat_sumsq_blocks(void) { return sfb::kGridSms * 4; }

extern "C" int sfb_flat_sumsq(const float* flat, int64_t n, double* partials, float max_norm, float inv_scale,
                              float* out3, void* stream) {
  if ((reinterpret_cast<uintptr_t>(flat) & 15) != 0) {
    sfb::set_error("sfb_flat_sumsq: the bucket must be 16-byte aligned");
    return -1;
  }
  const int nb = sfb_flat_sumsq_blocks();
  sfb::flat_sumsq_partial_kernel<<<nb, sfb::OPT_THREADS, 0, (cudaStream_t)stream>>>(flat, n, partials);
  if (int rc = sfb::launch_status("flat_sumsq_partial")) return rc;
  sfb::flat_sumsq_final_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(partials, nb, max_norm, inv_scale, out3);
  return sfb::launch_status("flat_sumsq_final");
}

extern "C" int32_t sfb_opt_chunk_size(void) { return int32_t(sizeof(sfb::OptChunk)); }

extern "C" int sfb_flat_sgd(const void* chunks, int32_t n_chunks, const float* grad, float* momentum_buf,
                            const float* group_lr, const float* group_wd, const float* gscale, float momentum,
                            float dampening, int32_t nesterov, int32_t first_step, void* stream) {
  if (n_chunks <= 0) return 0;
  sfb::flat_update_kernel<false><<<n_chunks, sfb::OPT_THREADS, 0, (cudaStream_t)stream>>>(
      (const sfb::OptChunk*)chunks, grad, momentum_buf, nullptr, group_lr, group_wd, gscale, momentum, dampening,
      nesterov, first_step, 0.f, 0.f, 0.f, 1.f, 1.f);
  return sfb::launch_status("flat_sgd");
}

extern "C" int sfb_flat_adamw(const void* chunks, int32_t n_chunks, const float* grad, float* exp_avg, float* exp_avg_sq,
                              const float* group_lr, const float* group_wd, const float* gscale, float beta1,
                              float beta2, float eps, int64_t step, void* stream) {
  if (n_chunks <= 0) return 0;
  const double bc1 = 1.0 - pow(double(beta1), double(step));
  const double bc2 = 1.0 - pow(double(beta2), double(step));
  sfb::flat_update_kernel<true><<<n_chunks, sfb::OPT_THREADS, 0, (cudaStream_t)stream>>>(
      (const sfb::OptChunk*)chunks, grad, exp_avg, exp_avg_sq, group_lr, group_wd, gscale, 0.f, 0.f, 0, 0, beta1, beta2,
      eps, float(bc1), float(sqrt(bc2)));
  return sfb::launch_status("flat_adamw");
}

extern "C" int32_t sfb_momentum_chunk_size(void) { return int32_t(sizeof(sfb::MomentumChunk)); }

extern "C" int sfb_momentum_update(const void* chunks, int32_t n_chunks, float c1, float c2, void* stream) {
  if (n_chunks <= 0) return 0;
  sfb::momentum_update_kernel<<<n_chunks, sfb::OPT_THREADS, 0, (cudaStream_t)stream>>>(
      (const sfb::MomentumChunk*)chunks, c1, c2);
  return sfb::launch_status("momentum_update");
}
