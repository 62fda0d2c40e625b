// Device-side head of the input pipeline (SURVEY.md section 8f-3): what the reference does on the host per clip before the
// fp32 H2D copy - `tensor_normalize` (slowfast/datasets/utils.py:278-297: uint8 -> float / 255, - mean, / std), the
// (T,H,W,C) -> (C,T,H,W) permute of the loaders (datasets/kinetics.py:375-405) and `pack_pathway_output`'s temporal
// sub-sampling for the slow pathway (datasets/utils.py:95-103: index_select at linspace(0, T-1, T // ALPHA).long()) - as one
// kernel, so that the H2D copy carries uint8 frames (4x fewer bytes per pathway; 5.3x for SlowFast's two pathways, which
// are both produced from the one uint8 clip).  Arithmetic order is the reference's ((x / 255 - mean) / std in fp32).
// HBM-bound: 1 B read per element (re-read from L2 for the second pathway) + 4 B written.
#include <cstdint>

#include "../../include/slowfast_b200.h"
#include "runtime.h"

namespace sfb {

// out[b, c, j, y, x] = (float(in[b, idx[j], y, x, cs]) / 255 - mean[cs]) / std[cs],  cs = reverse ? 2 - c : c
// one thread = 4 consecutive x of one (b, j, y) for all 3 channels: 12 contiguous input bytes, three 16-byte stores
__global__ void __launch_bounds__(256) clip_normalize_pack_kernel(const uint8_t* __restrict__ in, int B, int T, int H, int W,
                                                                 const int32_t* __restrict__ idx, int To, float m0,
                                                                 float m1, float m2, float s0, float s1, float s2,
                                                                 int reverse, float* __restrict__ out) {
  const int wq = W / 4;
  const int64_t items = int64_t(B) * To * H * wq;
  const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int xq = int(i % wq);
    int64_t t = i / wq;
    const int y = int(t % H);
    t /= H;
    const int j = int(t % To);
    const int b = int(t / To);
    const int f = idx ? idx[j] : j;
    const uint8_t* src = in + (((int64_t(b) * T + f) * H + y) * W + xq * 4) * 3;
    // 12 bytes, 4-byte aligned (W % 4 == 0): three 32-bit loads
    const uint32_t w0 = reinterpret_cast<const uint32_t*>(src)[0], w1 = reinterpret_cast<const uint32_t*>(src)[1],
                   w2 = reinterpret_cast<const uint32_t*>(src)[2];
    const uint8_t px[12] = {uint8_t(w0), uint8_t(w0 >> 8), uint8_t(w0 >> 16), uint8_t(w0 >> 24), uint8_t(w1), uint8_t(w1 >> 8),
                            uint8_t(w1 >> 16), uint8_t(w1 >> 24), uint8_t(w2), uint8_t(w2 >> 8), uint8_t(w2 >> 16),
                            uint8_t(w2 >> 24)};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int cs = reverse ? 2 - c : c;
      float4 v;
      // (the reference normalises first and reverses the channel order afterwards: statistics of the SOURCE channel)
      v.x = (float(px[0 + cs]) / 255.0f - mean[cs]) / stdv[cs];
      v.y = (float(px[3 + cs]) / 255.0f - mean[cs]) / stdv[cs];
      v.z = (float(px[6 + cs]) / 255.0f - mean[cs]) / stdv[cs];
      v.w = (float(px[9 + cs]) / 255.0f - mean[cs]) / stdv[cs];
      *reinterpret_cast<float4*>(out + (((int64_t(b) * 3 + c) * To + j) * H + y) * W + xq * 4) = v;
    }
  }
}
}  // namespace sfb

extern "C" int sfb_clip_normalize_pack(const uint8_t* frames, int32_t b, int32_t t, int32_t h, int32_t w,
                                       const int32_t* frame_idx, int32_t t_out, const float* mean3, const float* std3,
                                       int32_t reverse_channels, float* out, void* stream) {
  if (w % 4 || b <= 0 || t <= 0 || h <= 0 || t_out <= 0) {
    sfb::set_error("sfb_clip_normalize_pack: W=%d must be a multiple of 4 and all extents positive", w);
    return -10;
  }
  if ((reinterpret_cast<uintptr_t>(frames) & 3) || (reinterpret_cast<uintptr_t>(out) & 15)) {
    sfb::set_error("sfb_clip_normalize_pack: frames must be 4-byte and out 16-byte aligned");
    return -10;
  }
  const int64_t items = int64_t(b) * t_out * h * (w / 4);
  const int64_t want = (items + 255) / 256;
  const int grid = int(want > sfb::kGridSms * 16 ? sfb::kGridSms * 16 : want);
  sfb::clip_normalize_pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(frames, b, t, h, w, frame_idx, t_out, mean3[0],
                                                                        mean3[1], mean3[2], std3[0], std3[1], std3[2],
                                                                        reverse_channels, out);
  return sfb::launch_status("sfb_clip_normalize_pack");
}
