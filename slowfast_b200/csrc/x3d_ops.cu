// X3D-specific HBM-bound kernels (SURVEY.md section 8 rows a3/a4/a9/a11):
//   * channelwise (depthwise) Conv3d  kt x kh x kw, stride (st,sh,sw)           - resnet_helper.py:217-229 (X3DTransform.b),
//                                                                               stem_helper.py:268-276 (X3DStem.conv)
//     fwd (+ per-tile BatchNorm partial sums, tiles aligned to samples so that the SE average pool falls out of
//     the same partials), data gradient, weight gradient; fp32 input, 3x3x3 or 5x1x1 filters at temporal stride 1;
//   * BN -> [SE gate] -> ReLU | Swish, forward and backward, with the BN backward sums derived from per-sample sums
//     so that the SE branch costs no extra pass over the activation                 - operators.py:55-59 (SE.forward);
//   * the SE bottleneck itself (AvgPool -> 1x1x1 -> ReLU -> 1x1x1 -> Sigmoid), one block per sample.
// All activations are channels-last [rows = n*t*h*w, C] with a row pitch; C is the channel count padded to a
// multiple of 8 (X3D-M's 54 / 108 wide bottlenecks run as 56 / 112), `c_valid` the real count: pad channels carry
// exact zeros through every kernel.  4 channels (16 B fp32 / 8 B per bf16 plane) per thread.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "planes.cuh"
#include "runtime.h"

namespace sfb {

using bf = __nv_bfloat16;

static int x3_grid(int64_t items, int block, int waves = 8) {
  return capped_grid(items, block, int64_t(kGridSms) * waves);
}

// ============================================================================================ channelwise conv, v2
// Register-tiled kernels for fp32 inputs: one thread owns ONE channel (consecutive lanes = consecutive channels, so
// every load / store instruction of a warp is a contiguous 128-byte line) and a micro-tile of OTT x OHT x OWT
// outputs; the filter lives in registers, every loaded input value feeds up to KH*KW FMAs of several outputs
// (3.0 FMA per load for 3x3x3 stride 1 against 1.0 for a per-output gather).  The producer's BatchNorm + ReLU
// can be applied on the fly (x = relu(x*in_scale + in_shift)), so the activation between X3DTransform.a and .b is
// never materialised.  The same kernel computes stride-1 data gradients (correlation with the mirrored filter).
struct Dw2Params {
  const float* x; int64_t x_pitch;
  const float* in_scale; const float* in_shift; int in_relu;
  const float* w; int flip;
  float* y; int64_t y_pitch; int y_accumulate; bf* y_hi; bf* y_lo;
  float* stats;
  int n, T, H, W, C, Cv, oT, oH, oW, pt, ph, pw;
  int mt_t, mt_h, mt_w, MT;
  int tiles_per_sample, mts_per_tile, m_tiles;
  const float* dy; int64_t dy_pitch; float* dw;
  int64_t total_mts, mts_per_block;
  // ring kernels only: sample n = (outer, inner) = (n / n_inner, n % n_inner) with separate element strides per tensor
  // (MViT's pooling convs: outer = clip, inner = head; X3D: n_inner = 1, outer stride = T*H*W*pitch)
  int n_inner;
  int64_t x_so, x_si, y_so, y_si, dy_so, dy_si;
  int64_t aff_si;     // inner stride of in_scale / in_shift (per-head bias), 0 = shared
  int in_scale_one;   // in_scale == nullptr means scale 1 (x + in_shift): the fused-qkv bias of MViT
};

__device__ __forceinline__ float dw2_in(const Dw2Params& p, const float* ptr, float sc, float sh) {
  float v = *ptr;
  if (p.in_scale) {
    v = fmaf(v, sc, sh);
    if (p.in_relu) v = fmaxf(v, 0.f);
  }
  return v;
}

template <int KT, int KH, int KW, int S, int OTT, int OHT, int OWT>
__global__ void __launch_bounds__(512, 1) dw2_conv_kernel(const Dw2Params p) {
  constexpr int IT = OTT - 1 + KT, IH = (OHT - 1) * S + KH, IW = (OWT - 1) * S + KW, TAPS = KT * KH * KW;
  extern __shared__ float red[];  // [SP][2][C]
  const int C = p.C;
  const int SP = blockDim.x / C;
  const int sp = threadIdx.x / C;
  const int c = threadIdx.x - sp * C;
  const int tile = blockIdx.x;
  const int n = tile / p.tiles_per_sample;
  const int tl = tile - n * p.tiles_per_sample;
  const int mt0 = tl * p.mts_per_tile;
  const int mt1 = min(p.MT, mt0 + p.mts_per_tile);
  float w[TAPS];
#pragma unroll
  for (int k = 0; k < TAPS; ++k) w[k] = c < p.Cv ? p.w[c * TAPS + (p.flip ? TAPS - 1 - k : k)] : 0.f;
  float isc = 0.f, ish = 0.f;
  if (p.in_scale) {
    isc = p.in_scale[c];
    ish = p.in_shift[c];
  }
  float s = 0.f, s2 = 0.f;
  for (int mt = mt0 + sp; mt < mt1; mt += SP) {
    const int wi = mt % p.mt_w;
    const int r = mt / p.mt_w;
    const int hi = r % p.mt_h;
    const int ti = r / p.mt_h;
    const int oz0 = ti * OTT, oy0 = hi * OHT, ox0 = wi * OWT;
    float acc[OTT][OHT][OWT];
#pragma unroll
    for (int a = 0; a < OTT; ++a)
#pragma unroll
      for (int b = 0; b < OHT; ++b)
#pragma unroll
        for (int d = 0; d < OWT; ++d) acc[a][b][d] = 0.f;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
      const int iz = oz0 - p.pt + it;
      const bool zok = iz >= 0 && iz < p.T;
      // the whole IH x IW patch of this input frame is requested before any of it is consumed: IH*IW independent
      // loads in flight per thread (the kernel is latency-bound, not bandwidth-bound)
      float v[IH][IW];
      const int iy0 = oy0 * S - p.ph, ix0 = ox0 * S - p.pw;
      if (!zok) {
#pragma unroll
        for (int ih = 0; ih < IH; ++ih)
#pragma unroll
          for (int iw = 0; iw < IW; ++iw) v[ih][iw] = 0.f;
      } else if (iy0 >= 0 && iy0 + IH <= p.H && ix0 >= 0 && ix0 + IW <= p.W) {
        // interior patch (the common case): no bounds predicates, 32-bit offsets from one base pointer
        const float* base = p.x + (((int64_t(n) * p.T + iz) * p.H + iy0) * p.W + ix0) * p.x_pitch + c;
        const int pitch = int(p.x_pitch), rowp = p.W * pitch;
#pragma unroll
        for (int ih = 0; ih < IH; ++ih)
#pragma unroll
          for (int iw = 0; iw < IW; ++iw) v[ih][iw] = base[ih * rowp + iw * pitch];
        if (p.in_scale) {
#pragma unroll
          for (int ih = 0; ih < IH; ++ih)
#pragma unroll
            for (int iw = 0; iw < IW; ++iw) {
              const float t = fmaf(v[ih][iw], isc, ish);
              v[ih][iw] = p.in_relu ? fmaxf(t, 0.f) : t;
            }
        }
      } else {
#pragma unroll
        for (int ih = 0; ih < IH; ++ih) {
          const int iy = iy0 + ih;
          const bool yok = iy >= 0 && iy < p.H;
          const float* row = p.x + (((int64_t(n) * p.T + iz) * p.H + iy) * p.W) * p.x_pitch + c;
#pragma unroll
          for (int iw = 0; iw < IW; ++iw) {
            const int ix = ix0 + iw;
            float t = 0.f;
            if (yok && ix >= 0 && ix < p.W) {
              t = row[int64_t(ix) * p.x_pitch];
              if (p.in_scale) {
                t = fmaf(t, isc, ish);
                if (p.in_relu) t = fmaxf(t, 0.f);
              }
            }
            v[ih][iw] = t;  // padding is zero AFTER the transform
          }
        }
      }
#pragma unroll
      for (int ih = 0; ih < IH; ++ih) {
#pragma unroll
        for (int ot = 0; ot < OTT; ++ot) {
          const int kz = it - ot;
          if (kz < 0 || kz >= KT) continue;
#pragma unroll
          for (int oh = 0; oh < OHT; ++oh) {
            const int ky = ih - oh * S;
            if (ky < 0 || ky >= KH) continue;
#pragma unroll
            for (int ow = 0; ow < OWT; ++ow)
#pragma unroll
              for (int kx = 0; kx < KW; ++kx)
                acc[ot][oh][ow] = fmaf(v[ih][ow * S + kx], w[(kz * KH + ky) * KW + kx], acc[ot][oh][ow]);
          }
        }
      }
    }
#pragma unroll
    for (int ot = 0; ot < OTT; ++ot)
#pragma unroll
      for (int oh = 0; oh < OHT; ++oh)
#pragma unroll
        for (int ow = 0; ow < OWT; ++ow) {
          const int oz = oz0 + ot, oy = oy0 + oh, ox = ox0 + ow;
          if (oz < p.oT && oy < p.oH && ox < p.oW) {
            const int64_t off = (((int64_t(n) * p.oT + oz) * p.oH + oy) * p.oW + ox) * p.y_pitch + c;
            float a = acc[ot][oh][ow];
            if (p.y) {
              if (p.y_accumulate) a += p.y[off];
              p.y[off] = a;
            } else {
              const bf h = __float2bfloat16_rn(a);
              p.y_hi[off] = h;
              if (p.y_lo) p.y_lo[off] = __float2bfloat16_rn(a - __bfloat162float(h));
            }
            s += a;
            s2 = fmaf(a, a, s2);
          }
        }
  }
  if (!p.stats) return;
  red[(sp * 2 + 0) * C + c] = s;
  red[(sp * 2 + 1) * C + c] = s2;
  __syncthreads();
  for (int ch = threadIdx.x; ch < p.Cv; ch += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int j = 0; j < SP; ++j) {
      a += red[(j * 2 + 0) * C + ch];
      b += red[(j * 2 + 1) * C + ch];
    }
    p.stats[size_t(ch) * p.m_tiles + tile] = a;
    p.stats[(size_t(p.Cv) + ch) * p.m_tiles + tile] = b;
  }
}

// dw[c][k] += sum over this block's micro-tiles of dy * x(tap): 27 register accumulators per thread, block tree
// over the SP spatial lanes in shared memory, one atomic add per (channel, tap) and block into the zeroed slot
template <int KT, int KH, int KW, int S, int OTT, int OHT, int OWT>
__global__ void __launch_bounds__(512) dw2_wgrad_kernel(const Dw2Params p) {
  constexpr int IT = OTT - 1 + KT, IH = (OHT - 1) * S + KH, IW = (OWT - 1) * S + KW, TAPS = KT * KH * KW;
  extern __shared__ float red[];  // [SP][C][TAPS]
  const int C = p.C;
  const int SP = blockDim.x / C;
  const int sp = threadIdx.x / C;
  const int c = threadIdx.x - sp * C;
  const int64_t g0 = blockIdx.x * p.mts_per_block;
  const int64_t g1 = min(p.total_mts, g0 + p.mts_per_block);
  float wacc[TAPS];
#pragma unroll
  for (int k = 0; k < TAPS; ++k) wacc[k] = 0.f;
  float isc = 0.f, ish = 0.f;
  if (p.in_scale) {
    isc = p.in_scale[c];
    ish = p.in_shift[c];
  }
  for (int64_t gm = g0 + sp; gm < g1; gm += SP) {
    const int n = int(gm / p.MT);
    const int mt = int(gm - int64_t(n) * p.MT);
    const int wi = mt % p.mt_w;
    const int r = mt / p.mt_w;
    const int hi = r % p.mt_h;
    const int ti = r / p.mt_h;
    const int oz0 = ti * OTT, oy0 = hi * OHT, ox0 = wi * OWT;
    float g[OTT][OHT][OWT];
#pragma unroll
    for (int ot = 0; ot < OTT; ++ot)
#pragma unroll
      for (int oh = 0; oh < OHT; ++oh)
#pragma unroll
        for (int ow = 0; ow < OWT; ++ow) {
          const int oz = oz0 + ot, oy = oy0 + oh, ox = ox0 + ow;
          g[ot][oh][ow] = (oz < p.oT && oy < p.oH && ox < p.oW)
                              ? p.dy[(((int64_t(n) * p.oT + oz) * p.oH + oy) * p.oW + ox) * p.dy_pitch + c]
                              : 0.f;
        }
#pragma unroll
    for (int it = 0; it < IT; ++it) {
      const int iz = oz0 - p.pt + it;
      const bool zok = iz >= 0 && iz < p.T;
      float v[IH][IW];
      const int iy0 = oy0 * S - p.ph, ix0 = ox0 * S - p.pw;
      if (!zok) {
#pragma unroll
        for (int ih = 0; ih < IH; ++ih)
#pragma unroll
          for (int iw = 0; iw < IW; ++iw) v[ih][iw] = 0.f;
      } else if (iy0 >= 0 && iy0 + IH <= p.H && ix0 >= 0 && ix0 + IW <= p.W) {
        const float* base = p.x + (((int64_t(n) * p.T + iz) * p.H + iy0) * p.W + ix0) * p.x_pitch + c;
        const int pitch = int(p.x_pitch), rowp = p.W * pitch;
#pragma unroll
        for (int ih = 0; ih < IH; ++ih)
#pragma unroll
          for (int iw = 0; iw < IW; ++iw) v[ih][iw] = base[ih * rowp + iw * pitch];
        if (p.in_scale) {
#pragma unroll
          for (int ih = 0; ih < IH; ++ih)
#pragma unroll
            for (int iw = 0; iw < IW; ++iw) {
              const float t = fmaf(v[ih][iw], isc, ish);
              v[ih][iw] = p.in_relu ? fmaxf(t, 0.f) : t;
            }
        }
      } else {
#pragma unroll
        for (int ih = 0; ih < IH; ++ih) {
          const int iy = iy0 + ih;
          const bool yok = iy >= 0 && iy < p.H;
          const float* row = p.x + (((int64_t(n) * p.T + iz) * p.H + iy) * p.W) * p.x_pitch + c;
#pragma unroll
          for (int iw = 0; iw < IW; ++iw) {
            const int ix = ix0 + iw;
            float t = 0.f;
            if (yok && ix >= 0 && ix < p.W) {
              t = row[int64_t(ix) * p.x_pitch];
              if (p.in_scale) {
                t = fmaf(t, isc, ish);
                if (p.in_relu) t = fmaxf(t, 0.f);
              }
            }
            v[ih][iw] = t;
          }
        }
      }
#pragma unroll
      for (int ih = 0; ih < IH; ++ih) {
#pragma unroll
        for (int ot = 0; ot < OTT; ++ot) {
          const int kz = it - ot;
          if (kz < 0 || kz >= KT) continue;
#pragma unroll
          for (int oh = 0; oh < OHT; ++oh) {
            const int ky = ih - oh * S;
            if (ky < 0 || ky >= KH) continue;
#pragma unroll
            for (int ow = 0; ow < OWT; ++ow)
#pragma unroll
              for (int kx = 0; kx < KW; ++kx)
                wacc[(kz * KH + ky) * KW + kx] =
                    fmaf(g[ot][oh][ow], v[ih][ow * S + kx], wacc[(kz * KH + ky) * KW + kx]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < TAPS; ++k) red[(size_t(sp) * C + c) * TAPS + k] = wacc[k];
  __syncthreads();
  for (int i = threadIdx.x; i < p.Cv * TAPS; i += blockDim.x) {
    float v = 0.f;
    for (int j = 0; j < SP; ++j) v += red[size_t(j) * C * TAPS + i];
    atomicAdd(p.dw + i, v);
  }
}

// ============================================================================================ channelwise conv, v3
// Shared-memory ring kernels for the 3x3x3, stride-1, pad-1 layers on fp32 inputs (X3DTransform.b of every non-strided block
// and its stride-1 data gradient = the same correlation with the mirrored filter).  The v2 kernels above fetch every input
// element ~9x through L1 / L2 (profiles/r2_traffic.md: 0.8 TB/s effective); here a block owns one (sample, 32-channel slab,
// TH x TW spatial tile) and MARCHES over the frames: each input frame tile (+1 halo) is read from global memory ONCE into
// a 3-slot ring in shared memory (producer transform relu(x*scale+shift) applied while filling, so padding is zero after
// the transform), frame t+2 is prefetched into registers while frame t is computed, and every output frame reads its 3
// input frames from the ring.  lane = channel (every global / shared access of a warp is one contiguous 128-byte line, no
// bank conflicts), warp = a pair of output rows (two MH x 7 micro-tiles): 108 LDS + 378 FMA per 14 outputs.
// The forward emits BatchNorm partials per block with blocks aligned to samples (they double as the SE average pool).
constexpr int DW3_CB = 32;  // channels per block (= lanes)

// S = spatial stride (1, or 2 for the (1,2,2) layers: 7x7 output tiles read 15x15 input tiles); the temporal stride is 1
template <int TH, int TW, int S = 1>
struct Dw3Geo {
  static constexpr int IH = (TH - 1) * S + 3, IW = (TW - 1) * S + 3, SLOT = IH * IW * DW3_CB;  // floats per ring slot
  static constexpr int ROWS = (TH / 7 - 1) * S + 3;   // input rows of one warp's micro-tile ((MH - 1) * S + 3)
  static constexpr int COLS = 6 * S + 3;              // input columns of a 7-wide micro-tile
  static constexpr int WARPS = 7, THREADS = WARPS * 32;
  static constexpr int MH = TH / WARPS;          // output rows per warp: 2 (14x14 tile) or 1 (7x7 tile)
  static constexpr int NW = TW / 7;              // 7-wide micro-tiles per row
  static constexpr int FILL = (IH * IW + WARPS - 1) / WARPS;  // fill positions per thread
  static_assert(TH % WARPS == 0 && TW % 7 == 0, "tile must be a multiple of 7 rows x 7 columns");
};

__device__ __forceinline__ void dw3_cp_async16(float* dst_smem, const float* src) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(dst_smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
}
__device__ __forceinline__ void dw3_cp_commit_wait() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Fill mapping (different from the compute mapping): a lane moves 4 channels (16 bytes) and a warp instruction covers 4
// positions x 32 channels = 512 bytes.  The per-thread piece list is the same for every frame, so it is resolved ONCE:
// goff[i] = element offset of piece i inside a frame (>= 0), -1 = padding (zero store), -2 = no piece.
template <int TH, int TW, int S>
struct Dw3Fill {
  using G = Dw3Geo<TH, TW, S>;
  static constexpr int NQ = (G::IH * G::IW + 3) / 4, IT = (NQ + G::WARPS - 1) / G::WARPS;
  int goff[IT];
  __device__ __forceinline__ Dw3Fill(const Dw2Params& p, int h0, int w0, int ch0) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = lane >> 3, c4 = (lane & 7) * 4;
    const bool c_ok = ch0 + c4 < p.C;
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      const int q = (warp + G::WARPS * i) * 4 + sub;
      const int ih = q / G::IW, iw = q - ih * G::IW;
      const int iy = h0 * S - 1 + ih, ix = w0 * S - 1 + iw;
      goff[i] = q >= G::IH * G::IW ? -2
                : (c_ok && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) ? int((iy * p.W + ix) * p.x_pitch + ch0 + c4) : -1;
    }
  }
  // request frame iz into a ring slot: in-bounds pieces by cp.async (LDGSTS.128, no staging registers), padding by zero stores
  __device__ __forceinline__ void issue(const Dw2Params& p, float* slot, int n, int iz) const {
    if (iz < 0 || iz >= p.T) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* dst0 = slot + (warp * 4 + (lane >> 3)) * DW3_CB + (lane & 7) * 4;
    const float* base = p.x + (n / p.n_inner) * p.x_so + (n % p.n_inner) * p.x_si + int64_t(iz) * p.H * p.W * p.x_pitch;
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      float* dst = dst0 + i * (G::WARPS * 4 * DW3_CB);
      if (goff[i] >= 0) dw3_cp_async16(dst, base + goff[i]);
      else if (goff[i] == -1) *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // after the copies landed: the producer's BatchNorm (+ReLU) on the pieces THIS thread requested (padding stays zero)
  __device__ __forceinline__ void finish(const Dw2Params& p, float* slot, int iz, const float4& sc, const float4& sh) const {
    if (!(p.in_scale || p.in_scale_one) || iz < 0 || iz >= p.T) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* dst0 = slot + (warp * 4 + (lane >> 3)) * DW3_CB + (lane & 7) * 4;
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      if (goff[i] < 0) continue;
      float4* dst = reinterpret_cast<float4*>(dst0 + i * (G::WARPS * 4 * DW3_CB));
      float4 t = *dst;
      t.x = fmaf(t.x, sc.x, sh.x); t.y = fmaf(t.y, sc.y, sh.y); t.z = fmaf(t.z, sc.z, sh.z); t.w = fmaf(t.w, sc.w, sh.w);
      if (p.in_relu) {
        t.x = fmaxf(t.x, 0.f); t.y = fmaxf(t.y, 0.f); t.z = fmaxf(t.z, 0.f); t.w = fmaxf(t.w, 0.f);
      }
      *dst = t;
    }
  }
};

// one temporal tap (input frame in `slot`) of both micro-tiles of this warp
template <int TH, int TW, int S>
__device__ __forceinline__ void dw3_tap_conv(const float* slot, const float (&w)[27], int kz,
                                             float (&acc)[Dw3Geo<TH, TW, S>::NW][Dw3Geo<TH, TW, S>::MH][7]) {
  using G = Dw3Geo<TH, TW, S>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int half = 0; half < G::NW; ++half) {
#pragma unroll
    for (int r = 0; r < G::ROWS; ++r) {
      float row[G::COLS];
      const float* src = slot + ((warp * G::MH * S + r) * G::IW + half * 7 * S) * DW3_CB + lane;
#pragma unroll
      for (int j = 0; j < G::COLS; ++j) row[j] = src[j * DW3_CB];
#pragma unroll
      for (int a = 0; a < G::MH; ++a) {
        const int ky = r - a * S;
        if (ky < 0 || ky > 2) continue;
#pragma unroll
        for (int b = 0; b < 7; ++b)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) acc[half][a][b] = fmaf(row[b * S + kx], w[(kz * 3 + ky) * 3 + kx], acc[half][a][b]);
      }
    }
  }
}
template <int TH, int TW, int S>
__device__ __forceinline__ void dw3_tap_wgrad(const float* slot, float (&wacc)[27], int kz,
                                              const float (&g)[Dw3Geo<TH, TW, S>::NW][Dw3Geo<TH, TW, S>::MH][7]) {
  using G = Dw3Geo<TH, TW, S>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int half = 0; half < G::NW; ++half) {
#pragma unroll
    for (int r = 0; r < G::ROWS; ++r) {
      float row[G::COLS];
      const float* src = slot + ((warp * G::MH * S + r) * G::IW + half * 7 * S) * DW3_CB + lane;
#pragma unroll
      for (int j = 0; j < G::COLS; ++j) row[j] = src[j * DW3_CB];
#pragma unroll
      for (int a = 0; a < G::MH; ++a) {
        const int ky = r - a * S;
        if (ky < 0 || ky > 2) continue;
#pragma unroll
        for (int b = 0; b < 7; ++b)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx)
            wacc[(kz * 3 + ky) * 3 + kx] = fmaf(g[half][a][b], row[b * S + kx], wacc[(kz * 3 + ky) * 3 + kx]);
      }
    }
  }
}

// grid = (spatial tiles per sample, channel slabs, samples).  Per output frame oz: tap kz = 0 (frame oz-1) first, then the
// slot of frame oz-1 is free and receives frame oz+2 (asynchronously, under taps kz = 1, 2 and the output stores).
template <int TH, int TW, int S>
__global__ void __launch_bounds__(224, 2) dw3_conv_kernel(const Dw2Params p) {
  using G = Dw3Geo<TH, TW, S>;
  extern __shared__ __align__(16) float ring[];  // [3][IH][IW][32] (+ [WARPS][2][32] for the statistics)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tiles_w = p.oW / TW;
  const int th = blockIdx.x / tiles_w, tw = blockIdx.x - th * tiles_w;
  const int h0 = th * TH, w0 = tw * TW;
  const int n = blockIdx.z;
  const int ch0 = blockIdx.y * DW3_CB;
  const int ch = ch0 + lane;
  const bool ch_ok = ch < p.C;
  float w[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) w[k] = ch < p.Cv ? p.w[ch * 27 + (p.flip ? 26 - k : k)] : 0.f;
  const Dw3Fill<TH, TW, S> fill(p, h0, w0, ch0);
  float4 fsc = make_float4(1.f, 1.f, 1.f, 1.f), fsh = make_float4(0.f, 0.f, 0.f, 0.f);   // transform of this thread's fill channels
  if ((p.in_scale || p.in_scale_one) && ch0 + (lane & 7) * 4 < p.C) {
    const int64_t ao = (n % p.n_inner) * p.aff_si + ch0 + (lane & 7) * 4;
    if (p.in_scale) fsc = *reinterpret_cast<const float4*>(p.in_scale + ao);
    fsh = *reinterpret_cast<const float4*>(p.in_shift + ao);
  }
  fill.issue(p, ring, n, 0);
  fill.issue(p, ring + G::SLOT, n, 1);
  dw3_cp_commit_wait();
  fill.finish(p, ring, 0, fsc, fsh);
  fill.finish(p, ring + G::SLOT, 1, fsc, fsh);
  __syncthreads();
  float s = 0.f, s2 = 0.f;
  const int64_t ybase = (n / p.n_inner) * p.y_so + (n % p.n_inner) * p.y_si;
  for (int oz = 0; oz < p.T; ++oz) {
    float acc[G::NW][G::MH][7];
#pragma unroll
    for (int h = 0; h < G::NW; ++h)
#pragma unroll
      for (int a = 0; a < G::MH; ++a)
#pragma unroll
        for (int b = 0; b < 7; ++b) acc[h][a][b] = 0.f;
    if (oz >= 1) dw3_tap_conv<TH, TW, S>(ring + ((oz - 1) % 3) * G::SLOT, w, 0, acc);
    __syncthreads();                                       // slot (oz-1) % 3 == (oz+2) % 3 is free now
    float* incoming = ring + ((oz + 2) % 3) * G::SLOT;
    fill.issue(p, incoming, n, oz + 2);
    dw3_tap_conv<TH, TW, S>(ring + (oz % 3) * G::SLOT, w, 1, acc);
    if (oz + 1 < p.T) dw3_tap_conv<TH, TW, S>(ring + ((oz + 1) % 3) * G::SLOT, w, 2, acc);
    if (ch_ok) {
#pragma unroll
      for (int h = 0; h < G::NW; ++h)
#pragma unroll
        for (int a = 0; a < G::MH; ++a)
#pragma unroll
          for (int b = 0; b < 7; ++b) {
            const int oy = h0 + warp * G::MH + a, ox = w0 + h * 7 + b;
            const int64_t off = ybase + ((int64_t(oz) * p.oH + oy) * p.oW + ox) * p.y_pitch + ch;
            float v = acc[h][a][b];
            if (p.y) {
              if (p.y_accumulate) v += p.y[off];
              p.y[off] = v;
            } else {
              const bf hq = __float2bfloat16_rn(v);
              p.y_hi[off] = hq;
              if (p.y_lo) p.y_lo[off] = __float2bfloat16_rn(v - __bfloat162float(hq));
            }
            s += v;
            s2 = fmaf(v, v, s2);
          }
    }
    dw3_cp_commit_wait();
    fill.finish(p, incoming, oz + 2, fsc, fsh);
    __syncthreads();
  }
  if (!p.stats) return;
  float* red = ring + 3 * G::SLOT;
  red[(warp * 2 + 0) * DW3_CB + lane] = s;
  red[(warp * 2 + 1) * DW3_CB + lane] = s2;
  __syncthreads();
  if (warp == 0 && ch < p.Cv) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int j = 0; j < G::WARPS; ++j) {
      a += red[(j * 2 + 0) * DW3_CB + lane];
      b += red[(j * 2 + 1) * DW3_CB + lane];
    }
    const int tile = n * p.tiles_per_sample + blockIdx.x;
    p.stats[size_t(ch) * p.m_tiles + tile] = a;
    p.stats[(size_t(p.Cv) + ch) * p.m_tiles + tile] = b;
  }
}

// weight gradient with the same ring: dw[c][k] += sum over the block's outputs of dy * x(tap)
template <int TH, int TW, int S>
__global__ void __launch_bounds__(224, 2) dw3_wgrad_kernel(const Dw2Params p) {
  using G = Dw3Geo<TH, TW, S>;
  extern __shared__ __align__(16) float ring[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tiles_w = p.oW / TW;
  const int th = blockIdx.x / tiles_w, tw = blockIdx.x - th * tiles_w;
  const int h0 = th * TH, w0 = tw * TW;
  const int n = blockIdx.z;
  const int ch0 = blockIdx.y * DW3_CB;
  const int ch = ch0 + lane;
  const bool ch_ok = ch < p.C;
  float wacc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) wacc[k] = 0.f;
  const Dw3Fill<TH, TW, S> fill(p, h0, w0, ch0);
  float4 fsc = make_float4(1.f, 1.f, 1.f, 1.f), fsh = make_float4(0.f, 0.f, 0.f, 0.f);   // transform of this thread's fill channels
  if ((p.in_scale || p.in_scale_one) && ch0 + (lane & 7) * 4 < p.C) {
    const int64_t ao = (n % p.n_inner) * p.aff_si + ch0 + (lane & 7) * 4;
    if (p.in_scale) fsc = *reinterpret_cast<const float4*>(p.in_scale + ao);
    fsh = *reinterpret_cast<const float4*>(p.in_shift + ao);
  }
  fill.issue(p, ring, n, 0);
  fill.issue(p, ring + G::SLOT, n, 1);
  dw3_cp_commit_wait();
  fill.finish(p, ring, 0, fsc, fsh);
  fill.finish(p, ring + G::SLOT, 1, fsc, fsh);
  __syncthreads();
  const int64_t dybase = (n / p.n_inner) * p.dy_so + (n % p.n_inner) * p.dy_si;
  for (int oz = 0; oz < p.T; ++oz) {
    float g[G::NW][G::MH][7];
#pragma unroll
    for (int h = 0; h < G::NW; ++h)
#pragma unroll
      for (int a = 0; a < G::MH; ++a)
#pragma unroll
        for (int b = 0; b < 7; ++b) {
          const int oy = h0 + warp * G::MH + a, ox = w0 + h * 7 + b;
          g[h][a][b] = ch_ok ? p.dy[dybase + ((int64_t(oz) * p.oH + oy) * p.oW + ox) * p.dy_pitch + ch] : 0.f;
        }
    if (oz >= 1) dw3_tap_wgrad<TH, TW, S>(ring + ((oz - 1) % 3) * G::SLOT, wacc, 0, g);
    __syncthreads();
    float* incoming = ring + ((oz + 2) % 3) * G::SLOT;
    fill.issue(p, incoming, n, oz + 2);
    dw3_tap_wgrad<TH, TW, S>(ring + (oz % 3) * G::SLOT, wacc, 1, g);
    if (oz + 1 < p.T) dw3_tap_wgrad<TH, TW, S>(ring + ((oz + 1) % 3) * G::SLOT, wacc, 2, g);
    dw3_cp_commit_wait();
    fill.finish(p, incoming, oz + 2, fsc, fsh);
    __syncthreads();
  }
  // block tree over the 7 warps (the ring is free now), then one atomic per (channel, tap) and block
  float* red = ring;
#pragma unroll
  for (int k = 0; k < 27; ++k) red[(warp * 27 + k) * DW3_CB + lane] = wacc[k];
  __syncthreads();
  for (int i = threadIdx.x; i < 27 * DW3_CB; i += blockDim.x) {
    const int k = i / DW3_CB, l = i - k * DW3_CB;
    const int c = blockIdx.y * DW3_CB + l;
    if (c >= p.Cv) continue;
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < G::WARPS; ++j) v += red[(j * 27 + k) * DW3_CB + l];
    atomicAdd(p.dw + c * 27 + k, v);
  }
}

// data gradient of the 3x3x3, stride (1,2,2), padding (1,1,1) layers: micro-tile = 4x4 input positions at an even
// origin of one frame; they only ever touch a 3x3 patch of dy per temporal tap (27 loads for 108 FMAs)
__global__ void __launch_bounds__(512) dw2_dgrad_s2_kernel(const Dw2Params p) {
  // here (T,H,W) are the dims of dx (the conv's input) and (oT,oH,oW) those of dy; x = dy, y = dx
  const int C = p.C;
  const int SP = blockDim.x / C;
  const int sp = threadIdx.x / C;
  const int c = threadIdx.x - sp * C;
  float w[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) w[k] = c < p.Cv ? p.w[c * 27 + k] : 0.f;
  const int64_t g0 = blockIdx.x * p.mts_per_block;
  const int64_t g1 = min(p.total_mts, g0 + p.mts_per_block);
  for (int64_t gm = g0 + sp; gm < g1; gm += SP) {
    const int n = int(gm / p.MT);
    const int mt = int(gm - int64_t(n) * p.MT);
    const int wi = mt % p.mt_w;
    const int r = mt / p.mt_w;
    const int hi = r % p.mt_h;
    const int iz = r / p.mt_h;
    const int iy0 = hi * 4, ix0 = wi * 4;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
#pragma unroll
    for (int kz = 0; kz < 3; ++kz) {
      const int oz = iz + 1 - kz;
      const bool zok = oz >= 0 && oz < p.oT;
      float gv[3][3];
#pragma unroll
      for (int oyl = 0; oyl < 3; ++oyl) {
        const int oy = (iy0 >> 1) + oyl;
        const bool yok = zok && oy < p.oH;
#pragma unroll
        for (int oxl = 0; oxl < 3; ++oxl) {
          const int ox = (ix0 >> 1) + oxl;
          gv[oyl][oxl] = (yok && ox < p.oW)
                             ? p.x[(((int64_t(n) * p.oT + oz) * p.oH + oy) * p.oW + ox) * p.x_pitch + c]
                             : 0.f;
        }
      }
#pragma unroll
      for (int oyl = 0; oyl < 3; ++oyl) {
#pragma unroll
        for (int oxl = 0; oxl < 3; ++oxl) {
          const float g = gv[oyl][oxl];
#pragma unroll
          for (int iyl = 0; iyl < 4; ++iyl) {
            const int ky = iyl + 1 - 2 * oyl;
            if (ky < 0 || ky >= 3) continue;
#pragma unroll
            for (int ixl = 0; ixl < 4; ++ixl) {
              const int kx = ixl + 1 - 2 * oxl;
              if (kx < 0 || kx >= 3) continue;
              acc[iyl][ixl] = fmaf(g, w[(kz * 3 + ky) * 3 + kx], acc[iyl][ixl]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int iyl = 0; iyl < 4; ++iyl)
#pragma unroll
      for (int ixl = 0; ixl < 4; ++ixl) {
        const int iy = iy0 + iyl, ix = ix0 + ixl;
        if (iy < p.H && ix < p.W) {
          const int64_t off = (((int64_t(n) * p.T + iz) * p.H + iy) * p.W + ix) * p.y_pitch + c;
          float a = acc[iyl][ixl];
          if (p.y_accumulate) a += p.y[off];
          p.y[off] = a;
        }
      }
  }
}

// ============================================================================================ BN -> gate -> act
struct BnActParams {
  const float* y; int64_t y_pitch;
  const float* scale; const float* shift; const float* mean; const float* invstd;
  const float* gate; int act;
  int64_t rows, rps; int c;
  bf* o_hi; bf* o_lo; int64_t o_pitch;
  const float* dout; int64_t dout_pitch;
  float* partials; int tiles_per_sample; int tile_rows;
  const float* davg; const float* coef;
  float* dy; int64_t dy_pitch;
};
__device__ __forceinline__ float act_fwd(float u, int act) {
  if (act == 1) return fmaxf(u, 0.f);
  if (act == 2) return u / (1.f + __expf(-u));
  return u;
}
// derivative of the activation at u
__device__ __forceinline__ float act_grad(float u, int act) {
  if (act == 1) return u > 0.f ? 1.f : 0.f;
  if (act == 2) {
    const float s = 1.f / (1.f + __expf(-u));
    return s * (1.f + u * (1.f - s));  // pytorchvideo Swish backward: sigma(x) * (1 + x * (1 - sigma(x)))
  }
  return 1.f;
}
__global__ void bnact_fwd_kernel(const BnActParams p) {
  const int cq = p.c >> 2;
  const int64_t items = p.rows * cq;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cq;
    const int c = int(i - r * cq) * 4;
    const float4 y = *reinterpret_cast<const float4*>(p.y + r * p.y_pitch + c);
    const float4 sc = *reinterpret_cast<const float4*>(p.scale + c);
    const float4 sh = *reinterpret_cast<const float4*>(p.shift + c);
    float4 g = make_float4(1.f, 1.f, 1.f, 1.f);
    if (p.gate) g = *reinterpret_cast<const float4*>(p.gate + (r / p.rps) * p.c + c);
    float4 o;
    o.x = act_fwd(fmaf(y.x, sc.x, sh.x) * g.x, p.act);
    o.y = act_fwd(fmaf(y.y, sc.y, sh.y) * g.y, p.act);
    o.z = act_fwd(fmaf(y.z, sc.z, sh.z) * g.z, p.act);
    o.w = act_fwd(fmaf(y.w, sc.w, sh.w) * g.w, p.act);
    store_planes4(p.o_hi, p.o_lo, r * p.o_pitch + c, o);
  }
}

// g = dout * act'(u);  per tile (aligned to samples): partials[tile][0][c] = sum g, [tile][1][c] = sum g * xhat
__global__ void __launch_bounds__(256) bnact_bwd_reduce_kernel(const BnActParams p) {
  extern __shared__ float red[];  // [PL][2][c]
  const int cq = p.c >> 2;
  const int PL = blockDim.x / cq;
  const int tile = blockIdx.x;
  const int64_t n = tile / p.tiles_per_sample;
  const int tl = tile - int(n) * p.tiles_per_sample;
  const int64_t r0 = n * p.rps + int64_t(tl) * p.tile_rows;
  const int64_t r1 = min((n + 1) * p.rps, r0 + p.tile_rows);
  const int pl = threadIdx.x / cq;
  const int c = (threadIdx.x - pl * cq) * 4;
  if (pl < PL) {
    const float4 sc = *reinterpret_cast<const float4*>(p.scale + c);
    const float4 sh = *reinterpret_cast<const float4*>(p.shift + c);
    const float4 mu = *reinterpret_cast<const float4*>(p.mean + c);
    const float4 is = *reinterpret_cast<const float4*>(p.invstd + c);
    float4 gt = make_float4(1.f, 1.f, 1.f, 1.f);
    if (p.gate) gt = *reinterpret_cast<const float4*>(p.gate + n * p.c + c);
    float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), a2 = a1;
    for (int64_t r = r0 + pl; r < r1; r += PL) {
      const float4 y = *reinterpret_cast<const float4*>(p.y + r * p.y_pitch + c);
      const float4 d = *reinterpret_cast<const float4*>(p.dout + r * p.dout_pitch + c);
      float g;
      g = d.x * act_grad(fmaf(y.x, sc.x, sh.x) * gt.x, p.act); a1.x += g; a2.x = fmaf(g, (y.x - mu.x) * is.x, a2.x);
      g = d.y * act_grad(fmaf(y.y, sc.y, sh.y) * gt.y, p.act); a1.y += g; a2.y = fmaf(g, (y.y - mu.y) * is.y, a2.y);
      g = d.z * act_grad(fmaf(y.z, sc.z, sh.z) * gt.z, p.act); a1.z += g; a2.z = fmaf(g, (y.z - mu.z) * is.z, a2.z);
      g = d.w * act_grad(fmaf(y.w, sc.w, sh.w) * gt.w, p.act); a1.w += g; a2.w = fmaf(g, (y.w - mu.w) * is.w, a2.w);
    }
    *reinterpret_cast<float4*>(red + (pl * 2 + 0) * p.c + c) = a1;
    *reinterpret_cast<float4*>(red + (pl * 2 + 1) * p.c + c) = a2;
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < 2 * p.c; ch += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j < PL; ++j) a += red[size_t(j) * 2 * p.c + ch];
    p.partials[size_t(tile) * 2 * p.c + ch] = a;
  }
}

// dz = g * gate + davg[n];   dy = ca * dz - cb - xhat * cc     (fp32 output for the depthwise kernels)
__global__ void bnact_bwd_apply_kernel(const BnActParams p) {
  const int cq = p.c >> 2;
  const int64_t items = p.rows * cq;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < items; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cq;
    const int c = int(i - r * cq) * 4;
    const int64_t n = r / p.rps;
    const float4 y = *reinterpret_cast<const float4*>(p.y + r * p.y_pitch + c);
    const float4 d = *reinterpret_cast<const float4*>(p.dout + r * p.dout_pitch + c);
    const float4 sc = *reinterpret_cast<const float4*>(p.scale + c);
    const float4 sh = *reinterpret_cast<const float4*>(p.shift + c);
    const float4 mu = *reinterpret_cast<const float4*>(p.mean + c);
    const float4 is = *reinterpret_cast<const float4*>(p.invstd + c);
    const float4 ca = *reinterpret_cast<const float4*>(p.coef + c);
    const float4 cb = *reinterpret_cast<const float4*>(p.coef + p.c + c);
    const float4 cc = *reinterpret_cast<const float4*>(p.coef + 2 * p.c + c);
    float4 gt = make_float4(1.f, 1.f, 1.f, 1.f), da = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.gate) gt = *reinterpret_cast<const float4*>(p.gate + n * p.c + c);
    if (p.davg) da = *reinterpret_cast<const float4*>(p.davg + n * p.c + c);
    float4 o;
    float dz;
    dz = fmaf(d.x * act_grad(fmaf(y.x, sc.x, sh.x) * gt.x, p.act), gt.x, da.x);
    o.x = ca.x * dz - cb.x - (y.x - mu.x) * is.x * cc.x;
    dz = fmaf(d.y * act_grad(fmaf(y.y, sc.y, sh.y) * gt.y, p.act), gt.y, da.y);
    o.y = ca.y * dz - cb.y - (y.y - mu.y) * is.y * cc.y;
    dz = fmaf(d.z * act_grad(fmaf(y.z, sc.z, sh.z) * gt.z, p.act), gt.z, da.z);
    o.z = ca.z * dz - cb.z - (y.z - mu.z) * is.z * cc.z;
    dz = fmaf(d.w * act_grad(fmaf(y.w, sc.w, sh.w) * gt.w, p.act), gt.w, da.w);
    o.w = ca.w * dz - cb.w - (y.w - mu.w) * is.w * cc.w;
    *reinterpret_cast<float4*>(p.dy + r * p.dy_pitch + c) = o;
  }
}

// ============================================================================================ SE bottleneck
struct SeParams {
  int n, c, cp, f; float rps; int tps, m_tiles;
  const float* stats; const float* scale; const float* shift; const float* mean; const float* invstd;
  const float* w1; const float* b1; const float* w2; const float* b2;
  float* ymean; float* avg; float* hid; float* gate;
  const float* partials; int tps2;
  float* a12; float* do2; float* dhid; float* davg;
  const float* gamma; const float* beta;
  float* dw1; float* db1; float* dw2; float* db2; float* dgamma; float* dbeta; float* coef;
  int training, has_se; double count;
};
// one block per sample: per-sample channel means out of the conv's tile partials, then the two tiny FCs
__global__ void __launch_bounds__(256) se_fwd_kernel(const SeParams p) {
  extern __shared__ float sm[];  // avg[cp] | hid[f]
  float* s_avg = sm;
  float* s_hid = sm + p.cp;
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < p.cp; c += blockDim.x) {
    float ym = 0.f, a = 0.f;
    if (c < p.c) {
      const float* st = p.stats + size_t(c) * p.m_tiles + size_t(n) * p.tps;
      float s = 0.f;
      for (int t = 0; t < p.tps; ++t) s += st[t];
      ym = s / p.rps;
      a = fmaf(ym, p.scale[c], p.shift[c]);
    }
    p.ymean[size_t(n) * p.cp + c] = ym;
    p.avg[size_t(n) * p.cp + c] = a;
    s_avg[c] = a;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int f = warp; f < p.f; f += blockDim.x >> 5) {
    float v = 0.f;
    for (int c = lane; c < p.c; c += 32) v = fmaf(p.w1[size_t(f) * p.c + c], s_avg[c], v);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) {
      v = fmaxf(v + p.b1[f], 0.f);
      s_hid[f] = v;
      p.hid[size_t(n) * p.f + f] = v;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < p.cp; c += blockDim.x) {
    float g = 0.f;
    if (c < p.c) {
      float v = p.b2[c];
      for (int f = 0; f < p.f; ++f) v = fmaf(p.w2[size_t(c) * p.f + f], s_hid[f], v);
      g = 1.f / (1.f + expf(-v));
    }
    p.gate[size_t(n) * p.cp + c] = g;
  }
}
// backward, per sample: merge the tile partials (A1 = sum g, A2 = sum g*xhat), then back through the FCs
__global__ void __launch_bounds__(256) se_bwd_sample_kernel(const SeParams p) {
  extern __shared__ float sm[];  // do2[cp] | dhid[f]
  float* s_do2 = sm;
  float* s_dh = sm + p.cp;
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < p.cp; c += blockDim.x) {
    float a1 = 0.f, a2 = 0.f;
    for (int t = 0; t < p.tps2; ++t) {
      const float* pp = p.partials + (size_t(n) * p.tps2 + t) * 2 * p.cp;
      a1 += pp[c];
      a2 += pp[p.cp + c];
    }
    p.a12[(size_t(n) * 2 + 0) * p.cp + c] = a1;
    p.a12[(size_t(n) * 2 + 1) * p.cp + c] = a2;
    if (p.has_se) {
      float d = 0.f;
      if (c < p.c) {
        const float dg = p.gamma[c] * a2 + p.beta[c] * a1;  // sum_pos g * z,  z = gamma*xhat + beta
        const float g = p.gate[size_t(n) * p.cp + c];
        d = dg * g * (1.f - g);
      }
      s_do2[c] = d;
      p.do2[size_t(n) * p.cp + c] = d;
    }
  }
  if (!p.has_se) return;
  __syncthreads();
  for (int f = threadIdx.x; f < p.f; f += blockDim.x) {
    float v = 0.f;
    for (int c = 0; c < p.c; ++c) v = fmaf(p.w2[size_t(c) * p.f + f], s_do2[c], v);
    v = p.hid[size_t(n) * p.f + f] > 0.f ? v : 0.f;
    s_dh[f] = v;
    p.dhid[size_t(n) * p.f + f] = v;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < p.cp; c += blockDim.x) {
    float v = 0.f;
    if (c < p.c) {
      // d(avg)/d(z) = 1/rows_per_sample for every position of the sample; avg = mean_pos z
      for (int f = 0; f < p.f; ++f) v = fmaf(p.w1[size_t(f) * p.c + c], s_dh[f], v);
      v /= p.rps;
    }
    p.davg[size_t(n) * p.cp + c] = v;
  }
}
// per channel: BatchNorm sums / parameter gradients / apply coefficients and the SE parameter gradients
__global__ void __launch_bounds__(64) se_bwd_channel_kernel(const SeParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0 && p.has_se) {
    for (int f = threadIdx.x; f < p.f; f += blockDim.x) {
      float v = 0.f;
      for (int n = 0; n < p.n; ++n) v += p.dhid[size_t(n) * p.f + f];
      p.db1[f] = v;
    }
  }
  if (c >= p.cp) return;
  if (c >= p.c) {
    p.coef[c] = 0.f;
    p.coef[p.cp + c] = 0.f;
    p.coef[2 * p.cp + c] = 0.f;
    return;
  }
  double s1 = 0.0, s2 = 0.0;
  const float mu = p.mean[c], is = p.invstd[c];
  for (int n = 0; n < p.n; ++n) {
    const float a1 = p.a12[(size_t(n) * 2 + 0) * p.cp + c], a2 = p.a12[(size_t(n) * 2 + 1) * p.cp + c];
    if (p.has_se) {
      const float g = p.gate[size_t(n) * p.cp + c];
      const float da = p.davg[size_t(n) * p.cp + c];  // per position
      const float sx = (p.ymean[size_t(n) * p.cp + c] - mu) * is * p.rps;  // sum_pos xhat of this sample
      s1 += double(g) * a1 + double(da) * p.rps;
      s2 += double(g) * a2 + double(da) * sx;
    } else {
      s1 += a1;
      s2 += a2;
    }
  }
  p.dgamma[c] = float(s2);
  p.dbeta[c] = float(s1);
  const double a = double(p.gamma[c]) * double(is);
  p.coef[c] = float(a);
  p.coef[p.cp + c] = p.training ? float(a * s1 / p.count) : 0.f;
  p.coef[2 * p.cp + c] = p.training ? float(a * s2 / p.count) : 0.f;
  if (p.has_se) {
    float b2 = 0.f;
    for (int n = 0; n < p.n; ++n) b2 += p.do2[size_t(n) * p.cp + c];
    p.db2[c] = b2;
    for (int f = 0; f < p.f; ++f) {
      float v2 = 0.f, v1 = 0.f;
      for (int n = 0; n < p.n; ++n) {
        v2 = fmaf(p.do2[size_t(n) * p.cp + c], p.hid[size_t(n) * p.f + f], v2);
        v1 = fmaf(p.dhid[size_t(n) * p.f + f], p.avg[size_t(n) * p.cp + c], v1);
      }
      p.dw2[size_t(c) * p.f + f] = v2;
      p.dw1[size_t(f) * p.c + c] = v1;
    }
  }
}

__global__ void relu_fwd_kernel(float* x, int64_t n) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    x[i] = fmaxf(x[i], 0.f);
}
__global__ void relu_bwd_kernel(float* dx, const float* y, int64_t n) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    dx[i] = y[i] > 0.f ? dx[i] : 0.f;
}

// ------------------------------------------------------------------------------------------------ host helpers
static int dw_tiles_per_sample(int n, int64_t P) {
  int64_t want = (int64_t(kGridSms) * 8 + n - 1) / n;  // ~8 tiles per SM over the whole batch
  int64_t maxt = (P + 63) / 64;                   // at least 64 positions per tile
  if (want > maxt) want = maxt;
  return int(want < 1 ? 1 : want);
}
static void bnact_fill(BnActParams& p, const sfb_bnact_desc* d) {
  memset(&p, 0, sizeof(p));
  p.y = d->y; p.y_pitch = d->y_pitch; p.scale = d->scale; p.shift = d->shift; p.mean = d->mean; p.invstd = d->invstd;
  p.gate = d->gate; p.act = d->act; p.rows = d->rows; p.rps = d->rows_per_sample; p.c = d->c;
  p.o_hi = (bf*)d->out_hi; p.o_lo = (bf*)d->out_lo; p.o_pitch = d->out_pitch;
  p.dout = d->dout; p.dout_pitch = d->dout_pitch; p.partials = d->partials;
  const int n = int(d->rows / d->rows_per_sample);
  p.tiles_per_sample = dw_tiles_per_sample(n, d->rows_per_sample);
  p.tile_rows = int((d->rows_per_sample + p.tiles_per_sample - 1) / p.tiles_per_sample);
  p.davg = d->davg; p.coef = d->coef; p.dy = d->dy; p.dy_pitch = d->dy_pitch;
}
static int bnact_check(const sfb_bnact_desc* d, const char* who) {
  if (d->c % 8 || d->c <= 0 || d->c > 1024 || d->rows_per_sample <= 0 || d->rows % d->rows_per_sample) {
    set_error("%s: c=%d must be a multiple of 8 (<= 1024) and rows a multiple of rows_per_sample", who, d->c);
    return -10;
  }
  return 0;
}
static void se_fill(SeParams& p, const sfb_se_desc* d) {
  memset(&p, 0, sizeof(p));
  p.n = d->n; p.c = d->c; p.cp = d->c_pad; p.f = d->f; p.rps = float(d->rows_per_sample);
  p.tps = d->tiles_per_sample; p.m_tiles = d->m_tiles;
  p.stats = d->stats; p.scale = d->scale; p.shift = d->shift; p.mean = d->mean; p.invstd = d->invstd;
  p.w1 = d->w1; p.b1 = d->b1; p.w2 = d->w2; p.b2 = d->b2;
  p.ymean = d->ymean; p.avg = d->avg; p.hid = d->hid; p.gate = d->gate;
  p.partials = d->partials; p.tps2 = d->tiles2_per_sample;
  p.a12 = d->a12; p.do2 = d->do2; p.dhid = d->dhid; p.davg = d->davg;
  p.gamma = d->gamma; p.beta = d->beta;
  p.dw1 = d->dw1; p.db1 = d->db1; p.dw2 = d->dw2; p.db2 = d->db2; p.dgamma = d->dgamma; p.dbeta = d->dbeta;
  p.coef = d->coef; p.training = d->training; p.has_se = d->has_se;
  p.count = double(d->n) * double(d->rows_per_sample);
}


// ------------------------------------------------------------------------------------------------ v2 dispatch
// The geometries the channelwise kernels take: c a multiple of 8 up to 512 (one block of <= 512 threads spans the
// channels), temporal stride 1, and a 3x3x3 filter at spatial stride 1 or 2 or a 5x1x1 filter at stride 1.
// cfg: 0 = 3x3x3 stride (1,1,1), 1 = 3x3x3 stride (1,2,2), 2 = 5x1x1 stride 1;  -1 = no kernel takes the geometry
static int dw2_cfg(const sfb_dwconv_desc* d) {
  if (d->c % 8 || d->c <= 0 || d->c > 512 || d->st != 1) return -1;
  if (d->kt == 3 && d->kh == 3 && d->kw == 3 && d->sh == d->sw && (d->sh == 1 || d->sh == 2)) return d->sh == 1 ? 0 : 1;
  if (d->kt == 5 && d->kh == 1 && d->kw == 1 && d->sh == 1 && d->sw == 1) return 2;
  return -1;
}
// dw2_cfg of a convolution call, or -1 with the error set when no kernel takes its geometry or operands
static int dw2_cfg_checked(const sfb_dwconv_desc* d, const char* who) {
  const int cfg = dw2_cfg(d);
  if (cfg < 0) {
    set_error("%s: c=%d, filter %dx%dx%d, stride (%d,%d,%d): the channelwise kernels take c a multiple of 8 <= 512, "
              "temporal stride 1 and a 3x3x3 filter at spatial stride 1 or 2 or a 5x1x1 filter at stride 1",
              who, d->c, d->kt, d->kh, d->kw, d->st, d->sh, d->sw);
    return -1;
  }
  if (d->x_f32 == nullptr || d->x_pitch % 4 || d->c_valid <= 0 || d->c_valid > d->c) {
    set_error("%s: needs an fp32 input with a pitch multiple of 4 and 0 < c_valid=%d <= c=%d", who, d->c_valid, d->c);
    return -1;
  }
  return cfg;
}
static const int kDw2Tile[3][3] = {{1, 2, 4}, {1, 1, 4}, {4, 1, 1}};
// spatial lanes of a block: 512 threads over the channels
static int dw2_sp(int c) { return std::max(1, 512 / c); }
// forward tiling: micro-tiles per sample, tiles (= blocks = BatchNorm partial columns) per sample
static void dw2_fwd_tiling(int n, int ot, int oh, int ow, int c, int cfg, Dw2Params& p) {
  p.mt_t = (ot + kDw2Tile[cfg][0] - 1) / kDw2Tile[cfg][0];
  p.mt_h = (oh + kDw2Tile[cfg][1] - 1) / kDw2Tile[cfg][1];
  p.mt_w = (ow + kDw2Tile[cfg][2] - 1) / kDw2Tile[cfg][2];
  p.MT = p.mt_t * p.mt_h * p.mt_w;
  const int sp = dw2_sp(c);
  int want = (kGridSms * 8 + n - 1) / n;
  const int maxt = (p.MT + sp - 1) / sp;
  if (want > maxt) want = maxt;
  if (want < 1) want = 1;
  p.tiles_per_sample = want;
  p.mts_per_tile = (p.MT + want - 1) / want;
  p.m_tiles = n * want;
}
static void dw2_common(Dw2Params& p, const sfb_dwconv_desc* d) {
  memset(&p, 0, sizeof(p));
  p.x = d->x_f32; p.x_pitch = d->x_pitch;
  p.in_scale = d->in_scale; p.in_shift = d->in_shift; p.in_relu = d->in_relu;
  p.w = d->w;
  p.n = d->n; p.T = d->t; p.H = d->h; p.W = d->w_; p.C = d->c; p.Cv = d->c_valid;
  p.oT = d->ot; p.oH = d->oh; p.oW = d->ow; p.pt = d->pt; p.ph = d->ph; p.pw = d->pw;
}
static void dw2_block_split(Dw2Params& p, int c, int* blocks) {
  const int sp = dw2_sp(c);
  p.total_mts = int64_t(p.n) * p.MT;
  int64_t nb = (p.total_mts + sp - 1) / sp;
  if (nb > kGridSms * 4) nb = kGridSms * 4;
  if (nb < 1) nb = 1;
  p.mts_per_block = (p.total_mts + nb - 1) / nb;
  *blocks = int((p.total_mts + p.mts_per_block - 1) / p.mts_per_block);
}
// v3 (shared-memory ring) eligibility: 3x3x3, stride 1, padding 1, H and W multiples of 7.  tile = 14x14 or 7x7
// `samples` x `c` decide between 14x14 tiles (31 % halo) and 7x7 tiles (65 % halo, 4x the blocks): the big tile only when it
// still yields two blocks per SM (ncu r2h: 48-block launches at 255 GB/s on the 14x14 stages of MViT)
static int dw3_tile(int t, int h, int w, int ot, int oh, int ow, int kt, int kh, int kw, int st, int sh, int sw, int pt,
                    int ph, int pw, int samples, int c, bool wgrad = false) {
  if (kt != 3 || kh != 3 || kw != 3 || st != 1 || sh != 1 || sw != 1 || pt != 1 || ph != 1 ||
      pw != 1 || ot != t || oh != h || ow != w || t < 2)
    return 0;
  if (h % 14 == 0 && w % 14 == 0) {
    // measured (profiles/r2_dw_ring_probe.md): the conv wants >= 1 block per SM before the 4x smaller tile pays off; the
    // weight gradient (one atomic per channel, tap and block) keeps the big tile down to half a block per SM
    const int64_t blocks14 = int64_t(h / 14) * (w / 14) * ((c + DW3_CB - 1) / DW3_CB) * samples;
    return blocks14 >= (wgrad ? 64 : kGridSms) ? 14 : 7;
  }
  if (h % 7 == 0 && w % 7 == 0) return 7;
  return 0;
}
static int dw3_tile_of(const sfb_dwconv_desc* d, bool wgrad = false) {
  return dw3_tile(d->t, d->h, d->w_, d->ot, d->oh, d->ow, d->kt, d->kh, d->kw, d->st, d->sh, d->sw, d->pt, d->ph, d->pw,
                  d->n, d->c, wgrad);
}
template <int TILE, int S>
static size_t dw3_smem(bool wgrad) {
  using G = Dw3Geo<TILE, TILE, S>;
  const size_t ring = size_t(3) * G::SLOT * sizeof(float);
  const size_t tail = wgrad ? size_t(G::WARPS) * 27 * DW3_CB * sizeof(float) : size_t(G::WARPS) * 2 * DW3_CB * sizeof(float);
  return wgrad ? std::max(ring, tail) : ring + tail;
}
// p: geometry of the "input" (T,H,W,C), x / y / dy / dw / stats / flip set by the caller
static int dw3_launch(int tile, bool wgrad, Dw2Params& p, cudaStream_t st, int stride = 1) {
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(dw3_conv_kernel<14, 14, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024);
    cudaFuncSetAttribute(dw3_conv_kernel<7, 7, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024);
    cudaFuncSetAttribute(dw3_conv_kernel<7, 7, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024);
    cudaFuncSetAttribute(dw3_wgrad_kernel<14, 14, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024);
    cudaFuncSetAttribute(dw3_wgrad_kernel<7, 7, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024);
    cudaFuncSetAttribute(dw3_wgrad_kernel<7, 7, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 120 * 1024);
    attr = true;
  }
  p.tiles_per_sample = (p.oH / tile) * (p.oW / tile);
  p.m_tiles = p.n * p.tiles_per_sample;
  if (p.n_inner <= 0) {  // dense NDHWC tensors (X3D): one sample = T*H*W rows of each tensor
    p.n_inner = 1;
    p.x_so = int64_t(p.T) * p.H * p.W * p.x_pitch;
    p.y_so = int64_t(p.oT) * p.oH * p.oW * p.y_pitch;
    p.dy_so = int64_t(p.oT) * p.oH * p.oW * p.dy_pitch;
    p.x_si = p.y_si = p.dy_si = p.aff_si = 0;
  }
  const dim3 grid(p.tiles_per_sample, (p.C + DW3_CB - 1) / DW3_CB, p.n);
  if (stride == 2) {
    if (wgrad) dw3_wgrad_kernel<7, 7, 2><<<grid, 224, dw3_smem<7, 2>(true), st>>>(p);
    else dw3_conv_kernel<7, 7, 2><<<grid, 224, dw3_smem<7, 2>(false), st>>>(p);
  } else if (tile == 14) {
    if (wgrad) dw3_wgrad_kernel<14, 14, 1><<<grid, 224, dw3_smem<14, 1>(true), st>>>(p);
    else dw3_conv_kernel<14, 14, 1><<<grid, 224, dw3_smem<14, 1>(false), st>>>(p);
  } else {
    if (wgrad) dw3_wgrad_kernel<7, 7, 1><<<grid, 224, dw3_smem<7, 1>(true), st>>>(p);
    else dw3_conv_kernel<7, 7, 1><<<grid, 224, dw3_smem<7, 1>(false), st>>>(p);
  }
  return launch_status("sfb_dwconv (v3 ring kernel)");
}

// stride (1,2,2) eligibility: 3x3x3, padding 1, even input extents, output extents multiples of 7
static bool dw3_s2_ok(const sfb_dwconv_desc* d) {
  return d->kt == 3 && d->kh == 3 && d->kw == 3 && d->st == 1 && d->sh == 2 &&
         d->sw == 2 && d->pt == 1 && d->ph == 1 && d->pw == 1 && d->ot == d->t && d->h == 2 * d->oh && d->w_ == 2 * d->ow &&
         d->oh % 7 == 0 && d->ow % 7 == 0 && d->t >= 2;
}

// Entry for other translation units (mvit_ops.cu: attention_pool's depthwise conv on tokens).  mode 0 = conv / stride-1 data
// gradient (flip), 1 = weight gradient.  Returns -100 when the geometry is not eligible (caller falls back).
int dw3_run_strided(int mode, const float* x, int64_t x_pitch, int64_t x_so, int64_t x_si, const float* in_shift, int64_t aff_si,
                    const float* w, int flip, float* y, int64_t y_pitch, int64_t y_so, int64_t y_si, int y_accumulate,
                    const float* dy, int64_t dy_pitch, int64_t dy_so, int64_t dy_si, float* dw, int n_outer, int n_inner,
                    int T, int H, int W, int C, cudaStream_t st) {
  const int tile = dw3_tile(T, H, W, T, H, W, 3, 3, 3, 1, 1, 1, 1, 1, 1, n_outer * n_inner, C, mode == 1);
  if (!tile || C % 4) return -100;
  Dw2Params p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.x_pitch = x_pitch; p.in_shift = in_shift; p.in_scale_one = in_shift != nullptr; p.aff_si = aff_si;
  p.w = w; p.flip = flip;
  p.y = y; p.y_pitch = y_pitch; p.y_accumulate = y_accumulate;
  p.dy = dy; p.dy_pitch = dy_pitch; p.dw = dw;
  p.n = n_outer * n_inner; p.T = T; p.H = H; p.W = W; p.C = C; p.Cv = C;
  p.oT = T; p.oH = H; p.oW = W; p.pt = p.ph = p.pw = 1;
  p.n_inner = n_inner; p.x_so = x_so; p.x_si = x_si; p.y_so = y_so; p.y_si = y_si; p.dy_so = dy_so; p.dy_si = dy_si;
  return dw3_launch(tile, mode == 1, p, st);
}

template <typename K>
static void dw2_optin(K kernel) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
}
static int dw2_launch_conv(int cfg, const Dw2Params& p, int threads, size_t smem, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    dw2_optin(dw2_conv_kernel<3, 3, 3, 1, 1, 2, 4>);
    dw2_optin(dw2_conv_kernel<3, 3, 3, 2, 1, 1, 4>);
    dw2_optin(dw2_conv_kernel<5, 1, 1, 1, 4, 1, 1>);
    attr = true;
  }
  if (cfg == 0) dw2_conv_kernel<3, 3, 3, 1, 1, 2, 4><<<p.m_tiles, threads, smem, st>>>(p);
  else if (cfg == 1) dw2_conv_kernel<3, 3, 3, 2, 1, 1, 4><<<p.m_tiles, threads, smem, st>>>(p);
  else dw2_conv_kernel<5, 1, 1, 1, 4, 1, 1><<<p.m_tiles, threads, smem, st>>>(p);
  return launch_status("sfb_dwconv (v2 conv)");
}
static int dw2_launch_wgrad(int cfg, const Dw2Params& p, int blocks, int threads, size_t smem, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    dw2_optin(dw2_wgrad_kernel<3, 3, 3, 1, 1, 2, 4>);
    dw2_optin(dw2_wgrad_kernel<3, 3, 3, 2, 1, 1, 4>);
    dw2_optin(dw2_wgrad_kernel<5, 1, 1, 1, 4, 1, 1>);
    attr = true;
  }
  if (cfg == 0) dw2_wgrad_kernel<3, 3, 3, 1, 1, 2, 4><<<blocks, threads, smem, st>>>(p);
  else if (cfg == 1) dw2_wgrad_kernel<3, 3, 3, 2, 1, 1, 4><<<blocks, threads, smem, st>>>(p);
  else dw2_wgrad_kernel<5, 1, 1, 1, 4, 1, 1><<<blocks, threads, smem, st>>>(p);
  return launch_status("sfb_dwconv (v2 wgrad)");
}

}  // namespace sfb

using namespace sfb;

extern "C" int32_t sfb_dwconv_tiles_per_sample(const sfb_dwconv_desc* d) {
  const int cfg = dw2_cfg(d);
  if (cfg < 0) return 0;
  if (cfg == 0) {
    const int t3 = dw3_tile_of(d);
    if (t3) return (d->h / t3) * (d->w_ / t3);
  }
  if (cfg == 1 && dw3_s2_ok(d)) return (d->oh / 7) * (d->ow / 7);
  Dw2Params p;
  dw2_fwd_tiling(d->n, d->ot, d->oh, d->ow, d->c, cfg, p);
  return p.tiles_per_sample;
}
extern "C" int32_t sfb_dwconv_m_tiles(const sfb_dwconv_desc* d) { return d->n * sfb_dwconv_tiles_per_sample(d); }
extern "C" int sfb_dwconv_fwd(const sfb_dwconv_desc* d, void* stream) {
  const int cfg2 = dw2_cfg_checked(d, "sfb_dwconv_fwd");
  if (cfg2 < 0) return -10;
  if (cfg2 == 0) {
    if (const int t3 = dw3_tile_of(d)) {
      Dw2Params q;
      dw2_common(q, d);
      q.y = d->y; q.y_pitch = d->y_pitch; q.stats = d->stats;
      return dw3_launch(t3, false, q, (cudaStream_t)stream);
    }
  }
  if (cfg2 == 1 && dw3_s2_ok(d)) {
    Dw2Params q;
    dw2_common(q, d);
    q.y = d->y; q.y_pitch = d->y_pitch; q.stats = d->stats;
    return dw3_launch(7, false, q, (cudaStream_t)stream, 2);
  }
  Dw2Params q;
  dw2_common(q, d);
  dw2_fwd_tiling(d->n, d->ot, d->oh, d->ow, d->c, cfg2, q);
  q.y = d->y; q.y_pitch = d->y_pitch; q.stats = d->stats;
  const int sp = dw2_sp(d->c);
  return dw2_launch_conv(cfg2, q, sp * d->c, size_t(sp) * 2 * d->c * sizeof(float), (cudaStream_t)stream);
}
extern "C" int sfb_dwconv_bwd(const sfb_dwconv_desc* d, float* dw, void* stream) {
  const int cfg2 = dw2_cfg_checked(d, "sfb_dwconv_bwd");
  if (cfg2 < 0) return -10;
  const int taps = d->kt * d->kh * d->kw;
  cudaStream_t st = (cudaStream_t)stream;
  const int sp = dw2_sp(d->c);
  const int threads = sp * d->c;
  const int t3 = cfg2 == 0 ? dw3_tile_of(d) : 0;
  if (dw != nullptr && cfg2 == 1 && dw3_s2_ok(d)) {
    Dw2Params q;
    dw2_common(q, d);
    q.dy = d->dy; q.dy_pitch = d->dy_pitch; q.dw = dw;
    cudaMemsetAsync(dw, 0, size_t(d->c_valid) * taps * sizeof(float), st);
    if (int rc = dw3_launch(7, true, q, st, 2)) return rc;
  } else if (dw != nullptr && t3) {
    Dw2Params q;
    dw2_common(q, d);
    q.dy = d->dy; q.dy_pitch = d->dy_pitch; q.dw = dw;
    cudaMemsetAsync(dw, 0, size_t(d->c_valid) * taps * sizeof(float), st);
    if (int rc = dw3_launch(dw3_tile_of(d, true), true, q, st)) return rc;
  } else if (dw != nullptr) {
    Dw2Params q;
    dw2_common(q, d);
    dw2_fwd_tiling(d->n, d->ot, d->oh, d->ow, d->c, cfg2, q);
    q.dy = d->dy; q.dy_pitch = d->dy_pitch; q.dw = dw;
    int blocks = 1;
    dw2_block_split(q, d->c, &blocks);
    cudaMemsetAsync(dw, 0, size_t(d->c_valid) * taps * sizeof(float), st);
    if (int rc = dw2_launch_wgrad(cfg2, q, blocks, threads, size_t(sp) * d->c * taps * sizeof(float), st)) return rc;
  }
  if (d->dx != nullptr || d->dx_hi != nullptr) {
    Dw2Params q;
    dw2_common(q, d);
    q.in_scale = nullptr; q.in_shift = nullptr; q.in_relu = 0;
    q.x = d->dy; q.x_pitch = d->dy_pitch;
    q.y = d->dx; q.y_hi = (bf*)d->dx_hi; q.y_lo = (bf*)d->dx_lo; q.y_pitch = d->dx_pitch;
    q.y_accumulate = d->dx_accumulate;
    if (cfg2 == 1) {
      if (d->pt != 1 || d->ph != 1 || d->pw != 1 || d->dx == nullptr) {
        set_error("sfb_dwconv_bwd: the stride-2 data gradient expects padding (1,1,1) and an fp32 output");
        return -10;
      }
      // micro-tiles over the INPUT extent: one frame x 4 x 4 positions
      q.mt_t = d->t; q.mt_h = (d->h + 3) / 4; q.mt_w = (d->w_ + 3) / 4;
      q.MT = q.mt_t * q.mt_h * q.mt_w;
      int blocks = 1;
      dw2_block_split(q, d->c, &blocks);
      dw2_dgrad_s2_kernel<<<blocks, threads, 0, st>>>(q);
      if (int rc = launch_status("sfb_dwconv_bwd (v2 stride-2 data)")) return rc;
    } else {
      // stride 1: dx = correlation of dy with the mirrored filter, padding K-1-p; "input" = dy, "output" = dx
      q.flip = 1;
      q.T = d->ot; q.H = d->oh; q.W = d->ow;
      q.oT = d->t; q.oH = d->h; q.oW = d->w_;
      q.pt = d->kt - 1 - d->pt; q.ph = d->kh - 1 - d->ph; q.pw = d->kw - 1 - d->pw;
      if (t3) {  // same extents in and out, padding 1: the ring kernel with the mirrored filter
        q.stats = nullptr;
        if (int rc = dw3_launch(t3, false, q, st)) return rc;
        return 0;
      }
      dw2_fwd_tiling(d->n, d->t, d->h, d->w_, d->c, cfg2, q);
      if (int rc = dw2_launch_conv(cfg2, q, threads, size_t(sp) * 2 * d->c * sizeof(float), st)) return rc;
    }
  }
  return 0;
}

extern "C" int sfb_bnact_fwd(const sfb_bnact_desc* d, void* stream) {
  if (int rc = bnact_check(d, "sfb_bnact_fwd")) return rc;
  BnActParams p;
  bnact_fill(p, d);
  bnact_fwd_kernel<<<x3_grid(d->rows * (d->c / 4), 256, 16), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bnact_fwd");
}
extern "C" int32_t sfb_bnact_tiles_per_sample(int64_t rows, int64_t rows_per_sample) {
  return dw_tiles_per_sample(int(rows / rows_per_sample), rows_per_sample);
}
extern "C" int sfb_bnact_bwd_reduce(const sfb_bnact_desc* d, void* stream) {
  if (int rc = bnact_check(d, "sfb_bnact_bwd_reduce")) return rc;
  BnActParams p;
  bnact_fill(p, d);
  const int n = int(d->rows / d->rows_per_sample);
  const int PL = 256 / (d->c / 4);
  bnact_bwd_reduce_kernel<<<n * p.tiles_per_sample, 256, size_t(PL) * 2 * d->c * sizeof(float),
                            (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bnact_bwd_reduce");
}
extern "C" int sfb_bnact_bwd_apply(const sfb_bnact_desc* d, void* stream) {
  if (int rc = bnact_check(d, "sfb_bnact_bwd_apply")) return rc;
  BnActParams p;
  bnact_fill(p, d);
  bnact_bwd_apply_kernel<<<x3_grid(d->rows * (d->c / 4), 256, 16), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_bnact_bwd_apply");
}
extern "C" int sfb_se_fwd(const sfb_se_desc* d, void* stream) {
  SeParams p;
  se_fill(p, d);
  se_fwd_kernel<<<d->n, 256, size_t(d->c_pad + d->f) * sizeof(float), (cudaStream_t)stream>>>(p);
  return launch_status("sfb_se_fwd");
}
extern "C" int sfb_se_bwd(const sfb_se_desc* d, void* stream) {
  SeParams p;
  se_fill(p, d);
  se_bwd_sample_kernel<<<d->n, 256, size_t(d->c_pad + d->f) * sizeof(float), (cudaStream_t)stream>>>(p);
  if (int rc = launch_status("sfb_se_bwd(sample)")) return rc;
  se_bwd_channel_kernel<<<(d->c_pad + 63) / 64, 64, 0, (cudaStream_t)stream>>>(p);
  return launch_status("sfb_se_bwd(channel)");
}
extern "C" int sfb_relu_fwd(float* x, int64_t n, void* stream) {
  relu_fwd_kernel<<<x3_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n);
  return launch_status("sfb_relu_fwd");
}
extern "C" int sfb_relu_bwd(float* dx, const float* y, int64_t n, void* stream) {
  relu_bwd_kernel<<<x3_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(dx, y, n);
  return launch_status("sfb_relu_bwd");
}
