// Direct (fp32 SIMT) convolution for SMALL channel counts - an alternative body of sfb_conv_igemm (same descriptor,
// same packed filter planes, same output view and BatchNorm-partial layout), selected by sfb_conv_igemm when
// SFB_SIMT_SMALLC=1 and the layer is narrow.
//
// Why: the fast pathway's first stages (8..32 channels, 0.8 M pixels per layer) are bound by the TMA unit's per-pixel
// request rate on the tensor-core path (profiles/r1c_conv_igemm_notes.md: 113 us for 128 MB), while their arithmetic is
// tiny (<= 3 K MAC per pixel).  Here one thread owns one output pixel: it streams the pixel's input channels (16 B per
// plane and 8 channels, consecutive lanes = consecutive pixels: contiguous 512-byte warp loads for the tap-free case),
// multiplies with the filter staged in shared memory as fp32 (hi + lo planes re-joined, [k][cout] so that one LDS.128
// feeds 4 output channels, broadcast across the warp) and writes its fp32 output row.  One block = 128 pixels = one
// "m-tile", so the per-tile BatchNorm partials have exactly the layout the tensor-core kernel produces.
//
// Selection: sfb_set_simt_smallc(enabled, max_macs) at run time (tests / A-B probes), initial value from the environment
// (SFB_SIMT_SMALLC = 0 | 1, SFB_SIMT_MAX_MACS); layers with C_in, C_out <= 64 and taps*C_in*C_out <= max_macs take this body.
#include <cstdint>
#include <cstdlib>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "tmap.h"

// shipped default of the switch
#ifndef SFB_SIMT_DEFAULT
#define SFB_SIMT_DEFAULT 1
#endif

namespace sfb {

struct DirectParams {
  const __nv_bfloat16* a_hi; const __nv_bfloat16* a_lo; int64_t c_pitch;
  const __nv_bfloat16* b_hi; const __nv_bfloat16* b_lo;
  int nb, id, ih, iw, c, cout;
  int kd, kh, kw, dd, dh, dw, sd, sh, sw, ld, lh, lw, oz, op, oq;
  int M, m_tiles, ktot, coutp;  // coutp = COUT_T (register tile width)
  float* out; long long os_n, os_z, os_p, os_q; int accumulate; int ncols_store;
  float* stats;
};

__device__ __forceinline__ void dc_load8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t off, float (&x)[8]) {
  const uint4 h = *reinterpret_cast<const uint4*>(hi + off);
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[2 * i] = __uint_as_float(hw[i] << 16);
    x[2 * i + 1] = __uint_as_float(hw[i] & 0xffff0000u);
  }
  if (lo) {
    const uint4 l = *reinterpret_cast<const uint4*>(lo + off);
    const uint32_t lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      x[2 * i] += __uint_as_float(lw[i] << 16);
      x[2 * i + 1] += __uint_as_float(lw[i] & 0xffff0000u);
    }
  }
}

template <int COUT_T>
__global__ void __launch_bounds__(128) conv_direct_kernel(const DirectParams p) {
  extern __shared__ __align__(16) float wsm[];  // [ktot][COUT_T] fp32 filter, [4 warps][2][COUT_T] reduction scratch, out tile
  float* red = wsm + size_t(p.ktot) * COUT_T;
  // ---- stage the filter: B[co][k] planes -> wsm[k][co] (zero for co >= cout)
  for (int i = threadIdx.x; i < p.ktot * COUT_T; i += blockDim.x) {
    const int k = i / COUT_T, co = i - k * COUT_T;
    float v = 0.f;
    if (co < p.cout) {
      v = __bfloat162float(p.b_hi[size_t(co) * p.ktot + k]);
      if (p.b_lo) v += __bfloat162float(p.b_lo[size_t(co) * p.ktot + k]);
    }
    wsm[i] = v;
  }
  __syncthreads();
  const int mt = blockIdx.x;
  const int row = mt * 128 + threadIdx.x;
  const bool rvalid = row < p.M;
  float acc[COUT_T];
#pragma unroll
  for (int j = 0; j < COUT_T; ++j) acc[j] = 0.f;
  long long roff = 0;
  if (rvalid) {
    int t = row;
    const int oq_ = t % p.oq;
    t /= p.oq;
    const int op_ = t % p.op;
    t /= p.op;
    const int oz_ = t % p.oz;
    const int on_ = t / p.oz;
    roff = on_ * p.os_n + oz_ * p.os_z + op_ * p.os_p + oq_ * p.os_q;
    const int w0 = p.lw + oq_ * p.sw, h0 = p.lh + op_ * p.sh, d0 = p.ld + oz_ * p.sd;
    int tap = 0;
    for (int td = 0; td < p.kd; ++td) {
      const int id = d0 + td * p.dd;
      for (int th = 0; th < p.kh; ++th) {
        const int ih = h0 + th * p.dh;
        for (int tw = 0; tw < p.kw; ++tw, ++tap) {
          const int iw = w0 + tw * p.dw;
          if (id < 0 || id >= p.id || ih < 0 || ih >= p.ih || iw < 0 || iw >= p.iw) continue;  // zero padding
          const int64_t base = (((int64_t(on_) * p.id + id) * p.ih + ih) * p.iw + iw) * p.c_pitch;
          const float* wt = wsm + size_t(tap) * p.c * COUT_T;
          for (int c0 = 0; c0 < p.c; c0 += 8) {
            float x[8];
            dc_load8(p.a_hi, p.a_lo, base + c0, x);
#pragma unroll
            for (int ci = 0; ci < 8; ++ci) {
              const float xv = x[ci];
              const float4* w4 = reinterpret_cast<const float4*>(wt + size_t(c0 + ci) * COUT_T);
#pragma unroll
              for (int j = 0; j < COUT_T / 4; ++j) {
                const float4 w = w4[j];
                acc[4 * j + 0] = fmaf(xv, w.x, acc[4 * j + 0]);
                acc[4 * j + 1] = fmaf(xv, w.y, acc[4 * j + 1]);
                acc[4 * j + 2] = fmaf(xv, w.z, acc[4 * j + 2]);
                acc[4 * j + 3] = fmaf(xv, w.w, acc[4 * j + 3]);
              }
            }
          }
        }
      }
    }
  }
  // ---- output: staged through shared memory so that consecutive lanes store consecutive floats of a pixel's row (one
  //      128-byte line per warp store for 32 output channels) instead of one 16-byte piece of 32 different rows
  float* tile = red + 8 * COUT_T;                       // [128][COUT_T + 1]
  long long* roff_s = reinterpret_cast<long long*>(tile + 128 * (COUT_T + 1));
#pragma unroll
  for (int j = 0; j < COUT_T; ++j) tile[threadIdx.x * (COUT_T + 1) + j] = acc[j];
  roff_s[threadIdx.x] = rvalid ? roff : -1;
  __syncthreads();
  {
    const int ncols = p.ncols_store;
    for (int e = threadIdx.x; e < 128 * ncols; e += 128) {
      int px, col;
      if (ncols == COUT_T) {
        px = e / COUT_T;
        col = e - px * COUT_T;
      } else {
        px = e / ncols;
        col = e - px * ncols;
      }
      const long long off = roff_s[px];
      if (off < 0) continue;
      float v = tile[px * (COUT_T + 1) + col];
      float* dst = p.out + off + col;
      if (p.accumulate == 2) {
        atomicAdd(dst, v);               // result unused: RED, no dependent load
      } else {
        if (p.accumulate) v += *dst;
        *dst = v;
      }
    }
  }
  if (p.stats == nullptr) return;
  // ---- BatchNorm partials of this 128-pixel tile: warp shuffles, then the four warps through shared memory
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < COUT_T; ++j) {
    float s = rvalid ? acc[j] : 0.f;
    float s2 = s * s;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
      red[(warp * 2 + 0) * COUT_T + j] = s;
      red[(warp * 2 + 1) * COUT_T + j] = s2;
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < p.cout; j += blockDim.x) {
    float s = 0.f, s2 = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      s += red[(w * 2 + 0) * COUT_T + j];
      s2 += red[(w * 2 + 1) * COUT_T + j];
    }
    p.stats[size_t(j) * p.m_tiles + mt] = s;
    p.stats[(size_t(p.cout) + j) * p.m_tiles + mt] = s2;
  }
}

// 1 = handled here (rc in *rc_out), 0 = not eligible: the caller continues with the tensor-core path
static int g_simt_enabled = [] { const char* e = getenv("SFB_SIMT_SMALLC"); return e ? int(e[0] == '1') : SFB_SIMT_DEFAULT; }();
// the fp32 body is meant for layers where ONE pixel is a 16-byte TMA request (C_in = 8); from C_in = 16 on the tensor-core
// body streams its operands at full rate, so the limit is C_in <= 8 and <= 1024 MAC per pixel (tests/probes/smallc_probe.py
// compares the two)
static int g_simt_max_macs = [] { const char* e = getenv("SFB_SIMT_MAX_MACS"); return e ? atoi(e) : 1024; }();
static int g_simt_max_cin = [] { const char* e = getenv("SFB_SIMT_MAX_CIN"); return e ? atoi(e) : 8; }();

void conv_direct_configure(int enabled, int max_macs) {
  g_simt_enabled = enabled;
  if (max_macs > 0) g_simt_max_macs = max_macs;
}

int conv_direct_try(const sfb_conv_desc* d, cudaStream_t stream, int* rc_out) {
  if (!g_simt_enabled) return 0;
  const int taps = d->kt * d->kh * d->kw;
  const int64_t macs = int64_t(taps) * d->c * d->cout;
  int coutp = 8;
  while (coutp < d->cout) coutp <<= 1;
  const size_t smem = (size_t(taps) * d->c * coutp + size_t(8) * coutp + size_t(128) * (coutp + 1)) * sizeof(float) +
                      128 * sizeof(long long) + 8;
  if (d->c > 64 || d->cout > 64 || macs > g_simt_max_macs || smem > 96 * 1024) return 0;
  if (d->c > g_simt_max_cin && g_simt_max_macs <= 4096) return 0;  // (probe runs lift both limits through max_macs)
  DirectParams p;
  p.a_hi = (const __nv_bfloat16*)d->a_hi; p.a_lo = (const __nv_bfloat16*)d->a_lo; p.c_pitch = d->c_pitch;
  p.b_hi = (const __nv_bfloat16*)d->b_hi; p.b_lo = (const __nv_bfloat16*)d->b_lo;
  p.nb = d->n; p.id = d->d; p.ih = d->h; p.iw = d->w; p.c = d->c; p.cout = d->cout;
  p.kd = d->kt; p.kh = d->kh; p.kw = d->kw; p.dd = d->dil_t; p.dh = d->dil_h; p.dw = d->dil_w;
  p.sd = d->str_t; p.sh = d->str_h; p.sw = d->str_w; p.ld = d->low_t; p.lh = d->low_h; p.lw = d->low_w;
  p.oz = d->out_t; p.op = d->out_h; p.oq = d->out_w;
  p.M = int(int64_t(d->n) * d->out_t * d->out_h * d->out_w);
  p.m_tiles = (p.M + 127) / 128;
  p.ktot = taps * d->c;
  p.coutp = coutp;
  p.out = d->out; p.os_n = d->os_n; p.os_z = d->os_t; p.os_p = d->os_h; p.os_q = d->os_w;
  p.accumulate = d->accumulate;
  p.ncols_store = (d->cout + 3) & ~3;
  p.stats = d->stats;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(conv_direct_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(conv_direct_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(conv_direct_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(conv_direct_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    attr = true;
  }
  switch (coutp) {
    case 8: conv_direct_kernel<8><<<p.m_tiles, 128, smem, stream>>>(p); break;
    case 16: conv_direct_kernel<16><<<p.m_tiles, 128, smem, stream>>>(p); break;
    case 32: conv_direct_kernel<32><<<p.m_tiles, 128, smem, stream>>>(p); break;
    default: conv_direct_kernel<64><<<p.m_tiles, 128, smem, stream>>>(p); break;
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("sfb_conv_igemm (direct SIMT body) launch failed: %s", cudaGetErrorString(e));
    *rc_out = -20;
  } else {
    *rc_out = 0;
  }
  return 1;
}

}  // namespace sfb

extern "C" int sfb_set_simt_smallc(int32_t enabled, int32_t max_macs) {
  sfb::conv_direct_configure(enabled, max_macs);
  return 0;
}
