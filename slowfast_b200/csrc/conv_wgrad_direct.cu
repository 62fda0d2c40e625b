// Weight gradient of NARROW convolutions on the fp32 pipes (the fast pathway's res2 / res3 layers: 8 -> 8 1x3x3, 8 -> 32 and
// 32 -> 8 1x1x1 / 3x1x1, 16 -> 16 1x3x3, the 7x1x1 lateral convolutions; resnet_helper.py:259 BottleneckTransform a / b / c,
// video_model_builder.py:134 FuseFastToSlow conv_f2s).
//
// As a GEMM these are dW[cout <= 32, taps*cin <= 144] reduced over 0.2 - 0.8 M positions: the wgmma kernel fills 8 - 32 of
// its 128 accumulator rows and re-reads a 128-row dY tile per 8-channel chunk; measured 237 us for the 8 -> 8 1x3x3 layer
// whose operands are 51 MB (8 us of HBM time).  Here a WARP owns one job = (tap, 8 input channels, 8 output channels):
// lane = output position, 64 register accumulators per thread, operands are 16-byte loads (coalesced 512-byte warp rows,
// re-read across the jobs of a block from L1), 18 warps per SM hide the load latency, and
// the 32 lanes are folded with a halving shuffle tree (2 atomics per lane and job).  Products are exact fp32 of
// (hi + lo) x (hi + lo): at least the precision of the three split MMA products.
//
// Same entry point, same operands, same dW layout as the tensor-core kernel (sfb_conv_wgrad); selection by shape
// (wgrad_direct_try).  sfb_set_wgrad_direct(0) keeps every layer on the tensor-core kernel, which tests use as the
// reference for this one.
#include <algorithm>
#include <cstdint>
#include <cuda_bf16.h>

#include "../../include/slowfast_b200.h"
#include "runtime.h"

namespace sfb {

constexpr int WGD_MAX_WARPS = 9;
constexpr int WGD_CHUNK = 256;   // output positions of one frame a block walks per chunk (8 groups of 32)

struct WgdParams {
  const __nv_bfloat16* x_hi; const __nv_bfloat16* x_lo; long long c_pitch;
  const __nv_bfloat16* dy_hi; const __nv_bfloat16* dy_lo; long long dy_pitch;
  float* dw;
  int nb, id, ih, iw, c, cout;
  int kd, kh, kw, dd, dh, dwl, sd, sh, sw, ld, lh, lw, oz, op, oq;
  int ktot, ci_chunks, co_chunks, jobs, jobs_per_block, slices;
  int ppf, cpf, total_chunks;   // positions per output frame, chunks per frame, frames * cpf
  int nsplit;
};

__device__ __forceinline__ void wgd_unpack(const uint4& u, float (&f)[8]) {
  f[0] = __uint_as_float(u.x << 16); f[1] = __uint_as_float(u.x & 0xffff0000u);
  f[2] = __uint_as_float(u.y << 16); f[3] = __uint_as_float(u.y & 0xffff0000u);
  f[4] = __uint_as_float(u.z << 16); f[5] = __uint_as_float(u.z & 0xffff0000u);
  f[6] = __uint_as_float(u.w << 16); f[7] = __uint_as_float(u.w & 0xffff0000u);
}

template <int NSPLIT>
__global__ void __launch_bounds__(WGD_MAX_WARPS * 32, 2) conv_wgrad_direct_kernel(const WgdParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // warp = (job of this block's group, slice of the chunk sequence): narrow job lists still fill the block with warps
  const int slice = warp / p.jobs_per_block;
  const int job = blockIdx.y * p.jobs_per_block + (warp - slice * p.jobs_per_block);
  if (job >= p.jobs) return;
  const int coc = job % p.co_chunks;
  const int cic = (job / p.co_chunks) % p.ci_chunks;
  const int tap = job / (p.co_chunks * p.ci_chunks);
  const int kwi = tap % p.kw, khi = (tap / p.kw) % p.kh, kti = tap / (p.kw * p.kh);
  const int off_t = kti * p.dd + p.ld, off_h = khi * p.dh + p.lh, off_w = kwi * p.dwl + p.lw;
  // 16-byte granule views of the operand planes (element offsets fit 32 bits: checked on the host)
  const uint4* __restrict__ xh_g = reinterpret_cast<const uint4*>(p.x_hi + cic * 8);
  const uint4* __restrict__ xl_g = reinterpret_cast<const uint4*>(p.x_lo + cic * 8);
  const uint4* __restrict__ dh_g = reinterpret_cast<const uint4*>(p.dy_hi + coc * 8);
  const uint4* __restrict__ dl_g = reinterpret_cast<const uint4*>(p.dy_lo + coc * 8);
  const int xg = int(p.c_pitch >> 3), dg = int(p.dy_pitch >> 3);   // granules per position
  const int oq = p.oq, sh = p.sh, sw = p.sw, ihn = p.ih, iwn = p.iw;

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  for (int chunk = blockIdx.x * p.slices + slice; chunk < p.total_chunks; chunk += gridDim.x * p.slices) {
    const int frame = chunk / p.cpf, sub = chunk - frame * p.cpf;
    const int n = frame / p.oz, ot = frame - n * p.oz;
    const int it = ot * p.sd + off_t;
    if (it < 0 || it >= p.id) continue;     // the whole tap plane is padding for this output frame
    const int m0 = sub * WGD_CHUNK, m1 = min(p.ppf, m0 + WGD_CHUNK);
    const int xrow0 = (n * p.id + it) * ihn;
    const int dyrow0 = frame * p.ppf;

    // this lane's position, kept as (row, column) and advanced by 32 columns per group; latency is hidden by the other
    // 17 warps of the SM (2 blocks x 9 jobs), not by a register double buffer (measured: the copy + spill traffic of one cost
    // more than it hid)
    int ml = m0 + lane;
    int oh = ml / oq, ow = ml - oh * oq;
#pragma unroll 1
    for (int mg = m0; mg < m1; mg += 32) {
      uint4 xh = make_uint4(0u, 0u, 0u, 0u), xl = xh, dh = xh, dl = xh;
      if (ml < m1) {
        const int dyo = (dyrow0 + ml) * dg;
        dh = dh_g[dyo];
        if (NSPLIT == 3) dl = dl_g[dyo];
        const int ih = oh * sh + off_h, iw = ow * sw + off_w;
        if (unsigned(ih) < unsigned(ihn) && unsigned(iw) < unsigned(iwn)) {
          const int xo = ((xrow0 + ih) * iwn + iw) * xg;
          xh = xh_g[xo];
          if (NSPLIT == 3) xl = xl_g[xo];
        }
      }
      ml += 32;
      ow += 32;
      while (ow >= oq) {
        ow -= oq;
        ++oh;
      }
      float x[8], dy[8];
      wgd_unpack(xh, x);
      wgd_unpack(dh, dy);
      if (NSPLIT == 3) {
        float a[8];
        wgd_unpack(xl, a);
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] += a[i];
        wgd_unpack(dl, a);
#pragma unroll
        for (int i = 0; i < 8; ++i) dy[i] += a[i];
      }
#pragma unroll
      for (int ci = 0; ci < 8; ++ci)
#pragma unroll
        for (int co = 0; co < 8; ++co) acc[ci * 8 + co] = fmaf(x[ci], dy[co], acc[ci * 8 + co]);
    }
  }
  const int ci0 = cic * 8, co0 = coc * 8;

  // fold the 32 lanes: each round halves the live values, lanes with the partner bit set keep the upper half
#pragma unroll
  for (int o = 16, nv = 64; o >= 1; o >>= 1, nv >>= 1) {
    const bool up = (lane & o) != 0;
    const int half = nv >> 1;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i < half) {
        const float send = up ? acc[i] : acc[i + half];
        const float keep = up ? acc[i + half] : acc[i];
        acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    }
  }
  // lane L now holds elements idx = bits(L4 L3 L2 L1 L0 i) of the 64, idx = ci*8 + co
  const int base = (((lane >> 4) & 1) << 5) | (((lane >> 3) & 1) << 4) | (((lane >> 2) & 1) << 3) |
                   (((lane >> 1) & 1) << 2) | ((lane & 1) << 1);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = base + i;
    const int ci = idx >> 3, co = idx & 7;
    if (ci0 + ci < p.c && co0 + co < p.cout)
      atomicAdd(p.dw + static_cast<long long>(co0 + co) * p.ktot + tap * p.c + ci0 + ci, acc[i]);
  }
}

static int g_wgd_enabled = 1;

void wgrad_direct_configure(int enabled) { g_wgd_enabled = enabled; }

// Whether the direct kernel takes the job: narrow layers with many positions only (at most 8 channels on one side, at
// most 14 (tap, 8 x 8 channel block) jobs); wider layers fill the tensor-core kernel's tiles.
bool wgrad_direct_takes(const sfb_wgrad_desc* d) {
  if (!g_wgd_enabled) return false;
  const int taps = d->kt * d->kh * d->kw;
  const int64_t M = int64_t(d->n) * d->out_t * d->out_h * d->out_w;
  const int jobs = taps * (d->c / 8) * (d->cout / 8);
  if (d->c * d->cout > 256 || std::min(d->c, d->cout) > 8 || jobs > 14 || M < 32768) return false;
  return int64_t(d->n) * d->d * d->h * d->w * d->c_pitch < (int64_t(1) << 31) && M * d->dy_pitch < (int64_t(1) << 31);
}

// Returns 1 and sets *rc_out when the direct kernel took the job; `sms` is the device's SM count.
int wgrad_direct_try(const sfb_wgrad_desc* d, int sms, cudaStream_t stream, int* rc_out) {
  if (!wgrad_direct_takes(d)) return 0;
  const int taps = d->kt * d->kh * d->kw;
  const int jobs = taps * (d->c / 8) * (d->cout / 8);
  WgdParams p;
  p.x_hi = (const __nv_bfloat16*)d->x_hi; p.x_lo = (const __nv_bfloat16*)d->x_lo; p.c_pitch = d->c_pitch;
  p.dy_hi = (const __nv_bfloat16*)d->dy_hi; p.dy_lo = (const __nv_bfloat16*)d->dy_lo; p.dy_pitch = d->dy_pitch;
  p.dw = d->dw;
  p.nb = d->n; p.id = d->d; p.ih = d->h; p.iw = d->w; p.c = d->c; p.cout = d->cout;
  p.kd = d->kt; p.kh = d->kh; p.kw = d->kw; p.dd = d->dil_t; p.dh = d->dil_h; p.dwl = d->dil_w;
  p.sd = d->str_t; p.sh = d->str_h; p.sw = d->str_w; p.ld = d->low_t; p.lh = d->low_h; p.lw = d->low_w;
  p.oz = d->out_t; p.op = d->out_h; p.oq = d->out_w;
  p.ktot = taps * d->c;
  p.ci_chunks = d->c / 8; p.co_chunks = d->cout / 8;
  p.jobs = jobs;
  const int groups = (jobs + WGD_MAX_WARPS - 1) / WGD_MAX_WARPS;
  p.jobs_per_block = (jobs + groups - 1) / groups;
  p.ppf = d->out_h * d->out_w;
  p.cpf = (p.ppf + WGD_CHUNK - 1) / WGD_CHUNK;
  p.total_chunks = d->n * d->out_t * p.cpf;
  p.nsplit = d->nsplit;
  p.slices = std::max(1, WGD_MAX_WARPS / p.jobs_per_block);
  const int wpb = p.jobs_per_block * p.slices;                       // warps per block
  const int blocks_per_sm = std::max(2, 20 / wpb);                   // 96 registers per thread: ~21 warps fit an SM
  const int gx = std::max(1, std::min((p.total_chunks + p.slices - 1) / p.slices,
                                      (blocks_per_sm * sms + groups - 1) / groups));
  dim3 grid(gx, groups);
  const int threads = wpb * 32;
  if (d->nsplit == 3)
    conv_wgrad_direct_kernel<3><<<grid, threads, 0, stream>>>(p);
  else
    conv_wgrad_direct_kernel<1><<<grid, threads, 0, stream>>>(p);
  *rc_out = launch_status("sfb_conv_wgrad (direct)");
  return 1;
}

}  // namespace sfb

extern "C" int sfb_set_wgrad_direct(int32_t enabled) {
  sfb::wgrad_direct_configure(enabled);
  return 0;
}
