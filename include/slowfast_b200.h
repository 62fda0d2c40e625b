/*
 * slowfast_b200 — C ABI of the H100-native video-backbone engine.
 *
 * Drop-in boundary: the reference (facebookresearch/SlowFast) has no native layer; every FLOP of
 * `model(inputs)` / `loss.backward()` behind `slowfast.models.build_model` (slowfast/models/build.py:22)
 * is an ATen operator call.  This header declares what a reference-side binding would call instead of
 * those operator call sites (SURVEY.md §2b / §8b).  All entry points:
 *   - take raw device pointers + plain-old-data descriptors (no torch types),
 *   - enqueue work on the CUDA stream passed as `void* stream` (a cudaStream_t) and never synchronise,
 *   - borrow every pointer for the duration of the call only (owner = the caller's allocator),
 *   - return 0 on success, <0 on error; sfb_last_error() returns the message (thread-local).
 *
 * Activation layout: channels-last NDHWC ("N, T, H, W, C").  Tensor-core operands are carried as TWO bf16
 * planes (hi = bf16(x), lo = bf16(x - hi)) so that the 3-term split product hi*hi + hi*lo + lo*hi reproduces
 * fp32 operand precision (parity mode, nsplit = 3); the fast mode uses the hi plane only (nsplit = 1).
 */
#ifndef SLOWFAST_B200_H_
#define SLOWFAST_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* sfb_last_error(void);
/* Library/ABI version and build arch string, e.g. "sm_90a". */
int sfb_abi_version(void);
const char* sfb_build_arch(void);

/* ------------------------------------------------------------------------------------------------
 * Implicit-GEMM 3-D convolution on wgmma tensor cores, TMA im2col operand staging.
 * Replaces nn.Conv3d fprop (resnet_helper.py:332,346,362,485; stem_helper.py:182;
 * video_model_builder.py:147) and, with a transposed/flipped filter matrix and an output view, the
 * autograd dgrad of the same layers (SURVEY.md row a21).  nn.Linear (attention.py:193,195; common.py:20,22;
 * head_helper.py) is the kt=kh=kw=1 case.
 *
 *   out[n, z, p, q, co] (+)= sum_{tap, ci} A[n, low_t + z*str_t + it*dil_t, low_h + ..., low_w + ..., ci]
 *                                          * B[co, tap, ci]            (out-of-range A reads as 0)
 * ---------------------------------------------------------------------------------------------- */
typedef struct sfb_conv_desc {
  /* A operand: activation planes, channels-last [n, d, h, w, c], channel pitch c_pitch >= c */
  const void* a_hi;
  const void* a_lo; /* may be NULL when nsplit == 1 */
  int32_t n, d, h, w, c;
  int64_t c_pitch;
  /* B operand: filter matrix planes, bf16 [cout, kt*kh*kw*c], K index = ((it*kh + ih)*kw + iw)*c + ci */
  const void* b_hi;
  const void* b_lo; /* may be NULL when nsplit == 1 */
  int32_t cout;
  int32_t kt, kh, kw;
  int32_t dil_t, dil_h, dil_w;
  int32_t str_t, str_h, str_w;
  int32_t low_t, low_h, low_w; /* input coordinate of tap 0 for output index 0 (= -padding for fprop) */
  int32_t out_t, out_h, out_w; /* output grid */
  /* output view: fp32, channel stride 1, element strides for (n, t, h, w) */
  float* out;
  int64_t os_n, os_t, os_h, os_w;
  int32_t accumulate; /* 0: out = result, 1: out += result (read-modify-write), 2: out += result with red.global.add (each
                         element gets one add per call: same sums, no dependent load) */
  /* optional per-tile BatchNorm partials: [2][cout][m_tiles] = (sum, sum of squares) over each tile's rows */
  float* stats;
  int32_t nsplit; /* 1 (bf16 operands) or 3 (split-bf16, fp32-class operands) */
} sfb_conv_desc;

/* Number of 128-row output tiles (last extent of `stats`). */
int64_t sfb_conv_m_tiles(const sfb_conv_desc* d);
int sfb_conv_igemm(const sfb_conv_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Convolution weight gradient (autograd wgrad of nn.Conv3d / nn.Linear, SURVEY.md row a21).
 *   dw[co, (tap, ci)] += sum over output positions m of  dY[m, co] * X[input position of (m, tap), ci]
 * dw is fp32 in the SAME [cout, kt*kh*kw*c] matrix layout as the fprop filter matrix and must be zero-filled
 * (or hold a running sum) by the caller; split-K partials are combined with fp32 reductions.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sfb_wgrad_desc {
  const void* x_hi;
  const void* x_lo; /* forward input planes, channels-last [n, d, h, w, c], pitch c_pitch */
  int32_t n, d, h, w, c;
  int64_t c_pitch;
  const void* dy_hi;
  const void* dy_lo; /* output-gradient planes, dense [n*out_t*out_h*out_w, cout] with row pitch dy_pitch */
  int32_t cout;
  int64_t dy_pitch;
  int32_t kt, kh, kw;
  int32_t dil_t, dil_h, dil_w;
  int32_t str_t, str_h, str_w;
  int32_t low_t, low_h, low_w;
  int32_t out_t, out_h, out_w;
  float* dw;
  int32_t nsplit;
} sfb_wgrad_desc;

int sfb_conv_wgrad(const sfb_wgrad_desc* d, void* stream);
/* Layers with c*cout <= 512 and >= 32768 output positions (the fast pathway's narrow stages) take an fp32 SIMT body inside
 * sfb_conv_wgrad (csrc/conv_wgrad_direct.cu); enabled = 0 keeps every layer on the tensor-core kernel (A/B tests). */
int sfb_set_wgrad_direct(int32_t enabled);

/* Zero-fill a [rows, c] fp32 view (row pitch in elements) on the stream (gradient accumulators). */
int sfb_zero_f32_2d(float* ptr, int64_t rows, int64_t c, int64_t pitch, void* stream);

/* dst[rows, c] += src[rows, c] on fp32 views (row pitches in elements): merges a further contribution into an
 * activation gradient. */
int sfb_add_f32_2d(float* dst, const float* src, int64_t rows, int32_t c, int64_t dst_pitch, int64_t src_pitch,
                   void* stream);

/* ------------------------------------------------------------------------------------------------
 * Operand packing.
 * ---------------------------------------------------------------------------------------------- */
/* fp32 [rows, c] (row pitch x_pitch) -> split-bf16 planes (row pitch o_pitch); lo may be NULL. */
int sfb_split_planes(const float* x, int64_t rows, int32_t c, int64_t x_pitch, void* hi, void* lo,
                     int64_t o_pitch, void* stream);
/* Model input: NCDHW fp32 clip (what train_net.py:79-98 puts on the device) -> NDHWC planes, channels padded
 * with zeros to c_pad (multiple of 8, for the 16-byte TMA granule). */
int sfb_input_pack(const float* x, int32_t n, int32_t c, int32_t t, int32_t h, int32_t w, int32_t c_pad, void* hi,
                   void* lo, void* stream);
/* nn.Conv3d weight [cout, cin, kt, kh, kw] (fp32) -> GEMM filter matrix planes.
 *   transpose = 0: out[co][j][ci]  (fprop B operand; also the layout of the wgrad result)
 *   transpose = 1: out[ci][j][co]  (dgrad B operand)
 * j runs over ntaps selected source taps tapmap[j] (NULL = identity), taps_total = kt*kh*kw,
 * cols_pad >= inner channel count (zero padded). */
int sfb_filter_pack(const float* w, int32_t cout, int32_t cin, int32_t taps_total, const int32_t* tapmap,
                    int32_t ntaps, int32_t transpose, int32_t cols_pad, void* hi, void* lo, void* stream);
/* The same packing for MANY filters in one launch (one per phase of a step instead of one per layer).  `jobs_device`
 * is an array in DEVICE memory, sorted by first_block; job k owns grid blocks [first_block, first_block + n_blocks).
 * ntaps <= 32 (larger tap counts - the stems - keep using sfb_filter_pack). */
typedef struct sfb_pack_job {
  const float* w; void* hi; void* lo;
  int32_t cout, cin, taps_total, ntaps, transpose, cols_pad;
  int32_t first_block, n_blocks;
  int16_t tapmap[32];
} sfb_pack_job;
int32_t sfb_pack_job_size(void);
int sfb_filter_pack_multi(const sfb_pack_job* jobs_device, int32_t njobs, int32_t total_blocks, void* stream);
/* wgrad matrix [cout][taps][cin_pad] fp32 -> parameter-gradient layout [cout][cin][taps] (= or +=). */
int sfb_filter_unpack_grad(const float* dwm, float* dw, int32_t cout, int32_t cin, int32_t taps, int32_t cin_pad,
                           int32_t accumulate, void* stream);

/* ------------------------------------------------------------------------------------------------
 * BatchNorm3d (batchnorm_helper.py:16 -> nn.BatchNorm3d; resnet_helper.py:340,356,372,494; stem_helper.py:190).
 * Train mode: statistics come from the conv epilogue partials; finalize merges them (fp64), updates the running
 * statistics with torch's rule (momentum, unbiased variance) and emits scale/shift for the apply kernel.
 * ---------------------------------------------------------------------------------------------- */
int sfb_bn_finalize(const float* partials, int32_t m_tiles, int32_t c, int64_t count, const float* gamma,
                    const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                    int32_t training, float* scale, float* shift, float* save_mean, float* save_invstd,
                    void* stream);

/* out = act( y*scale + shift [+ y2*scale2 + shift2] [+ residual planes] ) written as split planes.
 * Covers BN+ReLU (a_bn/b_bn), the block tail relu(x + c_bn(..)) and relu(branch1_bn(..) + c_bn(..))
 * (resnet_helper.py:512-521), and FuseFastToSlow's BN+ReLU written into the concat slice
 * (video_model_builder.py:162-169). */
typedef struct sfb_bn_apply_desc {
  const float* y; int64_t y_pitch; const float* scale; const float* shift;
  const float* y2; int64_t y2_pitch; const float* scale2; const float* shift2; /* optional second BN branch */
  const void* res_hi; const void* res_lo; int64_t res_pitch;                    /* optional identity residual */
  void* out_hi; void* out_lo; int64_t out_pitch;
  int64_t rows; int32_t c; int32_t relu;
} sfb_bn_apply_desc;
int sfb_bn_apply(const sfb_bn_apply_desc* d, void* stream);

/* Backward of (BN -> [ReLU]) given dout = gradient w.r.t. the post-activation output:
 *   dz = dout * (mask > 0);  dgamma = sum dz*xhat;  dbeta = sum dz;
 *   dy = gamma*invstd * (dz - mean(dz) - xhat*mean(dz*xhat))   -> split planes (GEMM operands of dgrad/wgrad)
 * Optionally emits dz (fp32) as the gradient of an identity shortcut (dres). */
typedef struct sfb_bn_bwd_desc {
  const float* dout; int64_t dout_pitch;
  const void* mask_hi; int64_t mask_pitch; /* post-ReLU output plane, NULL when no ReLU follows */
  const float* y; int64_t y_pitch;         /* conv output saved by forward */
  const float* mean; const float* invstd; const float* gamma;
  float* dgamma; float* dbeta; int32_t accumulate_param_grads;
  int32_t training;
  void* dy_hi; void* dy_lo; int64_t dy_pitch;
  float* dres; int64_t dres_pitch; int32_t dres_accumulate;
  float* partials; /* scratch [sfb_bn_bwd_blocks(rows,c)][2][c] */
  float* coef;     /* scratch [3][c] */
  int64_t rows; int32_t c;
  int32_t c_valid; /* channels >= c_valid (> 0) are padding: zero coefficients, no parameter-gradient writes */
  /* alternative to mask_hi when the post-ReLU planes were never materialised (X3D: fused into the channelwise conv):
   * the ReLU mask is recomputed as y*mask_scale + mask_shift > 0 (the forward BN affine) */
  const float* mask_scale; const float* mask_shift;
} sfb_bn_bwd_desc;
int32_t sfb_bn_bwd_blocks(int64_t rows, int32_t c);
int sfb_bn_bwd(const sfb_bn_bwd_desc* d, void* stream);

/* Stem tail: BN -> ReLU -> MaxPool3d [1,kh,kw] stride [1,sh,sw] pad [0,ph,pw] (stem_helper.py:190-201), fused;
 * y is the dense conv output [n,t,h,w,c]; argmax [n,t,oh,ow,c] (uint8) is saved for the backward gather. */
typedef struct sfb_pool_desc {
  const float* y; const float* scale; const float* shift;
  int32_t n, t, h, w, c, oh, ow, kh, kw, sh, sw, ph, pw;
  void* out_hi; void* out_lo; int64_t out_pitch;
  uint8_t* argmax;
  const float* dout; int64_t dout_pitch; /* backward: gradient w.r.t. the pooled output */
  float* dz;                              /* backward: gradient w.r.t. relu(bn(y)), dense [n,t,h,w,c] */
} sfb_pool_desc;
int sfb_bn_relu_maxpool_fwd(const sfb_pool_desc* d, void* stream);
int sfb_bn_relu_maxpool_bwd(const sfb_pool_desc* d, void* stream);



/* MaxPool3d over a split-bf16 activation [n,t,h,w,c] -> [n,ot,oh,ow,c] (pathway pools of the C2D/I3D archs,
 * video_model_builder.py:543-549; MViT pool_skip, attention.py:486).  First maximum wins; argmax (uint8 window
 * index) [n,ot,oh,ow,c] is saved; bwd gathers dout (fp32, pooled shape) into din (fp32, input shape; = or +=). */
typedef struct sfb_pool3d_desc {
  const void* in_hi; const void* in_lo; int64_t in_pitch;
  void* out_hi; void* out_lo; int64_t out_pitch;
  uint8_t* argmax;
  int32_t n, t, h, w, c, ot, oh, ow;
  int32_t kt, kh, kw, st, sh, sw, pt, ph, pw;
  const float* dout; int64_t dout_pitch;
  float* din; int64_t din_pitch; int32_t din_accumulate;
} sfb_pool3d_desc;
int sfb_maxpool3d_fwd(const sfb_pool3d_desc* d, void* stream);
int sfb_maxpool3d_bwd(const sfb_pool3d_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Stem convolutions with C_in <= 4 and W stride 2 (stem_helper.py:182 ResNetBasicStem conv, :258 X3DStem conv_xy):
 * "W-shift" implicit GEMM - the clip is packed with W folded by the stride (one pixel pair = one 16-byte granule)
 * and all W taps of a (kt, kh) pair are read from ONE shared-memory segment through shifted UMMA descriptors.
 * No dgrad (the clip needs no gradient).
 * ---------------------------------------------------------------------------------------------- */
/* NCDHW fp32 clip -> folded planes [n, t, h, w/2, 8], channel = parity*cin + c. */
int sfb_stem_input_fold(const float* x, int32_t n, int32_t cin, int32_t t, int32_t h, int32_t w, void* hi, void* lo,
                        void* stream);
/* weight [cout][cin][kt][kh][kw] <-> folded filter matrix [cout][kt][kh][kwf][8]:
 *   reverse = 0: pack planes (hi, lo) from w;  reverse = 1: scatter the fp32 gradient matrix gmat into dw. */
int sfb_stem_filter_fold(const float* w, float* dw, int32_t cout, int32_t cin, int32_t kt, int32_t kh, int32_t kw,
                         int32_t pad_w, int32_t kwf, void* hi, void* lo, const float* gmat, int32_t reverse,
                         void* stream);
typedef struct sfb_stem_desc {
  const void* x_hi; const void* x_lo; /* folded clip planes [n, t, h, wf, 8] */
  int32_t n, t, h, wf;
  const void* f_hi; const void* f_lo;   /* fprop: folded filter matrix planes [cout, kt*kh*kwf*8] */
  const void* dy_hi; const void* dy_lo; /* wgrad: output-gradient planes, dense [n, out_t, out_h, out_w, cout] */
  int32_t cout, kt, kh, kwf;
  int32_t str_t, str_h, pad_t, pad_h, pad_wf; /* pad_wf = left padding in folded W coordinates */
  int32_t out_t, out_h, out_w;
  float* out;   /* fprop: fp32 dense [n, out_t, out_h, out_w, cout] */
  float* stats; /* fprop: optional BN partials [2][cout][sfb_stem_m_tiles()] */
  float* dwm;   /* wgrad: fp32 [cout, kt*kh*kwf*8], zero-filled by the caller */
  int32_t nsplit;
} sfb_stem_desc;
int64_t sfb_stem_m_tiles(const sfb_stem_desc* d);
int sfb_stem_fprop(const sfb_stem_desc* d, void* stream);
int sfb_stem_wgrad(const sfb_stem_desc* d, void* stream);
/* The fast pathway's stem (stem_helper.py:182 with dim_out = 8: Conv3d 3 -> 8, [kt,7,7], stride (1,2,2), pad (kt/2,3,3);
 * video_model_builder.py:219 SlowFast s1) as a "Toeplitz" implicit GEMM: one GEMM row = 8 consecutive output pixels, so the
 * MMA is 128 x 64 x 16 instead of 128 x 8 x 16 (csrc/conv_stem8.cu).  Same descriptor; differences:
 *   x_hi / x_lo : planes [n][2t + (h&1)][h/2][8][MR][8] written by sfb_stem8_input_fold, MR = out_w/8 + 1, wf = 8*MR
 *   f_hi / f_lo : planes [kt][92][8][8] written by sfb_stem8_filter_fold
 *   stats       : [2][8][sfb_stem8_m_tiles()]
 *   dwm         : the W-shift gradient matrix [8, kt*7*4*8] (zero-filled by the caller; unfold with sfb_stem_filter_fold). */
int sfb_stem8_supported(const sfb_stem_desc* d);
int64_t sfb_stem8_m_tiles(const sfb_stem_desc* d);
int sfb_stem8_input_fold(const float* x, int32_t n, int32_t cin, int32_t t, int32_t h, int32_t w, void* hi, void* lo,
                         void* stream);
int sfb_stem8_filter_fold(const float* w, int32_t cin, int32_t kt, void* hi, void* lo, void* stream);
int sfb_stem8_fprop(const sfb_stem_desc* d, void* stream);
int sfb_stem8_wgrad(const sfb_stem_desc* d, void* stream);
/* Direct (fp32 SIMT) weight gradient of the narrow stem (3 -> 8 channels, stride (1,2,2): the fast pathway's
 * conv, stem_helper.py:182): reads the fp32 NCTHW clip and the dY planes, writes dw in the parameter's own layout
 * [8][3][kt][kh][kw].  8 output channels would fill 8 of 128 UMMA rows; the fp32 pipes do this layer faster. */
int sfb_stem_wgrad_direct(const float* x, int32_t n, int32_t cin, int32_t t, int32_t h, int32_t w, const void* dy_hi,
                          const void* dy_lo, int32_t cout, int32_t kt, int32_t kh, int32_t kw, int32_t st, int32_t sh,
                          int32_t sw, int32_t pt, int32_t ph, int32_t pw, float* dw, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Batched GEMM for the attention products of MultiScaleAttention (attention.py:355 `(q*scale) @ k^T`, :379
 * `attn @ v`) and their autograd transposes:  out[b](m,n) (+)= alpha * sum_k A[b](m,k) * B[b](n,k).
 * An operand is K-major (memory [b][rows][K], pitch ld, K contiguous) or MN-major (memory [b][K][rows], rows
 * contiguous) - no transpose copies.  Pitches and batch strides in elements, multiples of 8.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sfb_bgemm_desc {
  const void* a_hi; const void* a_lo; int64_t lda, batch_stride_a; int32_t a_mn_major;
  const void* b_hi; const void* b_lo; int64_t ldb, batch_stride_b; int32_t b_mn_major;
  int32_t m, n, k, batch;
  float* out; int64_t ldd, batch_stride_d;
  float alpha;
  int32_t accumulate;
  int32_t nsplit;
} sfb_bgemm_desc;
int sfb_gemm_batched(const sfb_bgemm_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MViT token-path kernels (attention.py attention_pool :13, cal_rel_pos_* :64/:111, MultiScaleAttention.forward
 * :293, MultiScaleBlock.forward :491; common.py Mlp :26; stem_helper.py PatchEmbed :315).  Tokens are
 * [B, N = 1 + T*H*W, C] fp32 with the cls token first; GEMM operands are split-bf16 planes.
 * ---------------------------------------------------------------------------------------------- */
/* nn.LayerNorm(eps) over the last dim (C <= 768): planes and/or fp32 output, saves mean / rstd per row. */
int sfb_layernorm_fwd(const float* x, int64_t x_pitch, int64_t rows, int32_t c, const float* gamma, const float* beta,
                      float eps, void* o_hi, void* o_lo, float* o_f32, int64_t o_pitch, float* mean, float* rstd,
                      void* stream);
/* Row-slab count used by the reductions below (first extent of their `partials` scratch). */
int32_t sfb_rowslab_blocks(int64_t rows);
/* dx (= or +=), dgamma / dbeta (= or +=); partials scratch [sfb_rowslab_blocks(rows)][2][c]. */
int sfb_layernorm_bwd(const float* dy, int64_t dy_pitch, const float* x, int64_t x_pitch, int64_t rows, int32_t c,
                      const float* gamma, const float* mean, const float* rstd, float* dx, int64_t dx_pitch,
                      int32_t dx_accumulate, float* dgamma, float* dbeta, int32_t param_accumulate, float* partials,
                      void* stream);
/* out[c] (= or +=) column sums of src[rows, c] (bias gradients); partials scratch [sfb_rowslab_blocks(rows)][c]. */
int sfb_colsum(const float* src, int64_t pitch, int64_t rows, int32_t c, float* out, int32_t accumulate, float* partials,
               void* stream);
/* x[b,0,:] = cls; x[b,1+l,:] = y[b,l,:] + bias   (PatchEmbed output + cls token, video_model_builder.py:1180-1186) */
int sfb_tokens_assemble(const float* y, const float* bias, const float* cls, int32_t b, int32_t l, int32_t c, float* x,
                        void* stream);
int sfb_tokens_split_grad(const float* dx, int32_t b, int32_t l, int32_t c, void* dy_hi, void* dy_lo, float* dy_f32,
                          void* stream);
/* attention_pool with the depthwise Conv3d (groups = head_dim, weight shared by the heads, padding k/2):
 * src = fused-qkv GEMM output [B, 1+L, src_pitch] (+bias on real tokens), out = [B, heads, 1+L', hd] fp32. */
typedef struct sfb_dwpool_desc {
  const float* src; int64_t src_pitch; int32_t src_c0; const float* bias;
  const float* w; /* [hd][kt*kh*kw], NULL when has_pool == 0 */
  float* out;
  int32_t b, heads, hd, t, h, w_, ot, oh, ow, kt, kh, kw, st, sh, sw;
  int32_t has_pool;
  const float* dout; /* bwd: gradient w.r.t. out */
  float* dsrc;       /* bwd: gradient w.r.t. src (+=, same geometry as src) */
  float* wpartials;  /* unused since ABI v1 r1d (the weight gradient is accumulated atomically); kept for layout stability */
} sfb_dwpool_desc;
int sfb_dwpool_fwd(const sfb_dwpool_desc* d, void* stream);
int32_t sfb_dwpool_wgrad_blocks(const sfb_dwpool_desc* d);
int sfb_dwpool_bwd(const sfb_dwpool_desc* d, float* dw, int32_t dw_accumulate, void* stream);
/* softmax over keys of S + decomposed relative-position bias (cal_rel_pos_spatial / _temporal): RQ = q . [Rh;Rw;Rt]^T
 * per non-cls query; P is written as planes (pad columns zero).  bwd: dS planes and dRQ. */
typedef struct sfb_softmax_desc {
  const float* s; int64_t s_pitch;
  const float* rq; int64_t rq_pitch;
  void* p_hi; void* p_lo; int64_t p_pitch;
  int32_t bh, nq, nk, qt, qh, qw, kt, kh, kw;
  const float* dp; int64_t dp_pitch;
  void* ds_hi; void* ds_lo; int64_t ds_pitch;
  float* drq;
} sfb_softmax_desc;
int sfb_softmax_relpos_fwd(const sfb_softmax_desc* d, void* stream);
int sfb_softmax_relpos_bwd(const sfb_softmax_desc* d, void* stream);
/* merged[b,n,h*hd+c] = O[b,h,n,c] (+ q[b,h,n,c] for n > 0: residual pooling, attention.py:381-385) -> planes */
int sfb_attn_merge(const float* o, const void* q_hi, const void* q_lo, int32_t b, int32_t h, int32_t n, int32_t hd,
                   int32_t residual, void* m_hi, void* m_lo, void* stream);
int sfb_attn_split_grad(const float* dm, int32_t b, int32_t h, int32_t n, int32_t hd, int32_t residual, void* do_hi,
                        void* do_lo, float* dq, void* stream);
/* out = a [+ a_bias] + scale[sample] * (y + y_bias)   (residual adds with Linear biases and stochastic depth) */
int sfb_residual_add(const float* a, const float* a_bias, const float* y, const float* y_bias, const float* scale,
                     int64_t rows, int32_t c, int64_t rows_per_sample, float* out, void* stream);
int sfb_bias_gelu(const float* y, const float* bias, int64_t rows, int32_t c, void* hi, void* lo, void* stream);
int sfb_bias_gelu_bwd(const float* dh, const float* y, const float* bias, int64_t rows, int32_t c, void* hi, void* lo,
                      float* dpre, void* stream);
int sfb_scale_split(const float* src, const float* scale, int64_t rows, int32_t c, int64_t rows_per_sample, void* hi,
                    void* lo, float* f32, void* stream);
/* MaxPool3d skip path on tokens (cls passes through), kernel s+1 / stride s / padding k/2 (attention.py:485-489) */
typedef struct sfb_tokpool_desc {
  const float* x; float* out; uint8_t* argmax;
  int32_t b, c, t, h, w, ot, oh, ow, kt, kh, kw, st, sh, sw;
  const float* dout; float* dx; int32_t dx_accumulate;
} sfb_tokpool_desc;
int sfb_token_maxpool_fwd(const sfb_tokpool_desc* d, void* stream);
int sfb_token_maxpool_bwd(const sfb_tokpool_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Classification head (head_helper.py:305-350 ResNetBasicHead, :547-563 TransformerBasicHead):
 * AvgPool3d over the whole (T,H,W) extent, Dropout, Linear, eval-mode Softmax.
 * ---------------------------------------------------------------------------------------------- */
/* out[n, c] = mean over `spatial` positions of the (hi+lo) planes [n, spatial, c] (row pitch `pitch`). */
int sfb_global_avgpool_fwd(const void* hi, const void* lo, int64_t pitch, int32_t n, int32_t spatial, int32_t c,
                           float* out, int64_t out_pitch, void* stream);
int sfb_global_avgpool_bwd(const float* dpooled, int64_t dp_pitch, int32_t n, int32_t spatial, int32_t c, float* dx,
                           int64_t dx_pitch, void* stream);
/* Fully-convolutional inference of ResNetBasicHead (head_helper.py:250-255 AvgPool3d(pool_size, stride=1), :338-345
 * per-location softmax then mean over [1,2,3]): stride-1 window means of the planes -> fp32 rows
 * [n*ot*oh*ow, c] (row pitch out_pitch), and the mean of g consecutive rows. */
int sfb_window_avgpool_fwd(const void* hi, const void* lo, int64_t pitch, int32_t n, int32_t t, int32_t h, int32_t w,
                           int32_t c, int32_t kt, int32_t kh, int32_t kw, float* out, int64_t out_pitch, void* stream);
int sfb_rows_group_mean(const float* in, float* out, int32_t n, int32_t g, int32_t k, void* stream);
/* In-place inverted dropout with a counter-based generator; mask (uint8 keep flags) is saved for backward.
 * `step` (optional device counter) is mixed into the seed and incremented on the stream after use, so that replays
 * of a captured CUDA graph draw fresh masks. */
int sfb_dropout_fwd(float* x, uint8_t* mask, int64_t nelem, float p, uint64_t seed, uint64_t* step, void* stream);
int sfb_dropout_bwd(float* dx, const uint8_t* mask, int64_t nelem, float p, void* stream);
/* y[m,k] = x[m,j] . w[k,j] + b[k]  (fp32, small m).  bwd: dw/db (= or +=), dx; any of dw/dx may be NULL. */
int sfb_small_linear_fwd(const float* x, const float* w, const float* b, float* y, int32_t m, int32_t k, int32_t j,
                         void* stream);
int sfb_small_linear_bwd(const float* dy, const float* x, const float* w, float* dw, float* db, float* dx, int32_t m,
                         int32_t k, int32_t j, int32_t accumulate, void* stream);
int sfb_row_softmax(float* x, int32_t rows, int32_t cols, void* stream);
/* Stochastic depth (common.py:46-59): out[i*b + s] = floor(keep_i + U)/keep_i for n_rates drop rates and b samples. */
int sfb_droppath_scales(float* out, const float* rates, int32_t n_rates, int32_t b, uint64_t seed, uint64_t* step,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * X3D (video_model_builder.py:664 X3D, resnet_helper.py:253 X3DTransform, stem_helper.py:280 X3DStem,
 * operators.py:55 SE, head_helper.py:461 X3DHead).  Channel counts are padded to multiples of 8 (`c`), `c_valid`
 * is the module's real width; pad channels hold exact zeros.
 * ---------------------------------------------------------------------------------------------- */
/* Channelwise Conv3d (groups == channels; nn.Conv3d weight [c_valid, 1, kt, kh, kw], no bias), <= 27 taps.
 * Input = split planes (x_hi/x_lo) or fp32 (x_f32); output y fp32 + BatchNorm partials stats[2][c_valid][m_tiles]
 * (tiles never straddle samples: sample s owns tiles [s*tps, (s+1)*tps), which is what sfb_se_fwd pools over). */
typedef struct sfb_dwconv_desc {
  const void* x_hi; const void* x_lo; const float* x_f32; int64_t x_pitch;
  const float* w;
  float* y; int64_t y_pitch; float* stats;
  int32_t n, t, h, w_, c, c_valid, ot, oh, ow, kt, kh, kw, st, sh, sw, pt, ph, pw;
  const float* dy; int64_t dy_pitch;   /* bwd: gradient w.r.t. y (fp32) */
  float* dx;                           /* bwd: fp32 data gradient (stored, or += when dx_accumulate) ...     */
  void* dx_hi; void* dx_lo;            /* ... or, when dx == NULL, split planes (operand of the next wgrad)  */
  int64_t dx_pitch; int32_t dx_accumulate;
  float* wpartials;                    /* bwd scratch [sfb_dwconv_wgrad_blocks()][c][taps] */
  /* optional producer transform fused into every input read (fp32 input only): x := relu?(x*in_scale + in_shift),
   * i.e. the BatchNorm (+ReLU) of the layer that produced x; padding stays zero AFTER the transform */
  const float* in_scale; const float* in_shift; int32_t in_relu;
} sfb_dwconv_desc;
int32_t sfb_dwconv_m_tiles(const sfb_dwconv_desc* d);
int32_t sfb_dwconv_tiles_per_sample(const sfb_dwconv_desc* d);
int sfb_dwconv_fwd(const sfb_dwconv_desc* d, void* stream);
int32_t sfb_dwconv_wgrad_blocks(const sfb_dwconv_desc* d);
/* dw == NULL skips the weight gradient; dx == dx_hi == NULL skips the data gradient */
int sfb_dwconv_bwd(const sfb_dwconv_desc* d, float* dw, void* stream);
/* out = act( (y*scale + shift) * gate[sample] ),  act: 0 identity, 1 ReLU, 2 Swish (x*sigmoid(x)); planes out.
 * Backward in two passes: reduce -> partials[tile][2][c] (sum g, sum g*xhat per sample tile, g = dout*act'),
 * sfb_se_bwd turns them into the coefficients, apply -> dy = ca*(g*gate + davg[sample]) - cb - xhat*cc (fp32). */
typedef struct sfb_bnact_desc {
  const float* y; int64_t y_pitch;
  const float* scale; const float* shift; const float* mean; const float* invstd;
  const float* gate;  /* [n][c] or NULL */
  int32_t act;
  int64_t rows; int64_t rows_per_sample; int32_t c;
  void* out_hi; void* out_lo; int64_t out_pitch;
  const float* dout; int64_t dout_pitch;
  float* partials;    /* [n * sfb_bnact_tiles_per_sample()][2][c] */
  const float* davg;  /* [n][c] per-position gradient through the SE average pool, or NULL */
  const float* coef;  /* [3][c] */
  float* dy; int64_t dy_pitch;
} sfb_bnact_desc;
int sfb_bnact_fwd(const sfb_bnact_desc* d, void* stream);
int32_t sfb_bnact_tiles_per_sample(int64_t rows, int64_t rows_per_sample);
int sfb_bnact_bwd_reduce(const sfb_bnact_desc* d, void* stream);
int sfb_bnact_bwd_apply(const sfb_bnact_desc* d, void* stream);
/* SE bottleneck on the BN output z = y*scale+shift: avg = mean_pos z (from the conv's per-tile sums),
 * hid = relu(w1 avg + b1), gate = sigmoid(w2 hid + b2).  sfb_se_bwd (has_se = 0: plain BN -> act) merges the
 * bnact partials per sample, runs the SE backward, and emits dgamma/dbeta, the SE parameter gradients, davg and
 * the [3][c_pad] apply coefficients. */
typedef struct sfb_se_desc {
  int32_t n, c, c_pad, f; int64_t rows_per_sample; int32_t tiles_per_sample, m_tiles;
  const float* stats; const float* scale; const float* shift; const float* mean; const float* invstd;
  const float* w1; const float* b1; const float* w2; const float* b2;
  float* ymean; float* avg; float* hid; float* gate;       /* [n][c_pad], [n][c_pad], [n][f], [n][c_pad] */
  const float* partials; int32_t tiles2_per_sample;
  float* a12; float* do2; float* dhid; float* davg;        /* [n][2][c_pad], [n][c_pad], [n][f], [n][c_pad] */
  const float* gamma; const float* beta;
  float* dw1; float* db1; float* dw2; float* db2; float* dgamma; float* dbeta; float* coef;
  int32_t training, has_se;
} sfb_se_desc;
int sfb_se_fwd(const sfb_se_desc* d, void* stream);
int sfb_se_bwd(const sfb_se_desc* d, void* stream);
/* in-place ReLU on a small fp32 tensor (X3DHead lin_5_relu) and its backward dx = y > 0 ? dx : 0 */
int sfb_relu_fwd(float* x, int64_t n, void* stream);
int sfb_relu_bwd(float* dx, const float* y, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MaskFeat (masked.py:25 MaskMViT, :519 _maskfeat_forward; operators.py:79 HOGLayerC; head_helper.py:656
 * MSSeparateHead).  The encoder is the MViT path above; these are the wrapper's own operators.
 * ---------------------------------------------------------------------------------------------- */
/* out[b, (z,y,x)] = mask[b, z*mt/t, y*mh/h, x*mw/w]: F.interpolate(mode='nearest') of the loader's cube mask */
int sfb_mask_upsample(const float* mask, int32_t b, int32_t mt, int32_t mh, int32_t mw, int32_t t, int32_t h, int32_t w,
                      float* out, void* stream);
/* x[b,0] = cls; x[b,1+n] = (y[b,n] + bias) * (1 - m[b,n]) + mask_token * m[b,n]   (masked.py:551-565) */
int sfb_tokens_assemble_masked(const float* y, const float* bias, const float* cls, const float* mask_token,
                               const float* tokmask, int32_t b, int32_t l, int32_t c, float* x, void* stream);
/* backward: dy = dx[b,1+n] * (1 - m) as planes + fp32, dxm = dx[b,1+n] * m (its column sum is d mask_token) */
int sfb_tokens_split_grad_masked(const float* dx, const float* tokmask, int32_t b, int32_t l, int32_t c, void* dy_hi,
                                 void* dy_lo, float* dy_f32, float* dxm, void* stream);
/* prediction head rows: out[b, n, :c] = y[(b*(l+1) + 1 + n) * ldy + :c] + bias (drops the cls row), and the
 * gradient's way back: planes [b*(l+1)][cp] with zero cls rows / pad columns */
int sfb_rows_unpad_bias(const float* y, int64_t ldy, const float* bias, int32_t b, int32_t l, int32_t c, float* out,
                        void* stream);
int sfb_rows_pad_split(const float* d, int32_t b, int32_t l, int32_t c, int32_t cp, void* hi, void* lo, void* stream);
/* HOG targets of the frames x[:, :, ::t_stride] (x = [b, ch, t, h, w] fp32): out[b, t/t_stride, fs, fs,
 * ch*nbins*u*u] with u = (h/cell)/fs, feature index ((c*nbins + bin)*u + wy)*u + wx   (masked.py:254-281) */
int sfb_hog_targets(const float* x, int32_t b, int32_t ch, int32_t t, int32_t h, int32_t w, int32_t t_stride,
                    int32_t nbins, int32_t cell, int32_t fs, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimizer step + gradient norm / clipping on the flat gradient bucket (SURVEY.md section 8f-1).
 * Replaces: torch.optim.SGD(nesterov) / AdamW as built by slowfast/models/optimizer.py:105-136, get_grad_norm_
 * (optimizer.py:362-379) and clip_grad_norm_ / clip coefficient (tools/train_net.py:154-172).
 * ---------------------------------------------------------------------------------------------- */
typedef struct sfb_opt_chunk {
  float* param;      /* first element of this chunk inside its parameter tensor */
  int64_t offset;    /* element offset of the chunk in the flat bucket (gradient and optimizer state) */
  int32_t count;     /* elements in the chunk */
  int32_t group;     /* index into group_lr / group_wd */
} sfb_opt_chunk;
int32_t sfb_opt_chunk_size(void);
int32_t sfb_flat_sumsq_blocks(void);  /* length of the fp64 `partials` scratch */
/* out3[0] = ||flat||_2 * inv_scale; out3[1] = min(1, max_norm / (norm + 1e-6)) (1 if max_norm <= 0);
 * out3[2] = out3[1] * inv_scale = the factor the update kernels apply to every gradient (AMP unscale + clip). */
int sfb_flat_sumsq(const float* flat, int64_t n, double* partials, float max_norm, float inv_scale, float* out3,
                   void* stream);
/* One launch over `n_chunks` chunks.  gscale: NULL or the out3 array of sfb_flat_sumsq (device). */
int sfb_flat_sgd(const void* chunks, int32_t n_chunks, const float* grad, float* momentum_buf, const float* group_lr,
                 const float* group_wd, const float* gscale, float momentum, float dampening, int32_t nesterov,
                 int32_t first_step, void* stream);
int sfb_flat_adamw(const void* chunks, int32_t n_chunks, const float* grad, float* exp_avg, float* exp_avg_sq,
                   const float* group_lr, const float* group_wd, const float* gscale, float beta1, float beta2, float eps,
                   int64_t step, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused pooled-attention forward (MultiScaleAttention.forward, attention.py:355-385; rel-pos bias :64-147):
 * O = softmax(scale * q k^T + bias) v per (clip*head), scores and probabilities kept in shared memory.
 * q / k / v: split planes [bh, n, 96] (the LayerNorm-ed pooled tensors); rq = q_nocls . [Rh;Rw;Rt]^T [bh*(nq-1), rq_pitch]
 * or NULL (no rel-pos); out fp32 [bh, nq, 96]; p_hi/p_lo (optional): normalised probabilities as planes [bh*nq, p_pitch]
 * (pad columns zero) for the unfused backward; lse (optional) [bh*nq].  Fused for head_dim 96 and an 8x7x7 key grid
 * (nk = 393: the pooled K/V of 12 of MViTv2-S's 16 blocks) - sfb_attn_fwd_supported() says whether a geometry is; the
 * unfused sequence sfb_gemm_batched -> sfb_softmax_relpos_fwd -> sfb_gemm_batched covers the rest.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sfb_attn_fwd_desc {
  const void* q_hi; const void* q_lo; const void* k_hi; const void* k_lo; const void* v_hi; const void* v_lo;
  const float* rq; int64_t rq_pitch;
  int32_t bh, nq, nk, hd;
  int32_t qt, qh, qw, kt, kh, kw;
  float scale;
  float* out;
  void* p_hi; void* p_lo; int64_t p_pitch;
  float* lse;
  int32_t nsplit;
} sfb_attn_fwd_desc;
int32_t sfb_attn_fwd_supported(int32_t nk, int32_t hd, int32_t kt, int32_t kh, int32_t kw);
/* First half of the attention backward for the same key grids (attention.py:355-379 through autograd): dP = dO v^T in shared memory,
 * dS = P (dP - sum_k P dP) -> split planes [bh*nq, ds_pitch] (operand of the dq = scale dS k and dk = scale dS^T q products, pad
 * columns zero), and the gradient of the decomposed rel-pos bias, dRQ [bh*(nq-1), rq_pitch] (drq == NULL: no bias).  Replaces
 * sfb_gemm_batched (dP) + sfb_softmax_relpos_bwd.  p_hi / p_lo: the planes sfb_attn_fwd wrote. */
typedef struct sfb_attn_bwd_desc {
  const void* do_hi; const void* do_lo; const void* v_hi; const void* v_lo;
  const void* p_hi; const void* p_lo; int64_t p_pitch;
  void* ds_hi; void* ds_lo; int64_t ds_pitch;
  float* drq; int64_t rq_pitch;
  int32_t bh, nq, nk, hd;
  int32_t qt, qh, qw, kt, kh, kw;
  int32_t nsplit;
} sfb_attn_bwd_desc;
int sfb_attn_bwd_ds(const sfb_attn_bwd_desc* d, void* stream);
int sfb_attn_fwd(const sfb_attn_fwd_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Device-side input pipeline head (SURVEY.md section 8f-3): uint8 clip [b, t, h, w, 3] (decoder layout) ->
 * fp32 NCTHW [b, 3, t_out, h, w] = (x / 255 - mean[c]) / std[c] at the frames frame_idx[0..t_out) (NULL = all frames).
 * Replaces, on the host side of the reference: tensor_normalize (datasets/utils.py:278-297), the THWC -> CTHW permute
 * (datasets/kinetics.py:375-405), pack_pathway_output's slow-pathway index_select (datasets/utils.py:95-103) and
 * DATA.REVERSE_INPUT_CHANNEL (:89-90); the H2D copy then carries uint8.  mean3 / std3 are HOST pointers (3 floats).
 * ---------------------------------------------------------------------------------------------- */
int sfb_clip_normalize_pack(const uint8_t* frames, int32_t b, int32_t t, int32_t h, int32_t w, const int32_t* frame_idx,
                            int32_t t_out, const float* mean3, const float* std3, int32_t reverse_channels, float* out,
                            void* stream);

/* ------------------------------------------------------------------------------------------------
 * Data-parallel exchange (SURVEY.md section 8e): ONE in-place all-reduce of the flat fp32 gradient bucket on the caller's NCCL
 * communicator (`ncclComm_t` passed as void*) and stream; average != 0 -> ncclAvg (DDP semantics: sum / world size).
 * Replaces the DistributedDataParallel bucketing + per-bucket all-reduce of slowfast/models/build.py:66-76.
 * NCCL is resolved at run time from the copy the process already loaded (no link-time dependency).
 * ---------------------------------------------------------------------------------------------- */
int sfb_allreduce_flat(float* buf, int64_t count, void* nccl_comm, int32_t average, void* stream);

/* Narrow layers (C_in, C_out <= 64, taps*C_in*C_out <= max_macs) of sfb_conv_igemm on the fp32 pipes (csrc/conv_direct.cu)
 * instead of the tensor-core body: same descriptor, same results layout.  max_macs <= 0 keeps the current threshold. */
int sfb_set_simt_smallc(int32_t enabled, int32_t max_macs);

/* A/B switch of the shared-memory-ring channelwise 3x3x3 kernels (csrc/x3d_ops.cu "v3"); 1 = on (default). */
int sfb_set_dw3(int32_t enabled);

#ifdef __cplusplus
}
#endif
#endif /* SLOWFAST_B200_H_ */
