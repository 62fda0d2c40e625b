"""MViTv2 (video_model_builder.py:806 MViT; attention.py MultiScaleBlock / MultiScaleAttention) on the engine.

Module tree, parameter names and initialisation mirror the reference (patch_embed.proj, cls_token, blocks.{i}.norm1 /
attn.{qkv,proj,pool_{q,k,v},norm_{q,k,v},rel_pos_{h,w,t}} / norm2 / mlp.{fc1,fc2} / proj, norm, head.projection).
Execution:
  * every Linear (qkv, proj, fc1, fc2, block proj) and the patch embedding run on the wgmma implicit-GEMM kernel;
    their wgrad / dgrad on the same kernels as the conv nets;
  * pooled attention: depthwise pooling convs read the fused-qkv GEMM output in place (no permute/contiguous copies),
    QK^T / PV and the four backward products are batched wgmma GEMMs in all operand-major combinations, the
    decomposed relative-position bias is ONE extra GEMM of q against the concatenated [Rh;Rw;Rt] tables plus an
    index lookup inside the softmax kernel (SURVEY.md section 7.6: identical to cal_rel_pos_spatial/_temporal);
  * LayerNorm, GELU, residual/bias/stochastic-depth combines, max-pool skip are fused row kernels.
Scope: the MViTv2 configuration family of the reference's Kinetics configs (cls token on, no absolute position
embedding, conv pooling, pool_first False, DIM_MUL_IN_ATT True).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import List, Optional

import torch
import torch.nn as nn

from .. import lib as L
from .. import ops
from ..config import nsplit_of
from ..engine import Ctx, ModelFunction, Namespace
from ..ops import F32, Planes

BF16 = torch.bfloat16


def round_width(width, multiplier, min_width=1, divisor=1):
    """models/utils.py:10-24."""
    if not multiplier:
        return width
    width *= multiplier
    min_width = min_width or divisor
    out = max(min_width, int(width + divisor / 2) // divisor * divisor)
    if out < 0.9 * width:
        out += divisor
    return int(out)


def block_specs(cfg):
    """Per-block geometry exactly as MViT.__init__ derives it (video_model_builder.py:914-1030)."""
    mv = cfg.MVIT
    depth = mv.DEPTH
    dim_mul, head_mul = [1.0] * (depth + 1), [1.0] * (depth + 1)
    for i, m in mv.DIM_MUL:
        dim_mul[int(i)] = m
    for i, m in mv.HEAD_MUL:
        head_mul[int(i)] = m
    pool_q, pool_kv = [[] for _ in range(depth)], [[] for _ in range(depth)]
    stride_q, stride_kv = [[] for _ in range(depth)], [[] for _ in range(depth)]
    kvq = mv.POOL_KVQ_KERNEL
    for e in mv.POOL_Q_STRIDE:
        stride_q[e[0]] = list(e[1:])
        pool_q[e[0]] = list(kvq) if kvq is not None else [s + 1 if s > 1 else s for s in e[1:]]
    kv_list = [list(e) for e in mv.POOL_KV_STRIDE]
    if mv.POOL_KV_STRIDE_ADAPTIVE is not None:
        cur = list(mv.POOL_KV_STRIDE_ADAPTIVE)
        kv_list = []
        for i in range(depth):
            if len(stride_q[i]) > 0:
                cur = [max(cur[d] // stride_q[i][d], 1) for d in range(len(cur))]
            kv_list.append([i] + cur)
    for e in kv_list:
        stride_kv[e[0]] = list(e[1:])
        pool_kv[e[0]] = list(kvq) if kvq is not None else [s + 1 if s > 1 else s for s in e[1:]]
    ps = list(mv.PATCH_STRIDE)
    size = [cfg.DATA.NUM_FRAMES // ps[0], cfg.DATA.TRAIN_CROP_SIZE // ps[1], cfg.DATA.TRAIN_CROP_SIZE // ps[2]]
    embed, heads = mv.EMBED_DIM, mv.NUM_HEADS
    specs = []
    for i in range(depth):
        heads = round_width(heads, head_mul[i])
        if mv.DIM_MUL_IN_ATT:
            dim_out = round_width(embed, dim_mul[i], divisor=round_width(heads, head_mul[i]))
        else:
            dim_out = round_width(embed, dim_mul[i + 1], divisor=round_width(heads, head_mul[i + 1]))
        specs.append(dict(dim=embed, dim_out=dim_out, heads=heads, kq=pool_q[i], kkv=pool_kv[i], sq=stride_q[i],
                          skv=stride_kv[i], size=list(size)))
        if len(stride_q[i]) > 0:
            size = [s // st for s, st in zip(size, stride_q[i])]
        embed = dim_out
    return specs


def _is_pool(kernel, stride) -> bool:
    """MultiScaleAttention skips pooling with kernel and stride (1,1,1) (attention.py:199-203)."""
    return len(kernel) > 0 and not (math.prod(kernel) == 1 and math.prod(stride) == 1)


class AttentionModule(Namespace):
    """MultiScaleAttention parameter container (attention.py:151-291)."""

    def __init__(self, dim, dim_out, heads, size, kq, kkv, sq, skv, qkv_bias, rel_sp, rel_t, rel_zero):
        super().__init__()
        hd = dim_out // heads
        # construction order = the reference's (same RNG stream => bit-identical initialisation)
        self.qkv = nn.Linear(dim, dim_out * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim_out, dim_out)
        for name, k, s in (("q", kq, sq), ("k", kkv, skv), ("v", kkv, skv)):
            if _is_pool(k, s):
                setattr(self, f"pool_{name}", nn.Conv3d(hd, hd, k, stride=s, padding=[int(x // 2) for x in k],
                                                       groups=hd, bias=False))
                setattr(self, f"norm_{name}", nn.LayerNorm(hd, eps=1e-6))
        if rel_sp:
            assert size[1] == size[2]
            q_size = size[1] // sq[1] if len(sq) > 0 else size[1]
            kv_size = size[1] // skv[1] if len(skv) > 0 else size[1]
            n = 2 * max(q_size, kv_size) - 1
            self.rel_pos_h = nn.Parameter(torch.zeros(n, hd))
            self.rel_pos_w = nn.Parameter(torch.zeros(n, hd))
            if not rel_zero:
                nn.init.trunc_normal_(self.rel_pos_h, std=0.02)
                nn.init.trunc_normal_(self.rel_pos_w, std=0.02)
        if rel_t:
            self.rel_pos_t = nn.Parameter(torch.zeros(2 * size[0] - 1, hd))
            if not rel_zero:
                nn.init.trunc_normal_(self.rel_pos_t, std=0.02)


class MlpModule(Namespace):
    def __init__(self, dim, hidden, out):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, out)


class BlockModule(Namespace):
    """MultiScaleBlock parameter container (attention.py:396-489)."""

    def __init__(self, spec, mlp_ratio, qkv_bias, rel_sp, rel_t, rel_zero, dim_mul_in_att):
        super().__init__()
        dim, dim_out = spec["dim"], spec["dim_out"]
        att_dim = dim_out if dim_mul_in_att else dim
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = AttentionModule(dim, att_dim, spec["heads"], spec["size"], spec["kq"], spec["kkv"], spec["sq"],
                                    spec["skv"], qkv_bias, rel_sp, rel_t, rel_zero)
        self.drop_path = nn.Identity()
        self.norm2 = nn.LayerNorm(att_dim, eps=1e-6)
        self.mlp = MlpModule(att_dim, int(att_dim * mlp_ratio), dim_out)
        if dim != dim_out:
            self.proj = nn.Linear(dim, dim_out)
        self.dim, self.dim_out = dim, dim_out


class PatchEmbedModule(Namespace):
    def __init__(self, cin, cout, kernel, stride, padding):
        super().__init__()
        self.proj = nn.Conv3d(cin, cout, kernel_size=tuple(kernel), stride=tuple(stride), padding=tuple(padding))


class TransformerHeadModule(Namespace):
    def __init__(self, dim_in, num_classes, dropout_rate, act_func):
        super().__init__()
        if dropout_rate > 0.0:
            self.dropout = nn.Dropout(dropout_rate)
        self.projection = nn.Linear(dim_in, num_classes, bias=True)  # the reference constructs it twice (:515,:517)
        self.projection = nn.Linear(dim_in, num_classes, bias=True)
        self.dropout_rate = dropout_rate
        self.act_func = act_func


# fused pooled attention (csrc/attn_fused.cu), opt-in with SFB_ATTN_FUSED=1 / SFB_ATTN_FUSED_BWD=1: on one H100 (400 W) the
# MViTv2-S step runs 59.0 clips/s with it and 67.3 with the unfused sequence (gemm_batched -> softmax_relpos -> gemm_batched),
# because the fused kernel is not yet tuned (one warpgroup per CTA, loads not overlapped with the MMAs)
ATTN_FUSED = os.environ.get("SFB_ATTN_FUSED", "0") != "0"
# fused first half of the attention backward (dP in shared memory -> dS planes + dRQ); 0 = dP GEMM + softmax_relpos_bwd
ATTN_FUSED_BWD = os.environ.get("SFB_ATTN_FUSED_BWD", "0") != "0"


def _ptr(t):
    return None if t is None else t.data_ptr()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class B200MViT(nn.Module):
    """MViTv2 on the engine (drop-in for the reference's registered ``MViT``)."""

    cuda_graphs = True
    graph_warmup = 2

    def __init__(self, cfg):
        super().__init__()
        mv = cfg.MVIT
        assert cfg.DATA.TRAIN_CROP_SIZE == cfg.DATA.TEST_CROP_SIZE
        assert mv.MODE == "conv" and mv.CLS_EMBED_ON and not mv.USE_ABS_POS and not mv.POOL_FIRST
        assert not mv.SEPARATE_QKV and not mv.NORM_STEM and not mv.USE_MEAN_POOLING
        assert not mv.PATCH_2D and not mv.REV.ENABLE and not cfg.DETECTION.ENABLE and mv.NORM == "layernorm"
        assert float(mv.LAYER_SCALE_INIT_VALUE) == 0.0 and float(mv.DROPOUT_RATE) == 0.0
        self.cfg = cfg
        self.ctx = Ctx(nsplit_of(cfg))
        self.specs = block_specs(cfg)
        self.patch_stride = list(mv.PATCH_STRIDE)
        self.T = cfg.DATA.NUM_FRAMES // self.patch_stride[0]
        self.H = cfg.DATA.TRAIN_CROP_SIZE // self.patch_stride[1]
        self.W = cfg.DATA.TRAIN_CROP_SIZE // self.patch_stride[2]
        self.num_classes = cfg.MODEL.NUM_CLASSES
        self.residual_pooling = bool(mv.RESIDUAL_POOLING)
        self.dim_mul_in_att = bool(mv.DIM_MUL_IN_ATT)
        self.patch_embed = PatchEmbedModule(cfg.DATA.INPUT_CHANNEL_NUM[0], mv.EMBED_DIM, mv.PATCH_KERNEL, mv.PATCH_STRIDE,
                                            mv.PATCH_PADDING)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, mv.EMBED_DIM))
        self.blocks = nn.ModuleList()
        for spec in self.specs:
            self.blocks.append(BlockModule(spec, mv.MLP_RATIO, mv.QKV_BIAS, mv.REL_POS_SPATIAL, mv.REL_POS_TEMPORAL,
                                           mv.REL_POS_ZERO_INIT, mv.DIM_MUL_IN_ATT))
        embed = self.specs[-1]["dim_out"]
        self.norm = nn.LayerNorm(embed, eps=1e-6)
        self.head = TransformerHeadModule(embed, self.num_classes, cfg.MODEL.DROPOUT_RATE, cfg.MODEL.HEAD_ACT)
        nn.init.trunc_normal_(self.cls_token, std=0.02)
        self.apply(self._init_weights)
        self.head.projection.weight.data.mul_(mv.HEAD_INIT_SCALE)
        self.head.projection.bias.data.mul_(mv.HEAD_INIT_SCALE)
        depth = mv.DEPTH
        self.drop_rates = [x.item() for x in torch.linspace(0, float(mv.DROPPATH_RATE), depth)]
        object.__setattr__(self, "_graphs", {})
        object.__setattr__(self, "_graph_seen", {})
        b200 = getattr(cfg, "B200", None)
        if b200 is not None and "CUDA_GRAPH" in b200:
            self.cuda_graphs = bool(b200["CUDA_GRAPH"])
        self._seed = int(getattr(cfg, "RNG_SEED", 0))
        object.__setattr__(self, "_saved", None)

    @staticmethod
    def _init_weights(m):
        """MViT._init_weights (video_model_builder.py:1085-1093)."""
        if isinstance(m, (nn.Linear, nn.Conv2d, nn.Conv3d)):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.constant_(m.bias, 0.02)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0.02)
            nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        names = []
        if self.cfg.MVIT.ZERO_DECAY_POS_CLS:
            if self.cfg.MVIT.REL_POS_SPATIAL:
                names.extend(["rel_pos_h", "rel_pos_w", "rel_pos_hw"])
            if self.cfg.MVIT.REL_POS_TEMPORAL:
                names.extend(["rel_pos_t"])
            names.append("cls_token")
        return names

    def forward(self, x, bboxes=None, return_attn=False):
        assert bboxes is None and not return_attn
        x = [x[0]]
        params = [p for p in self.parameters()]
        return ModelFunction.apply(self, 1, *x, *params)

    def allreduce_gradients(self, group=None) -> None:
        from ..engine import allreduce_flat_gradients
        assert self.ctx.flat_grad is not None, "call after backward()"
        allreduce_flat_gradients(self.ctx.flat_grad, list(self.parameters()), group,
                                 repoint=not getattr(self, "flat_grad_only", False))

    # ================================================================================== helpers
    def _lin_fwd(self, key, lin: nn.Linear, x: Planes) -> torch.Tensor:
        """y[rows, out] = x[rows, in] . W^T  (no bias; consumers add it)."""
        ctx = self.ctx
        out_f, in_f = lin.weight.shape
        f = ctx.scratch("lin.f.hi", out_f * in_f, BF16).view(out_f, in_f)
        flo = ctx.scratch("lin.f.lo", out_f * in_f, BF16).view(out_f, in_f) if ctx.nsplit == 3 else None
        fm = ops.FilterMat(f, flo, out_f, 1, in_f)
        ops.filter_pack(lin.weight, fm)
        rows = x.rows
        y = ctx.buf(key, (rows, out_f))
        ops.conv_igemm(x, fm, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (x.t, x.h, x.w)), y,
                       (rows * out_f, rows * out_f, rows * out_f, out_f), nsplit=ctx.nsplit)
        return y

    def _lin_bwd(self, lin: nn.Linear, dy: Planes, dy_f32: Optional[torch.Tensor], x: Planes,
                 dx: Optional[torch.Tensor], bias_grad: bool = True) -> None:
        """dW (grad slot), db (column sum of dy), dx[rows, in] = dy . W  (plain store)."""
        ctx = self.ctx
        out_f, in_f = lin.weight.shape
        gw = ctx.grad_of(lin.weight)
        ops.zero_f32(ops.f32view(gw))
        geom = ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (x.t, x.h, x.w))
        ops.conv_wgrad(x, dy, geom, gw, nsplit=ctx.nsplit)
        if bias_grad and lin.bias is not None:
            self._colsum(dy_f32, dy.rows, out_f, ctx.grad_of(lin.bias))
        if dx is not None:
            f = ctx.scratch("lin.ft.hi", out_f * in_f, BF16).view(in_f, out_f)
            flo = ctx.scratch("lin.ft.lo", out_f * in_f, BF16).view(in_f, out_f) if ctx.nsplit == 3 else None
            fm = ops.FilterMat(f, flo, in_f, 1, out_f)
            ops.filter_pack(lin.weight, fm, tapmap=[0], transpose=True)
            rows = dy.rows
            ops.conv_igemm(dy, fm, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (dy.t, dy.h, dy.w)), dx,
                           (rows * in_f, rows * in_f, rows * in_f, in_f), nsplit=ctx.nsplit)

    def _rows_planes(self, key, rows, c, scratch=False) -> Planes:
        ctx = self.ctx
        if scratch:
            return ctx.scratch_planes(key, 1, 1, 1, rows, c)
        s = ctx.storage(key, 1, 1, 1, rows, c)
        return Planes(s.hi, s.lo, 1, 1, 1, rows, c, 0)

    def _colsum(self, src: torch.Tensor, rows, c, out: torch.Tensor, pitch=None, accumulate=False):
        lib = L.load()
        nb = lib.sfb_rowslab_blocks(rows)
        part = self.ctx.scratch("colsum.part", nb * c, F32)
        L.check(lib.sfb_colsum(src.data_ptr(), pitch or c, rows, c, out.data_ptr(), 1 if accumulate else 0,
                               part.data_ptr(), _st()), "sfb_colsum")
        ops._count(2)

    def _ln_fwd(self, x: torch.Tensor, x_pitch, rows, c, ln: nn.LayerNorm, out: Optional[Planes], out_f32, mean, rstd):
        lib = L.load()
        L.check(lib.sfb_layernorm_fwd(x.data_ptr(), x_pitch, rows, c, ln.weight.data_ptr(), ln.bias.data_ptr(), ln.eps,
                                      out.hi_ptr() if out is not None else None,
                                      out.lo_ptr() if out is not None else None, _ptr(out_f32), c, _ptr(mean),
                                      _ptr(rstd), _st()), "sfb_layernorm_fwd")
        ops._count()

    def _ln_bwd(self, dy, dy_pitch, x, x_pitch, rows, c, ln: nn.LayerNorm, mean, rstd, dx, dx_pitch, dx_acc,
                param_acc=False):
        lib = L.load()
        nb = lib.sfb_rowslab_blocks(rows)
        part = self.ctx.scratch("ln.part", nb * 2 * c, F32)
        L.check(lib.sfb_layernorm_bwd(dy.data_ptr(), dy_pitch, x.data_ptr(), x_pitch, rows, c, ln.weight.data_ptr(),
                                      mean.data_ptr(), rstd.data_ptr(), dx.data_ptr(), dx_pitch, 1 if dx_acc else 0,
                                      self.ctx.grad_of(ln.weight).data_ptr(), self.ctx.grad_of(ln.bias).data_ptr(),
                                      1 if param_acc else 0, part.data_ptr(), _st()), "sfb_layernorm_bwd")
        ops._count(2)

    def _bgemm(self, a: Planes, a_shape, a_mn, b: Planes, b_shape, b_mn, m, n, k, batch, out, ldd, alpha=1.0,
               accumulate=False):
        """a_shape / b_shape = (pitch, batch_stride) in elements of the storage as laid out in memory."""
        lib = L.load()
        d = L.BgemmDesc()
        d.a_hi, d.a_lo, d.lda, d.batch_stride_a, d.a_mn_major = a.hi_ptr(), a.lo_ptr(), a_shape[0], a_shape[1], int(a_mn)
        d.b_hi, d.b_lo, d.ldb, d.batch_stride_b, d.b_mn_major = b.hi_ptr(), b.lo_ptr(), b_shape[0], b_shape[1], int(b_mn)
        d.m, d.n, d.k, d.batch = m, n, k, batch
        d.out, d.ldd, d.batch_stride_d = out.data_ptr(), ldd, m * ldd
        d.alpha, d.accumulate, d.nsplit = alpha, 1 if accumulate else 0, self.ctx.nsplit
        L.check(lib.sfb_gemm_batched(C.byref(d), _st()), "sfb_gemm_batched")
        ops._count()

    # ================================================================================== forward program
    def _engine_forward(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx, lib = self.ctx, L.load()
        x = inputs[0]
        ctx.device = x.device
        ctx.training = self.training
        if x.device.type != "cuda":
            raise L.NativeLibraryError("slowfast_b200 runs on CUDA devices only (no CPU fallback)")
        B = x.shape[0]
        pe = self.patch_embed.proj
        # ---- patch embedding: clip -> [B, L, 96] (+bias, cls) -------------------------------------------------
        n, cin, t, h, w = x.shape
        xin = ctx.storage(("pe.in",), n, t, h, w, 8)
        xin_p = Planes(xin.hi, xin.lo, n, t, h, w, 8, 0)
        ops.input_pack(x.contiguous().float(), xin_p)
        k3, s3, p3 = tuple(pe.kernel_size), tuple(pe.stride), tuple(pe.padding)
        taps = k3[0] * k3[1] * k3[2]
        E = pe.out_channels
        f = ctx.buf(("pe.f.hi",), (E, taps * 8), BF16)
        flo = ctx.buf(("pe.f.lo",), (E, taps * 8), BF16) if ctx.nsplit == 3 else None
        fm = ops.FilterMat(f, flo, E, taps, 8)
        ops.filter_pack(pe.weight, fm)
        geom = ops.fprop_geom(xin_p, k3, s3, p3)
        T, H, W = geom.out
        assert (T, H, W) == (self.T, self.H, self.W), ((T, H, W), (self.T, self.H, self.W))
        Lt = T * H * W
        ype = ctx.buf(("pe.y",), (B, Lt, E))
        ops.conv_igemm(xin_p, fm, geom, ype, (Lt * E, H * W * E, W * E, E), nsplit=ctx.nsplit)
        x0 = ctx.buf(("x", 0), (B, Lt + 1, E))
        self._tokens_assemble(ype, x0, B, Lt, E, inputs)
        # ---- stochastic depth scales ---------------------------------------------------------------------------
        dp = None
        if ctx.training and max(self.drop_rates) > 0.0:
            nb = len(self.blocks)
            # rates and the device-side step counter are per MODEL (not per arena): captured programs of every input
            # signature read the same two tensors, and the counter keeps advancing across signatures
            rates = getattr(self, "_dp_rates_set", None)
            if rates is None or rates.device != ctx.device:
                rates = torch.tensor([r for r in self.drop_rates for _ in (0, 1)], dtype=torch.float32).to(ctx.device)
                object.__setattr__(self, "_dp_rates_set", rates)
                object.__setattr__(self, "_dp_counter", torch.zeros(1, dtype=torch.int64, device=ctx.device))
            dp = ctx.buf(("dp.scales",), (2 * nb, B))
            L.check(lib.sfb_droppath_scales(dp.data_ptr(), rates.data_ptr(), 2 * nb, B, self._seed,
                                            self._dp_counter.data_ptr(), _st()), "sfb_droppath_scales")
            ops._count(2)
        # ---- blocks --------------------------------------------------------------------------------------------
        saved = []
        cur, thw = x0, [T, H, W]
        for i, (blk, spec) in enumerate(zip(self.blocks, self.specs)):
            cur, thw, sv = self._block_forward(i, blk, spec, cur, thw, B, dp)
            saved.append(sv)
        object.__setattr__(self, "_saved", dict(xin=xin_p, geom=geom, blocks=saved, dp=dp, B=B, thw0=(T, H, W)))
        return self._final_forward(cur, thw, B)

    # ---- hooks the MaskFeat wrapper overrides -------------------------------------------------------------------
    def _tokens_assemble(self, ype, x0, B, Lt, E, inputs) -> None:
        """[cls ; patch embedding + bias] (video_model_builder.py:1166-1181)."""
        pe = self.patch_embed.proj
        L.check(L.load().sfb_tokens_assemble(ype.data_ptr(), pe.bias.data_ptr(), self.cls_token.data_ptr(), B, Lt, E,
                                             x0.data_ptr(), _st()), "sfb_tokens_assemble")
        ops._count()

    def _tokens_split_grad(self, dx, B, Lt, E):
        """Gradient of the token sequence -> patch-embedding output gradient (planes + fp32)."""
        ctx = self.ctx
        dyp = self._rows_planes("pe.dy", B * Lt, E, scratch=True)
        dyf = ctx.scratch("pe.dyf", B * Lt * E, F32)
        L.check(L.load().sfb_tokens_split_grad(dx.data_ptr(), B, Lt, E, dyp.hi_ptr(), dyp.lo_ptr(), dyf.data_ptr(),
                                               _st()), "sfb_tokens_split_grad")
        ops._count()
        return dyp, dyf

    def _final_forward(self, cur: torch.Tensor, thw, B) -> torch.Tensor:
        """Final LayerNorm on the cls rows + TransformerBasicHead (video_model_builder.py:1200-1215)."""
        ctx = self.ctx
        Nf, Cf = cur.shape[1], cur.shape[2]
        cls_n = ctx.buf(("final.cls",), (B, Cf))
        fmean, frstd = ctx.buf(("final.mean",), (B,)), ctx.buf(("final.rstd",), (B,))
        self._ln_fwd(cur, Nf * Cf, B, Cf, self.norm, None, cls_n, fmean, frstd)
        head = self.head
        feat = cls_n
        mask = None
        if ctx.training and head.dropout_rate > 0.0:
            feat = ctx.buf(("head.feat",), (B, Cf))
            feat.copy_(cls_n)
            mask = ctx.buf(("head.mask",), (B, Cf), torch.uint8)
            if getattr(self, "_drop_counter", None) is None or self._drop_counter.device != ctx.device:
                object.__setattr__(self, "_drop_counter", torch.zeros(1, dtype=torch.int64, device=ctx.device))
            ops.dropout_fwd(feat, mask, head.dropout_rate, self._seed + 17, self._drop_counter)
        logits = torch.empty((B, self.num_classes), dtype=F32, device=ctx.device)
        ops.small_linear_fwd(feat, head.projection.weight, head.projection.bias, logits)
        if not ctx.training and head.act_func == "softmax":
            ops.row_softmax(logits)
        self._saved["final"] = (cur, fmean, frstd, feat, mask)
        return logits

    def _final_backward(self, dlogits: torch.Tensor) -> torch.Tensor:
        """Returns the gradient w.r.t. the block stack output [B, Nf, Cf] (zero except the cls rows)."""
        ctx = self.ctx
        sv = self._saved
        B = sv["B"]
        cur, fmean, frstd, feat, mask = sv["final"]
        Nf, Cf = cur.shape[1], cur.shape[2]
        head = self.head
        dfeat = ctx.buf(("head.dfeat",), (B, Cf))
        proj = head.projection
        ops.small_linear_bwd(dlogits, feat, proj.weight, ctx.grad_of(proj.weight), ctx.grad_of(proj.bias), dfeat)
        if mask is not None:
            ops.dropout_bwd(dfeat, mask, head.dropout_rate)
        dx = ctx.scratch("dx.a", B * Nf * Cf, F32).view(B, Nf, Cf)
        ops.zero_f32(ops.f32view(dx.view(B * Nf, Cf)))
        self._ln_bwd(dfeat, Cf, cur, Nf * Cf, B, Cf, self.norm, fmean, frstd, dx, Nf * Cf, False)
        return dx

    def _pool_geom(self, thw, kernel, stride):
        if not _is_pool(kernel, stride):
            return list(thw), False
        return [ops.conv_out_size(i, k, s, k // 2) for i, k, s in zip(thw, kernel, stride)], True

    def _block_forward(self, i, blk: BlockModule, spec, x_in: torch.Tensor, thw, B, dp):
        ctx, lib = self.ctx, L.load()
        # D: block input width, A: attention width (= Do with DIM_MUL_IN_ATT, = D without), Do: block output width
        D, Do, Hn = spec["dim"], spec["dim_out"], spec["heads"]
        A = Do if self.dim_mul_in_att else D
        hd = A // Hn
        T, Hh, W = thw
        Lin = T * Hh * W
        N = Lin + 1
        rows = B * N
        at = blk.attn
        # LN1 -> planes
        xn = self._rows_planes(("b", i, "xn"), rows, D)
        mean1, rstd1 = ctx.buf(("b", i, "m1"), (rows,)), ctx.buf(("b", i, "r1"), (rows,))
        self._ln_fwd(x_in, D, rows, D, blk.norm1, xn, None, mean1, rstd1)
        yqkv = self._lin_fwd(("b", i, "yqkv"), at.qkv, xn)  # [rows, 3A]
        # pooled q, k, v (+ per-head LayerNorm) -> planes [B, H, n', hd]
        pooled, pl, stats, geo = {}, {}, {}, {}
        for j, (name, kern, strd) in enumerate((("q", spec["kq"], spec["sq"]), ("k", spec["kkv"], spec["skv"]),
                                                ("v", spec["kkv"], spec["skv"]))):
            othw, has = self._pool_geom(thw, kern, strd)
            Lo = othw[0] * othw[1] * othw[2]
            d = L.DwPoolDesc()
            d.src, d.src_pitch, d.src_c0 = yqkv.data_ptr(), 3 * A, j * A
            d.bias = _ptr(at.qkv.bias)
            out = ctx.buf(("b", i, "pool", name), (B, Hn, Lo + 1, hd))
            d.out = out.data_ptr()
            d.b, d.heads, d.hd, d.t, d.h, d.w_ = B, Hn, hd, T, Hh, W
            d.ot, d.oh, d.ow = othw
            d.has_pool = 1 if has else 0
            if has:
                d.w = getattr(at, f"pool_{name}").weight.data_ptr()
                d.kt, d.kh, d.kw = kern
                d.st, d.sh, d.sw = strd
            else:
                d.kt = d.kh = d.kw = d.st = d.sh = d.sw = 1
            L.check(lib.sfb_dwpool_fwd(C.byref(d), _st()), "sfb_dwpool_fwd")
            ops._count()
            prow = B * Hn * (Lo + 1)
            pp = self._rows_planes(("b", i, "pl", name), prow, hd)
            if has:
                m_, r_ = ctx.buf(("b", i, "pm", name), (prow,)), ctx.buf(("b", i, "pr", name), (prow,))
                self._ln_fwd(out, hd, prow, hd, getattr(at, f"norm_{name}"), pp, None, m_, r_)
                stats[name] = (m_, r_)
            else:
                ops.split_planes(out.view(1, 1, 1, prow, hd), pp)
            pooled[name], pl[name], geo[name] = out, pp, (othw, has, kern, strd)
        q_thw, k_thw = geo["q"][0], geo["k"][0]
        Lq, Lk = math.prod(q_thw), math.prod(k_thw)
        Nq, Nk = Lq + 1, Lk + 1
        Nkp = ops.pad8(Nk)
        BH = B * Hn
        # fused path (csrc/attn_fused.cu): S, the rel-pos bias, the softmax and P.V in ONE kernel with the scores in shared memory,
        # for the geometry it covers (head_dim 96, 8x7x7 key grid: 12 of MViTv2-S's 16 blocks); else the unfused sequence
        fused = bool(ATTN_FUSED and lib.sfb_attn_fwd_supported(Nk, hd, *k_thw))
        S = None
        if not fused:
            # S = scale * q k^T
            S = ctx.scratch("attn.S", BH * Nq * Nkp, F32).view(BH, Nq, Nkp)
            self._bgemm(pl["q"], (hd, Nq * hd), False, pl["k"], (hd, Nk * hd), False, Nq, Nk, hd, BH, S, Nkp,
                        alpha=hd ** -0.5)
        # decomposed relative positions: RQ = q_nocls . [Rh; Rw; Rt]^T
        rq, Ltp, tab = None, 0, None
        has_rel = hasattr(at, "rel_pos_h")
        if has_rel:
            Lh_, Lw_, Lt_ = at.rel_pos_h.shape[0], at.rel_pos_w.shape[0], at.rel_pos_t.shape[0]
            assert Lh_ == 2 * max(q_thw[1], k_thw[1]) - 1 and Lt_ == 2 * max(q_thw[0], k_thw[0]) - 1, \
                "rel-pos table interpolation is not on the engine path"
            Ltot = Lh_ + Lw_ + Lt_
            Ltp = ops.pad8(Ltot)
            tab_s = ctx.storage(("b", i, "tab"), 1, 1, 1, Ltp, hd)
            tab = Planes(tab_s.hi, tab_s.lo, 1, 1, 1, Ltp, hd, 0)
            tab_s.hi.zero_()
            if tab_s.lo is not None:
                tab_s.lo.zero_()
            off = 0
            for prm in (at.rel_pos_h, at.rel_pos_w, at.rel_pos_t):
                n_ = prm.shape[0]
                sub = Planes(tab_s.hi[..., off:off + n_, :], None if tab_s.lo is None else tab_s.lo[..., off:off + n_, :],
                             1, 1, 1, n_, hd, 0)
                L.check(lib.sfb_split_planes(prm.data_ptr(), n_, hd, hd, sub.hi.data_ptr(),
                                             None if sub.lo is None else sub.lo.data_ptr(), hd, _st()), "split(tab)")
                ops._count()
                off += n_
            rq = ctx.scratch("attn.RQ", BH * Lq * Ltp, F32).view(BH * Lq, Ltp)
            qv = Planes(pl["q"].hi, pl["q"].lo, BH, 1, 1, Nq, hd, 0)
            fm = ops.FilterMat(tab.hi.view(Ltp, hd), None if tab.lo is None else tab.lo.view(Ltp, hd), Ltp, 1, hd)
            ops.conv_igemm(qv, fm, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 1), (1, 1, Lq)), rq,
                           (Lq * Ltp, Lq * Ltp, Lq * Ltp, Ltp), nsplit=ctx.nsplit)
        P = self._rows_planes(("b", i, "P"), BH * Nq, Nkp)
        O = ctx.scratch("attn.O", BH * Nq * hd, F32).view(BH, Nq, hd)
        if fused:
            fd = L.AttnFwdDesc()
            fd.q_hi, fd.q_lo = pl["q"].hi_ptr(), pl["q"].lo_ptr()
            fd.k_hi, fd.k_lo = pl["k"].hi_ptr(), pl["k"].lo_ptr()
            fd.v_hi, fd.v_lo = pl["v"].hi_ptr(), pl["v"].lo_ptr()
            fd.rq, fd.rq_pitch = _ptr(rq), Ltp
            fd.bh, fd.nq, fd.nk, fd.hd = BH, Nq, Nk, hd
            fd.qt, fd.qh, fd.qw = q_thw
            fd.kt, fd.kh, fd.kw = k_thw
            fd.scale = hd ** -0.5
            fd.out = O.data_ptr()
            fd.p_hi, fd.p_lo, fd.p_pitch = P.hi_ptr(), P.lo_ptr(), Nkp   # (the unfused backward reads P)
            fd.nsplit = ctx.nsplit
            L.check(lib.sfb_attn_fwd(C.byref(fd), _st()), "sfb_attn_fwd")
            ops._count()
        else:
            # softmax (+ bias) -> P planes
            sd = L.SoftmaxDesc()
            sd.s, sd.s_pitch = S.data_ptr(), Nkp
            sd.rq, sd.rq_pitch = _ptr(rq), Ltp
            sd.p_hi, sd.p_lo, sd.p_pitch = P.hi_ptr(), P.lo_ptr(), Nkp
            sd.bh, sd.nq, sd.nk = BH, Nq, Nk
            sd.qt, sd.qh, sd.qw = q_thw
            sd.kt, sd.kh, sd.kw = k_thw
            L.check(lib.sfb_softmax_relpos_fwd(C.byref(sd), _st()), "sfb_softmax_relpos_fwd")
            ops._count()
            # O = P v  (v is MN-major: memory [bh][k][hd])
            self._bgemm(P, (Nkp, Nq * Nkp), False, pl["v"], (hd, Nk * hd), True, Nq, hd, Nk, BH, O, hd)
        merged = self._rows_planes(("b", i, "merged"), B * Nq, A)
        L.check(lib.sfb_attn_merge(O.data_ptr(), pl["q"].hi_ptr(), pl["q"].lo_ptr(), B, Hn, Nq, hd,
                                   1 if self.residual_pooling else 0, merged.hi_ptr(), merged.lo_ptr(), _st()),
                "sfb_attn_merge")
        ops._count()
        yproj = self._lin_fwd(("b", i, "yproj"), at.proj, merged)
        # skip path
        if D != A:
            src = self._lin_fwd(("b", i, "yskip"), blk.proj, xn)
            src_bias = blk.proj.bias
        else:
            src, src_bias = x_in.view(rows, D), None
        sq = spec["sq"]
        pool_skip = len(sq) > 0 and math.prod(sq) > 1
        amax = None
        if pool_skip:
            ks = [s + 1 if s > 1 else s for s in sq]
            xsp = ctx.buf(("b", i, "xsp"), (B, Nq, A))
            amax = ctx.buf(("b", i, "amax"), (B, Nq, A), torch.uint8)
            td = L.TokPoolDesc()
            td.x, td.out, td.argmax = src.data_ptr(), xsp.data_ptr(), amax.data_ptr()
            td.b, td.c, td.t, td.h, td.w = B, A, T, Hh, W
            td.ot, td.oh, td.ow = q_thw
            td.kt, td.kh, td.kw = ks
            td.st, td.sh, td.sw = sq
            L.check(lib.sfb_token_maxpool_fwd(C.byref(td), _st()), "sfb_token_maxpool_fwd")
            ops._count()
            src = xsp.view(B * Nq, A)
        rq_rows = B * Nq
        x1 = ctx.buf(("b", i, "x1"), (rq_rows, A))
        s1 = dp[2 * i] if dp is not None else None
        s2 = dp[2 * i + 1] if dp is not None else None
        L.check(lib.sfb_residual_add(src.data_ptr(), _ptr(src_bias), yproj.data_ptr(), at.proj.bias.data_ptr(), _ptr(s1),
                                     rq_rows, A, Nq, x1.data_ptr(), _st()), "sfb_residual_add")
        ops._count()
        # MLP
        x1n = self._rows_planes(("b", i, "x1n"), rq_rows, A)
        mean2, rstd2 = ctx.buf(("b", i, "m2"), (rq_rows,)), ctx.buf(("b", i, "r2"), (rq_rows,))
        self._ln_fwd(x1, A, rq_rows, A, blk.norm2, x1n, None, mean2, rstd2)
        yfc1 = self._lin_fwd(("b", i, "yfc1"), blk.mlp.fc1, x1n)
        hidden = blk.mlp.fc1.out_features
        hpl = self._rows_planes(("b", i, "h"), rq_rows, hidden)
        L.check(lib.sfb_bias_gelu(yfc1.data_ptr(), blk.mlp.fc1.bias.data_ptr(), rq_rows, hidden, hpl.hi_ptr(),
                                  hpl.lo_ptr(), _st()), "sfb_bias_gelu")
        ops._count()
        yfc2 = self._lin_fwd(("b", i, "yfc2"), blk.mlp.fc2, hpl)
        x2 = ctx.buf(("x", i + 1), (B, Nq, Do))
        if A != Do:  # channel expansion in the MLP: the residual is proj(norm2(x1)) (attention.py:507-508)
            base, base_bias = self._lin_fwd(("b", i, "ybase"), blk.proj, x1n), blk.proj.bias
        else:
            base, base_bias = x1, None
        L.check(lib.sfb_residual_add(base.data_ptr(), _ptr(base_bias), yfc2.data_ptr(), blk.mlp.fc2.bias.data_ptr(),
                                     _ptr(s2), rq_rows, Do, Nq, x2.data_ptr(), _st()), "sfb_residual_add")
        ops._count()
        sv = dict(x_in=x_in, thw=list(thw), xn=xn, mean1=mean1, rstd1=rstd1, yqkv=yqkv, pooled=pooled, pl=pl,
                  stats=stats, geo=geo, P=P, tab=tab, Ltp=Ltp, merged=merged, x1=x1, x1n=x1n, mean2=mean2, rstd2=rstd2,
                  yfc1=yfc1, hpl=hpl, amax=amax, pool_skip=pool_skip, q_thw=q_thw, k_thw=k_thw, s1=s1, s2=s2, fused=fused)
        return x2, list(q_thw), sv

    # ================================================================================== backward program
    def _engine_backward(self, dlogits: torch.Tensor):
        ctx, lib = self.ctx, L.load()
        params = [p for p in self.parameters()]
        ctx.begin_backward(params)
        sv = self._saved
        B = sv["B"]
        dx = self._final_backward(dlogits)
        which = "a"
        for i in range(len(self.blocks) - 1, -1, -1):
            which = "b" if which == "a" else "a"
            dx = self._block_backward(i, self.blocks[i], self.specs[i], sv["blocks"][i], dx, B, which)
        # patch embedding
        T, H, W = sv["thw0"]
        Lt = T * H * W
        pe = self.patch_embed.proj
        E = pe.out_channels
        dyp, dyf = self._tokens_split_grad(dx, B, Lt, E)
        self._colsum(dyf, B * Lt, E, ctx.grad_of(pe.bias))
        self._colsum(dx, B, E, ctx.grad_of(self.cls_token).view(E), pitch=(Lt + 1) * E)
        taps = math.prod(pe.kernel_size)
        dwm = ctx.scratch("pe.dwm", E * taps * 8, F32).view(E, taps * 8)
        ops.zero_f32(ops.f32view(dwm))
        ops.conv_wgrad(sv["xin"], Planes(dyp.hi, dyp.lo, B, T, H, W, E, 0), sv["geom"], dwm, nsplit=ctx.nsplit)
        ops.filter_unpack_grad(dwm, ctx.grad_of(pe.weight), 8, accumulate=False)
        return [ctx.grad_of(p) for p in params]

    def _block_backward(self, i, blk: BlockModule, spec, sv, dx2: torch.Tensor, B, which: str) -> torch.Tensor:
        """dx2: gradient w.r.t. the block output [B, Nq, A] (clobbered).  Returns the gradient w.r.t. the block input."""
        ctx, lib = self.ctx, L.load()
        D, Do, Hn = spec["dim"], spec["dim_out"], spec["heads"]
        A = Do if self.dim_mul_in_att else D
        hd = A // Hn
        T, Hh, W = sv["thw"]
        N = T * Hh * W + 1
        rows = B * N
        q_thw, k_thw = sv["q_thw"], sv["k_thw"]
        Lq, Lk = math.prod(q_thw), math.prod(k_thw)
        Nq, Nk = Lq + 1, Lk + 1
        Nkp = ops.pad8(Nk)
        BH = B * Hn
        rq_rows = B * Nq
        at = blk.attn
        hidden = blk.mlp.fc1.out_features
        dx2 = dx2.view(rq_rows, Do)
        # ---------------- MLP branch: x2 = base + s2 * (fc2(gelu(fc1(LN2(x1)) + b1)) + b2),  base = x1 | proj(LN2(x1))
        g2 = self._rows_planes("g.small", rq_rows, Do, scratch=True)
        g2f = ctx.scratch("g.small.f", rq_rows * Do, F32)
        L.check(lib.sfb_scale_split(dx2.data_ptr(), _ptr(sv["s2"]), rq_rows, Do, Nq, g2.hi_ptr(), g2.lo_ptr(),
                                    g2f.data_ptr(), _st()), "sfb_scale_split")
        ops._count()
        dH = ctx.scratch("g.hidden.f", rq_rows * hidden, F32).view(rq_rows, hidden)
        self._lin_bwd(blk.mlp.fc2, g2, g2f, sv["hpl"], dH)
        g1 = self._rows_planes("g.hidden", rq_rows, hidden, scratch=True)
        g1f = ctx.scratch("g.hidden.f2", rq_rows * hidden, F32)
        L.check(lib.sfb_bias_gelu_bwd(dH.data_ptr(), sv["yfc1"].data_ptr(), blk.mlp.fc1.bias.data_ptr(), rq_rows, hidden,
                                      g1.hi_ptr(), g1.lo_ptr(), g1f.data_ptr(), _st()), "sfb_bias_gelu_bwd")
        ops._count()
        dx1n = ctx.scratch("g.small.f2", rq_rows * A, F32).view(rq_rows, A)
        self._lin_bwd(blk.mlp.fc1, g1, g1f, sv["x1n"], dx1n)
        if A != Do:
            # base = proj(LN2(x1)) + b: its gradient is dx2 itself (no stochastic-depth scale on the residual path)
            self._colsum(dx2, rq_rows, Do, ctx.grad_of(blk.proj.bias))
            gb = self._rows_planes("g.base", rq_rows, Do, scratch=True)
            ops.split_planes(dx2.view(1, 1, 1, rq_rows, Do), gb)
            dx1n_b = ctx.scratch("g.base.f", rq_rows * A, F32).view(rq_rows, A)
            self._lin_bwd(blk.proj, gb, None, sv["x1n"], dx1n_b, bias_grad=False)
            ops.add_f32(ops.f32view(dx1n), ops.f32view(dx1n_b))
            dx1 = ctx.scratch("g.x1.f", rq_rows * A, F32).view(rq_rows, A)
            self._ln_bwd(dx1n, A, sv["x1"], A, rq_rows, A, blk.norm2, sv["mean2"], sv["rstd2"], dx1, A, False)
        else:
            # dx1 = dx2 + LN2-branch gradient (in place)
            self._ln_bwd(dx1n, A, sv["x1"], A, rq_rows, A, blk.norm2, sv["mean2"], sv["rstd2"], dx2, A, True)
            dx1 = dx2
        # ---------------- attention branch: x1 = skip + s1 * (proj(merged) + bproj)
        gp = self._rows_planes("g.small", rq_rows, A, scratch=True)
        gpf = ctx.scratch("g.small.f", rq_rows * A, F32)
        L.check(lib.sfb_scale_split(dx1.data_ptr(), _ptr(sv["s1"]), rq_rows, A, Nq, gp.hi_ptr(), gp.lo_ptr(),
                                    gpf.data_ptr(), _st()), "sfb_scale_split")
        ops._count()
        dmerged = ctx.scratch("g.small.f2", rq_rows * A, F32).view(rq_rows, A)
        self._lin_bwd(at.proj, gp, gpf, sv["merged"], dmerged)
        dO = self._rows_planes("attn.dO", BH * Nq, hd, scratch=True)
        dq = ctx.scratch("attn.dq", BH * Nq * hd, F32).view(BH, Nq, hd)
        L.check(lib.sfb_attn_split_grad(dmerged.data_ptr(), B, Hn, Nq, hd, 1 if self.residual_pooling else 0,
                                        dO.hi_ptr(), dO.lo_ptr(), dq.data_ptr(), _st()), "sfb_attn_split_grad")
        ops._count()
        pl, P = sv["pl"], sv["P"]
        dv = ctx.scratch("attn.dv", BH * Nk * hd, F32).view(BH, Nk, hd)
        self._bgemm(P, (Nkp, Nq * Nkp), True, dO, (hd, Nq * hd), True, Nk, hd, Nq, BH, dv, hd)
        dS = self._rows_planes("attn.dS", BH * Nq, Nkp, scratch=True)
        Ltp = sv["Ltp"]
        drq = ctx.scratch("attn.RQ", BH * Lq * Ltp, F32).view(BH * Lq, Ltp) if Ltp else None
        if sv["fused"] and ATTN_FUSED_BWD and Nkp == 400:
            # dP = dO v^T stays in shared memory; dS planes and dRQ come out of one kernel (csrc/attn_fused.cu)
            bd = L.AttnBwdDesc()
            bd.do_hi, bd.do_lo = dO.hi_ptr(), dO.lo_ptr()
            bd.v_hi, bd.v_lo = pl["v"].hi_ptr(), pl["v"].lo_ptr()
            bd.p_hi, bd.p_lo, bd.p_pitch = P.hi_ptr(), P.lo_ptr(), Nkp
            bd.ds_hi, bd.ds_lo, bd.ds_pitch = dS.hi_ptr(), dS.lo_ptr(), Nkp
            bd.drq, bd.rq_pitch = _ptr(drq), Ltp
            bd.bh, bd.nq, bd.nk, bd.hd = BH, Nq, Nk, hd
            bd.qt, bd.qh, bd.qw = q_thw
            bd.kt, bd.kh, bd.kw = k_thw
            bd.nsplit = ctx.nsplit
            L.check(lib.sfb_attn_bwd_ds(C.byref(bd), _st()), "sfb_attn_bwd_ds")
            ops._count()
        else:
            dP = ctx.scratch("attn.S", BH * Nq * Nkp, F32).view(BH, Nq, Nkp)
            self._bgemm(dO, (hd, Nq * hd), False, pl["v"], (hd, Nk * hd), False, Nq, Nk, hd, BH, dP, Nkp)
            sd = L.SoftmaxDesc()
            sd.p_hi, sd.p_lo, sd.p_pitch = P.hi_ptr(), P.lo_ptr(), Nkp
            sd.bh, sd.nq, sd.nk = BH, Nq, Nk
            sd.qt, sd.qh, sd.qw = q_thw
            sd.kt, sd.kh, sd.kw = k_thw
            sd.dp, sd.dp_pitch = dP.data_ptr(), Nkp
            sd.ds_hi, sd.ds_lo, sd.ds_pitch = dS.hi_ptr(), dS.lo_ptr(), Nkp
            sd.drq, sd.rq_pitch = _ptr(drq), Ltp
            L.check(lib.sfb_softmax_relpos_bwd(C.byref(sd), _st()), "sfb_softmax_relpos_bwd")
            ops._count()
        scale = hd ** -0.5
        # dq += scale * dS k ;  dk = scale * dS^T q
        self._bgemm(dS, (Nkp, Nq * Nkp), False, pl["k"], (hd, Nk * hd), True, Nq, hd, Nk, BH, dq, hd, alpha=scale,
                    accumulate=True)
        dk = ctx.scratch("attn.dk", BH * Nk * hd, F32).view(BH, Nk, hd)
        self._bgemm(dS, (Nkp, Nq * Nkp), True, pl["q"], (hd, Nq * hd), True, Nk, hd, Nq, BH, dk, hd, alpha=scale)
        if Ltp:
            tab = sv["tab"]
            drq_p = self._rows_planes("attn.dRQp", BH * Lq, Ltp, scratch=True)
            ops.split_planes(drq.view(1, 1, 1, BH * Lq, Ltp), drq_p)
            # dq[non-cls] += dRQ . tables   (filter = tables^T [hd, Ltp]; B operand MN-major would also do; reuse pack)
            ft = ctx.scratch("attn.tabT.hi", hd * Ltp, BF16).view(hd, Ltp)
            ftl = ctx.scratch("attn.tabT.lo", hd * Ltp, BF16).view(hd, Ltp) if ctx.nsplit == 3 else None
            ft.copy_(tab.hi.view(Ltp, hd).t())
            if ftl is not None:
                ftl.copy_(tab.lo.view(Ltp, hd).t())
            fm = ops.FilterMat(ft, ftl, hd, 1, Ltp)
            drq_v = Planes(drq_p.hi, drq_p.lo, BH, 1, 1, Lq, Ltp, 0)
            ops.conv_igemm(drq_v, fm, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, Lq)), dq,
                           (Nq * hd, Nq * hd, Nq * hd, hd), out_offset=hd, accumulate=True, nsplit=ctx.nsplit)
            # d tables = dRQ^T . q_nocls
            dtab = ctx.scratch("attn.dtab", Ltp * hd, F32).view(Ltp, hd)
            ops.zero_f32(ops.f32view(dtab))
            qv = Planes(pl["q"].hi, pl["q"].lo, BH, 1, 1, Nq, hd, 0)
            ops.conv_wgrad(qv, Planes(drq_p.hi, drq_p.lo, BH, 1, 1, Lq, Ltp, 0),
                           ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 1), (1, 1, Lq)), dtab, nsplit=ctx.nsplit)
            off = 0
            for prm in (at.rel_pos_h, at.rel_pos_w, at.rel_pos_t):
                n_ = prm.shape[0]
                g = ctx.grad_of(prm)
                ops.zero_f32(ops.f32view(g))
                ops.add_f32(ops.f32view(g), ops.F32View(dtab, n_, hd, hd, off * hd))
                off += n_
        # ---------------- pooled q/k/v -> fused qkv gradient
        dyqkv = ctx.scratch("g.qkv.f", rows * 3 * A, F32).view(rows, 3 * A)
        ops.zero_f32(ops.f32view(dyqkv))
        for j, (name, grad) in enumerate((("q", dq), ("k", dk), ("v", dv))):
            othw, has, kern, strd = sv["geo"][name]
            Lo = math.prod(othw)
            prow = BH * (Lo + 1)
            if has:
                dpool = ctx.scratch("attn.dpool", prow * hd, F32).view(prow, hd)
                m_, r_ = sv["stats"][name]
                self._ln_bwd(grad.view(prow, hd), hd, sv["pooled"][name], hd, prow, hd, getattr(at, f"norm_{name}"), m_,
                             r_, dpool, hd, False)
            else:
                dpool = grad.view(prow, hd)
            d = L.DwPoolDesc()
            d.src, d.src_pitch, d.src_c0 = sv["yqkv"].data_ptr(), 3 * A, j * A
            d.bias = _ptr(at.qkv.bias)
            d.b, d.heads, d.hd, d.t, d.h, d.w_ = B, Hn, hd, T, Hh, W
            d.ot, d.oh, d.ow = othw
            d.has_pool = 1 if has else 0
            d.dout, d.dsrc = dpool.data_ptr(), dyqkv.data_ptr()
            dw = None
            if has:
                pool = getattr(at, f"pool_{name}")
                d.w = pool.weight.data_ptr()
                d.kt, d.kh, d.kw = kern
                d.st, d.sh, d.sw = strd
                nb = lib.sfb_dwpool_wgrad_blocks(C.byref(d))
                wp = ctx.scratch("attn.wpart", nb * hd * math.prod(kern), F32)
                d.wpartials = wp.data_ptr()
                dw = ctx.grad_of(pool.weight)
            else:
                d.kt = d.kh = d.kw = d.st = d.sh = d.sw = 1
            L.check(lib.sfb_dwpool_bwd(C.byref(d), _ptr(dw), 0, _st()), "sfb_dwpool_bwd")
            ops._count(3 if has else 1)
        if at.qkv.bias is not None:
            self._colsum(dyqkv, rows, 3 * A, ctx.grad_of(at.qkv.bias))
        gq = self._rows_planes("g.qkv", rows, 3 * A, scratch=True)
        ops.split_planes(dyqkv.view(1, 1, 1, rows, 3 * A), gq)
        dxn = ctx.scratch("g.xn.f", rows * D, F32).view(rows, D)
        self._lin_bwd(at.qkv, gq, None, sv["xn"], dxn, bias_grad=False)
        # ---------------- skip path: d(skip + bias) = dx1
        dsrc = dx1
        if sv["pool_skip"]:
            sq = spec["sq"]
            ks = [s + 1 if s > 1 else s for s in sq]
            dsrc = ctx.scratch("g.skip.f", rows * A, F32).view(rows, A)
            td = L.TokPoolDesc()
            td.argmax = sv["amax"].data_ptr()
            td.b, td.c, td.t, td.h, td.w = B, A, T, Hh, W
            td.ot, td.oh, td.ow = q_thw
            td.kt, td.kh, td.kw = ks
            td.st, td.sh, td.sw = sq
            td.dout, td.dx, td.dx_accumulate = dx1.data_ptr(), dsrc.data_ptr(), 0
            L.check(lib.sfb_token_maxpool_bwd(C.byref(td), _st()), "sfb_token_maxpool_bwd")
            ops._count()
        dx_in = ctx.scratch("dx." + which, rows * D, F32).view(B, N, D)
        if D != A:
            self._colsum(dsrc, rows, A, ctx.grad_of(blk.proj.bias))
            gs = self._rows_planes("g.skip", rows, A, scratch=True)
            ops.split_planes(dsrc.view(1, 1, 1, rows, A), gs)
            dxn2 = ctx.scratch("g.xn.f2", rows * D, F32).view(rows, D)
            self._lin_bwd(blk.proj, gs, None, sv["xn"], dxn2, bias_grad=False)
            ops.add_f32(ops.f32view(dxn), ops.f32view(dxn2))
            self._ln_bwd(dxn, D, sv["x_in"], D, rows, D, blk.norm1, sv["mean1"], sv["rstd1"], dx_in, D, False)
        else:
            # x feeds both the residual path (dsrc) and LN1
            if dsrc.data_ptr() != dx_in.data_ptr():
                dx_in.view(rows, D).copy_(dsrc.view(rows, D))
            self._ln_bwd(dxn, D, sv["x_in"], D, rows, D, blk.norm1, sv["mean1"], sv["rstd1"], dx_in, D, True)
        return dx_in
