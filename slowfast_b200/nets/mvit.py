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
Scope: the MViTv2 configuration family of the reference's Kinetics configs (cls token on, conv pooling, pool_first False,
both DIM_MUL_IN_ATT modes), MViTv1 and ViT with separable absolute position tables (SEP_POS_EMBED) added in the token
assembly, and the mean-token readout (USE_MEAN_POOLING) of the MaskFeat fine-tuning recipes.  A patch embedding with
stride == kernel and no padding (ViT's 2x16x16) is packed into rows and runs as one plain GEMM.
Image recipes (PATCH_2D: configs/ImageNet, in1k fine-tuning): the image [B, 3, H, W] is the memory of a T = 1 clip, so
the Conv2d embedding runs as a (1, kh, kw) convolution on the same kernels; they add the cls-free token layout
(CLS_EMBED_ON False, every token-path kernel in its kCls = 0 instantiation), the joint pos_embed table and the default
readout (norm on every token, then the mean).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn

from .. import ops
from ..engine import EngineModel, Namespace, check_head_act
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
    ps = ([1] if mv.PATCH_2D else []) + list(mv.PATCH_STRIDE)  # video_model_builder.py:832-836
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
    def __init__(self, cin, cout, kernel, stride, padding, conv_2d=False):
        super().__init__()
        conv = nn.Conv2d if conv_2d else nn.Conv3d
        self.proj = conv(cin, cout, kernel_size=tuple(kernel), stride=tuple(stride), padding=tuple(padding))


class TransformerHeadModule(Namespace):
    """TransformerBasicHead container: dropout, projection.  ``detach_final_fc`` (MODEL.DETACH_FINAL_FC,
    head_helper.py:550-551): the features are detached after the dropout, so the backward runs the projection only."""

    def __init__(self, dim_in, num_classes, dropout_rate, act_func, detach_final_fc=False):
        super().__init__()
        check_head_act(act_func)
        if dropout_rate > 0.0:
            self.dropout = nn.Dropout(dropout_rate)
        self.projection = nn.Linear(dim_in, num_classes, bias=True)  # the reference constructs it twice (:515,:517)
        self.projection = nn.Linear(dim_in, num_classes, bias=True)
        self.dropout_rate = dropout_rate
        self.act_func = act_func
        self.detach_final_fc = bool(detach_final_fc)

    def params_after_detach(self) -> List[nn.Parameter]:
        """The parameters behind the detach: the projection's weight and bias."""
        return [self.projection.weight, self.projection.bias]


class B200MViT(EngineModel):
    """MViTv2 on the engine (drop-in for the reference's registered ``MViT``)."""

    def __init__(self, cfg):
        super().__init__(cfg)
        mv = cfg.MVIT
        assert cfg.DATA.TRAIN_CROP_SIZE == cfg.DATA.TEST_CROP_SIZE
        assert mv.MODE == "conv" and not mv.POOL_FIRST
        assert not mv.SEPARATE_QKV and not mv.NORM_STEM
        assert not cfg.DETECTION.ENABLE and mv.NORM == "layernorm"
        assert float(mv.LAYER_SCALE_INIT_VALUE) == 0.0
        self._reject_unsupported(cfg)
        self.specs = block_specs(cfg)
        self.patch_2d = bool(mv.PATCH_2D)
        self.patch_stride = ([1] if self.patch_2d else []) + list(mv.PATCH_STRIDE)
        self.T = cfg.DATA.NUM_FRAMES // self.patch_stride[0]
        self.H = cfg.DATA.TRAIN_CROP_SIZE // self.patch_stride[1]
        self.W = cfg.DATA.TRAIN_CROP_SIZE // self.patch_stride[2]
        self.num_classes = cfg.MODEL.NUM_CLASSES
        self.residual_pooling = bool(mv.RESIDUAL_POOLING)
        self.dim_mul_in_att = bool(mv.DIM_MUL_IN_ATT)
        self.use_abs_pos = bool(mv.USE_ABS_POS)
        self.use_mean_pooling = bool(mv.USE_MEAN_POOLING)
        self.sep_pos_embed = bool(mv.SEP_POS_EMBED)
        self.ncls = 1 if mv.CLS_EMBED_ON else 0  # rows ahead of the token grid in every token tensor
        cin = cfg.DATA.INPUT_CHANNEL_NUM[0]
        # non-overlapping patches (ViT's 2x16x16) are packed into rows and run as one plain GEMM; overlapping ones
        # (MViT's 3x7x7 / stride 2x4x4) take the implicit-GEMM convolution
        self.patchify = (list(mv.PATCH_KERNEL) == list(mv.PATCH_STRIDE) and not any(mv.PATCH_PADDING)
                         and cin * math.prod(mv.PATCH_KERNEL) % 8 == 0)
        self.patch_embed = PatchEmbedModule(cin, mv.EMBED_DIM, mv.PATCH_KERNEL, mv.PATCH_STRIDE, mv.PATCH_PADDING,
                                            conv_2d=self.patch_2d)
        if self.ncls:
            self.cls_token = nn.Parameter(torch.zeros(1, 1, mv.EMBED_DIM))
        if self.use_abs_pos and self.sep_pos_embed:  # video_model_builder.py:892-910 (zeros: no RNG draw here)
            self.pos_embed_spatial = nn.Parameter(torch.zeros(1, self.H * self.W, mv.EMBED_DIM))
            self.pos_embed_temporal = nn.Parameter(torch.zeros(1, self.T, mv.EMBED_DIM))
            self.pos_embed_class = nn.Parameter(torch.zeros(1, 1, mv.EMBED_DIM))
        elif self.use_abs_pos:
            self.pos_embed = nn.Parameter(torch.zeros(1, self.T * self.H * self.W + self.ncls, mv.EMBED_DIM))
        self.blocks = nn.ModuleList()
        for spec in self.specs:
            self.blocks.append(BlockModule(spec, mv.MLP_RATIO, mv.QKV_BIAS, mv.REL_POS_SPATIAL, mv.REL_POS_TEMPORAL,
                                           mv.REL_POS_ZERO_INIT, mv.DIM_MUL_IN_ATT))
        embed = self.specs[-1]["dim_out"]
        self.norm = nn.LayerNorm(embed, eps=1e-6)
        self.head = TransformerHeadModule(embed, self.num_classes, cfg.MODEL.DROPOUT_RATE, cfg.MODEL.HEAD_ACT,
                                          cfg.MODEL.DETACH_FINAL_FC)
        if self.use_abs_pos and self.sep_pos_embed:  # drawn after the head and before cls_token, as the reference does
            nn.init.trunc_normal_(self.pos_embed_spatial, std=0.02)  # (:1057-1077)
            nn.init.trunc_normal_(self.pos_embed_temporal, std=0.02)
            nn.init.trunc_normal_(self.pos_embed_class, std=0.02)
        elif self.use_abs_pos:
            nn.init.trunc_normal_(self.pos_embed, std=0.02)
        if self.ncls:
            nn.init.trunc_normal_(self.cls_token, std=0.02)
        self.apply(self._init_weights)
        self.head.projection.weight.data.mul_(mv.HEAD_INIT_SCALE)
        self.head.projection.bias.data.mul_(mv.HEAD_INIT_SCALE)
        depth = mv.DEPTH
        self.drop_rates = [x.item() for x in torch.linspace(0, float(mv.DROPPATH_RATE), depth)]
        object.__setattr__(self, "_saved", None)

    @staticmethod
    def _reject_unsupported(cfg):
        """Configurations the reference builds but the engine program does not run fail here, naming the option.  The
        option checks run before anything reads the patch geometry."""
        mv = cfg.MVIT
        p2d = bool(mv.PATCH_2D)
        # the cls-free layout and the joint table are built for image patches; video keeps cls-first separable tables
        bad = [
            (not mv.CLS_EMBED_ON and not p2d,
             "MVIT.CLS_EMBED_ON False with 3-D patches (the engine's video token layout keeps the cls token first)"),
            (float(mv.DROPOUT_RATE) != 0.0, "MVIT.DROPOUT_RATE > 0 (position / attention / MLP dropout)"),
            (p2d and any(len(v) != 2 for v in (mv.PATCH_KERNEL, mv.PATCH_STRIDE, mv.PATCH_PADDING)),
             "MVIT.PATCH_2D with a 3-element PATCH_KERNEL / PATCH_STRIDE / PATCH_PADDING (a 2-D embedding takes [h, w])"),
            (p2d and cfg.DATA.NUM_FRAMES != 1, "MVIT.PATCH_2D with DATA.NUM_FRAMES != 1 (images are one frame)"),
            (bool(mv.REV.ENABLE), "MVIT.REV.ENABLE (reversible MViT)"),
            (bool(mv.USE_ABS_POS) and not mv.SEP_POS_EMBED and not p2d,
             "MVIT.USE_ABS_POS with SEP_POS_EMBED False (a joint pos_embed table) with 3-D patches"),
            (bool(mv.USE_ABS_POS) and mv.SEP_POS_EMBED and not mv.CLS_EMBED_ON,
             "MVIT.SEP_POS_EMBED with CLS_EMBED_ON False (separable tables without pos_embed_class)"),
            (bool(mv.USE_FIXED_SINCOS_POS), "MVIT.USE_FIXED_SINCOS_POS (fixed sin-cos position table)"),
            (bool(mv.REL_POS_TEMPORAL) and not mv.REL_POS_SPATIAL,
             "MVIT.REL_POS_TEMPORAL without REL_POS_SPATIAL (a temporal-only relative-position bias)"),
        ]
        for cond, what in bad:
            if cond:
                raise NotImplementedError(f"{what} is not on the engine path")
        bad = []
        for i, s in enumerate(block_specs(cfg)):
            for name, k, st in (("q", s["kq"], s["sq"]), ("kv", s["kkv"], s["skv"])):
                # dwpool_bwd's weight gradient accumulates at most 3 taps per axis (csrc/mvit_ops.cu)
                bad.append((_is_pool(k, st) and max(k) > 3,
                            f"block {i} {name} pooling kernel {list(k)} (more than 3 taps per axis; set "
                            f"MVIT.POOL_KVQ_KERNEL, e.g. [3, 3, 3])"))
        for cond, what in bad:
            if cond:
                raise NotImplementedError(f"{what} is not on the engine path")

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
        names = []  # video_model_builder.py:1095-1116
        if self.cfg.MVIT.ZERO_DECAY_POS_CLS:
            if self.use_abs_pos and self.sep_pos_embed:
                names.extend(["pos_embed_spatial", "pos_embed_temporal", "pos_embed_class"])
            elif self.use_abs_pos:
                names.append("pos_embed")
            if self.cfg.MVIT.REL_POS_SPATIAL:
                names.extend(["rel_pos_h", "rel_pos_w", "rel_pos_hw"])
            if self.cfg.MVIT.REL_POS_TEMPORAL:
                names.extend(["rel_pos_t"])
            if self.ncls:
                names.append("cls_token")
        return names

    def forward(self, x, bboxes=None, return_attn=False):
        assert bboxes is None and not return_attn
        x = [x[0]]
        if self.patch_2d and x[0].dim() != 4:
            raise ValueError(f"MVIT.PATCH_2D takes images [B, C, H, W]; got a {x[0].dim()}-D input of shape "
                             f"{tuple(x[0].shape)}")
        return self._run(x)

    # ================================================================================== helpers
    def _lin_fwd(self, key, lin: nn.Linear, x: Planes) -> torch.Tensor:
        """y[rows, out] = x[rows, in] . W^T  (no bias; consumers add it)."""
        return self._mat_fwd(key, lin.weight, x)

    def _mat_fwd(self, key, weight: torch.Tensor, x: Planes) -> torch.Tensor:
        ctx = self.ctx
        out_f, in_f = weight.shape
        f = ctx.scratch("lin.f.hi", out_f * in_f, BF16).view(out_f, in_f)
        flo = ctx.scratch("lin.f.lo", out_f * in_f, BF16).view(out_f, in_f) if ctx.nsplit == 3 else None
        fm = ops.FilterMat(f, flo, out_f, 1, in_f)
        ops.filter_pack(weight, fm)
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
        part = self.ctx.scratch("colsum.part", ops.colsum_blocks(rows) * c, F32)
        ops.colsum(src, rows, c, out, part, pitch=pitch, accumulate=accumulate)

    def _ln_fwd(self, x: torch.Tensor, x_pitch, rows, c, ln: nn.LayerNorm, out: Optional[Planes], out_f32, mean, rstd):
        ops.layernorm_fwd(x, x_pitch, rows, c, ln.weight, ln.bias, ln.eps, mean, rstd, out=out, out_f32=out_f32)

    def _ln_bwd(self, dy, dy_pitch, x, x_pitch, rows, c, ln: nn.LayerNorm, mean, rstd, dx, dx_pitch, dx_acc,
                param_acc=False):
        ctx = self.ctx
        part = ctx.scratch("ln.part", ops.colsum_blocks(rows) * 2 * c, F32)
        ops.layernorm_bwd(dy, dy_pitch, x, x_pitch, rows, c, ln.weight, mean, rstd, dx, dx_pitch, ctx.grad_of(ln.weight),
                          ctx.grad_of(ln.bias), part, dx_accumulate=dx_acc, param_accumulate=param_acc)

    # ================================================================================== forward program
    def _forward_program(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
        x = inputs[0]
        if self.patch_2d:
            x = x.unsqueeze(2)  # [B, C, H, W] -> [B, C, 1, H, W]: the same memory as a one-frame clip
        B = x.shape[0]
        pe = self.patch_embed.proj
        # ---- patch embedding: clip -> [B, L, 96] (+bias, cls) -------------------------------------------------
        n, cin, t, h, w = x.shape
        k3, s3, p3 = self._pe_geometry()
        E = pe.out_channels
        if self.patchify:
            # stride == kernel: the clip packs into [B*L, cin*kt*kh*kw] rows and the weight is a plain [E, K] matrix
            T, H, W = t // k3[0], h // k3[1], w // k3[2]
            assert (T, H, W) == (self.T, self.H, self.W), ((T, H, W), (self.T, self.H, self.W))
            Lt = T * H * W
            K = cin * math.prod(k3)
            xin_p = self._rows_planes(("pe.rows",), B * Lt, K)
            ops.patchify(x.contiguous().float(), k3, xin_p)
            geom = None
            ype = self._mat_fwd(("pe.y",), pe.weight.view(E, K), xin_p)
        else:
            xin = ctx.storage(("pe.in",), n, t, h, w, 8)
            xin_p = Planes(xin.hi, xin.lo, n, t, h, w, 8, 0)
            ops.input_pack(x.contiguous().float(), xin_p)
            taps = k3[0] * k3[1] * k3[2]
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
        x0 = ctx.buf(("x", 0), (B, Lt + self.ncls, E))
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
            ops.droppath_scales(dp, rates, self._seed, self._dp_counter)
        # ---- blocks --------------------------------------------------------------------------------------------
        saved = []
        cur, thw = x0, [T, H, W]
        for i, (blk, spec) in enumerate(zip(self.blocks, self.specs)):
            cur, thw, sv = self._block_forward(i, blk, spec, cur, thw, B, dp)
            saved.append(sv)
        object.__setattr__(self, "_saved", dict(xin=xin_p, geom=geom, blocks=saved, dp=dp, B=B, thw0=(T, H, W)))
        return self._final_forward(cur, thw, B)

    def _pe_geometry(self):
        """(kernel, stride, padding) of the patch embedding as a 3-D convolution (a Conv2d is its (1, kh, kw) case; its
        [E, C, kh, kw] weight has the tap order of [E, C, 1, kh, kw])."""
        pe = self.patch_embed.proj
        k, s, p = tuple(pe.kernel_size), tuple(pe.stride), tuple(pe.padding)
        if self.patch_2d:
            return (1,) + k, (1,) + s, (0,) + p
        return k, s, p

    # ---- hooks the MaskFeat wrapper overrides -------------------------------------------------------------------
    def _tokens_assemble(self, ype, x0, B, Lt, E, inputs) -> None:
        """[cls ; patch embedding + bias] (+ separable positions) (video_model_builder.py:1166-1199)."""
        pe = self.patch_embed.proj
        if not self.ncls or (self.use_abs_pos and not self.sep_pos_embed):
            # cls-free layout and / or the joint table: (y + bias) + pos[n], the cls row cls + pos[0]
            ops.tokens_assemble_joint(ype, pe.bias, self.cls_token if self.ncls else None,
                                      self.pos_embed if self.use_abs_pos else None, B, Lt, E, x0)
            return
        pos = [None] * 3
        if self.use_abs_pos:
            pos = [self.pos_embed_spatial, self.pos_embed_temporal, self.pos_embed_class]
        ops.tokens_assemble(ype, pe.bias, self.cls_token, *pos, B, Lt, self.H * self.W, E, x0)

    def _tokens_split_grad(self, dx, B, Lt, E):
        """Gradient of the token sequence -> patch-embedding output gradient (planes + fp32)."""
        ctx = self.ctx
        dyp = self._rows_planes("pe.dy", B * Lt, E, scratch=True)
        if not self.ncls:  # the token gradient is the embedding's output gradient
            ops.split_planes(dx.view(1, 1, 1, B * Lt, E), dyp)
            return dyp, dx.view(B * Lt, E)
        dyf = ctx.scratch("pe.dyf", B * Lt * E, F32)
        ops.tokens_split_grad(dx, B, Lt, E, dyp, dyf)
        return dyp, dyf

    def _final_forward(self, cur: torch.Tensor, thw, B) -> torch.Tensor:
        """Final LayerNorm on the cls rows, or on the mean of the other tokens (USE_MEAN_POOLING), or (no cls token, the
        default readout) on every token and then the mean, + TransformerBasicHead (video_model_builder.py:1230-1242)."""
        ctx = self.ctx
        Nf, Cf = cur.shape[1], cur.shape[2]
        if self.use_mean_pooling:
            ln_in, ln_pitch = ctx.buf(("final.pool",), (B, Cf)), Cf
            part = ctx.scratch("final.pool.part", B * ops.segment_slabs(B, Nf - self.ncls) * Cf, F32)
            ops.token_mean_fwd(cur, B, Nf, Cf, ln_in, part, cls=bool(self.ncls))
        else:
            ln_in, ln_pitch = cur, Nf * Cf
        cls_n = ctx.buf(("final.cls",), (B, Cf))
        if not self.use_mean_pooling and not self.ncls:
            # norm on all B * Nf rows, then the per-image mean (deterministic slab sums)
            normed = ctx.buf(("final.normed",), (B * Nf, Cf))
            fmean, frstd = ctx.buf(("final.mean",), (B * Nf,)), ctx.buf(("final.rstd",), (B * Nf,))
            self._ln_fwd(cur, Cf, B * Nf, Cf, self.norm, None, normed, fmean, frstd)
            part = ctx.scratch("final.pool.part", B * ops.segment_slabs(B, Nf) * Cf, F32)
            ops.token_mean_fwd(normed, B, Nf, Cf, cls_n, part, cls=False)
        else:
            fmean, frstd = ctx.buf(("final.mean",), (B,)), ctx.buf(("final.rstd",), (B,))
            self._ln_fwd(ln_in, ln_pitch, B, Cf, self.norm, None, cls_n, fmean, frstd)
        head = self.head
        feat = cls_n
        mask = None
        if ctx.training and head.dropout_rate > 0.0:
            feat = ctx.buf(("head.feat",), (B, Cf))
            feat.copy_(cls_n)
            mask = ctx.buf(("head.mask",), (B, Cf), torch.uint8)
            ops.dropout_fwd(feat, mask, head.dropout_rate, self._seed + 17, self._head_drop_counter())
        logits = torch.empty((B, self.num_classes), dtype=F32, device=ctx.device)
        ops.small_linear_fwd(feat, head.projection.weight, head.projection.bias, logits)
        if not ctx.training:
            ops.head_act(logits, head.act_func)
        self._saved["final"] = (cur, ln_in, ln_pitch, fmean, frstd, feat, mask)
        return logits

    def _final_backward(self, dlogits: torch.Tensor) -> Optional[torch.Tensor]:
        """Returns the gradient w.r.t. the block stack output [B, Nf, Cf] (zero except the cls rows, or zero on the cls
        rows under USE_MEAN_POOLING); None under MODEL.DETACH_FINAL_FC."""
        ctx = self.ctx
        sv = self._saved
        B = sv["B"]
        cur, ln_in, ln_pitch, fmean, frstd, feat, mask = sv["final"]
        Nf, Cf = cur.shape[1], cur.shape[2]
        head = self.head
        dfeat = ctx.buf(("head.dfeat",), (B, Cf))
        proj = head.projection
        if head.detach_final_fc:  # nothing before the detach has a gradient
            ops.small_linear_bwd(dlogits, feat, proj.weight, ctx.grad_of(proj.weight), ctx.grad_of(proj.bias), None)
            return None
        ops.small_linear_bwd(dlogits, feat, proj.weight, ctx.grad_of(proj.weight), ctx.grad_of(proj.bias), dfeat)
        if mask is not None:
            ops.dropout_bwd(dfeat, mask, head.dropout_rate)
        dx = ctx.scratch("dx.a", B * Nf * Cf, F32).view(B, Nf, Cf)
        if self.use_mean_pooling:
            dpool = ctx.scratch("final.dpool", B * Cf, F32).view(B, Cf)
            self._ln_bwd(dfeat, Cf, ln_in, ln_pitch, B, Cf, self.norm, fmean, frstd, dpool, Cf, False)
            ops.token_mean_bwd(dpool, B, Nf, Cf, dx, cls=bool(self.ncls))
            return dx
        if not self.ncls:
            # dmean / Nf on every row, then the norm's backward over all B * Nf rows
            dn = ctx.scratch("final.dnormed", B * Nf * Cf, F32)
            ops.token_mean_bwd(dfeat, B, Nf, Cf, dn, cls=False)
            self._ln_bwd(dn, Cf, cur, Cf, B * Nf, Cf, self.norm, fmean, frstd, dx, Cf, False)
            return dx
        ops.zero_f32(ops.f32view(dx.view(B * Nf, Cf)))
        self._ln_bwd(dfeat, Cf, cur, Nf * Cf, B, Cf, self.norm, fmean, frstd, dx, Nf * Cf, False)
        return dx

    @staticmethod
    def _rel_tables(at) -> list:
        """The block's relative-position tables in RQ column order: [Rh, Rw, Rt], [Rh, Rw] (spatial only) or []."""
        return [getattr(at, n) for n in ("rel_pos_h", "rel_pos_w", "rel_pos_t") if hasattr(at, n)]

    def _pool_geom(self, thw, kernel, stride):
        if not _is_pool(kernel, stride):
            return list(thw), False
        return [ops.conv_out_size(i, k, s, k // 2) for i, k, s in zip(thw, kernel, stride)], True

    def _block_forward(self, i, blk: BlockModule, spec, x_in: torch.Tensor, thw, B, dp):
        ctx = self.ctx
        # D: block input width, A: attention width (= Do with DIM_MUL_IN_ATT, = D without), Do: block output width
        D, Do, Hn = spec["dim"], spec["dim_out"], spec["heads"]
        A = Do if self.dim_mul_in_att else D
        hd = A // Hn
        T, Hh, W = thw
        Lin = T * Hh * W
        nc = self.ncls
        N = Lin + nc
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
            out = ctx.buf(("b", i, "pool", name), (B, Hn, Lo + nc, hd))
            ops.dwpool_fwd(yqkv, j * A, at.qkv.bias, getattr(at, f"pool_{name}").weight if has else None, B, Hn, hd, thw,
                           othw, kern, strd, out, cls=bool(nc))
            prow = B * Hn * (Lo + nc)
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
        Nq, Nk = Lq + nc, Lk + nc
        Nkp = ops.pad8(Nk)
        BH = B * Hn
        # S = scale * q k^T
        S = ctx.scratch("attn.S", BH * Nq * Nkp, F32).view(BH, Nq, Nkp)
        ops.gemm_batched(pl["q"], (hd, Nq * hd), False, pl["k"], (hd, Nk * hd), False, Nq, Nk, hd, BH, S, Nkp,
                         alpha=hd ** -0.5, nsplit=ctx.nsplit)
        # decomposed relative positions: RQ = q_nocls . [Rh; Rw; Rt]^T  (Rt absent: spatial terms only)
        rq, Ltp, tab = None, 0, None
        tabs = self._rel_tables(at)
        if tabs:
            Lh_ = at.rel_pos_h.shape[0]
            assert Lh_ == 2 * max(q_thw[1], k_thw[1]) - 1, "rel-pos table interpolation is not on the engine path"
            assert len(tabs) == 2 or tabs[2].shape[0] == 2 * max(q_thw[0], k_thw[0]) - 1, \
                "rel-pos table interpolation is not on the engine path"
            Ltot = sum(t_.shape[0] for t_ in tabs)
            Ltp = ops.pad8(Ltot)
            tab_s = ctx.storage(("b", i, "tab"), 1, 1, 1, Ltp, hd)
            tab = Planes(tab_s.hi, tab_s.lo, 1, 1, 1, Ltp, hd, 0)
            tab_s.hi.zero_()
            if tab_s.lo is not None:
                tab_s.lo.zero_()
            off = 0
            for prm in tabs:
                n_ = prm.shape[0]
                sub = Planes(tab_s.hi[..., off:off + n_, :], None if tab_s.lo is None else tab_s.lo[..., off:off + n_, :],
                             1, 1, 1, n_, hd, 0)
                ops.split_planes(prm, sub)
                off += n_
            rq = ctx.scratch("attn.RQ", BH * Lq * Ltp, F32).view(BH * Lq, Ltp)
            qv = Planes(pl["q"].hi, pl["q"].lo, BH, 1, 1, Nq, hd, 0)
            fm = ops.FilterMat(tab.hi.view(Ltp, hd), None if tab.lo is None else tab.lo.view(Ltp, hd), Ltp, 1, hd)
            ops.conv_igemm(qv, fm, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, nc), (1, 1, Lq)), rq,
                           (Lq * Ltp, Lq * Ltp, Lq * Ltp, Ltp), nsplit=ctx.nsplit)
        P = self._rows_planes(("b", i, "P"), BH * Nq, Nkp)
        O = ctx.scratch("attn.O", BH * Nq * hd, F32).view(BH, Nq, hd)
        # softmax (+ bias) -> P planes
        ops.softmax_relpos_fwd(S, P, BH, Nq, Nk, q_thw, k_thw, rq=rq, cls=bool(nc), spatial_only=len(tabs) == 2)
        # O = P v  (v is MN-major: memory [bh][k][hd])
        ops.gemm_batched(P, (Nkp, Nq * Nkp), False, pl["v"], (hd, Nk * hd), True, Nq, hd, Nk, BH, O, hd, nsplit=ctx.nsplit)
        merged = self._rows_planes(("b", i, "merged"), B * Nq, A)
        ops.attn_merge(O, pl["q"], B, Hn, Nq, hd, self.residual_pooling, merged, cls=bool(nc))
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
            ops.token_maxpool_fwd(src, B, A, thw, q_thw, ks, sq, xsp, amax, cls=bool(nc))
            src = xsp.view(B * Nq, A)
        rq_rows = B * Nq
        x1 = ctx.buf(("b", i, "x1"), (rq_rows, A))
        s1 = dp[2 * i] if dp is not None else None
        s2 = dp[2 * i + 1] if dp is not None else None
        ops.residual_add(src, src_bias, yproj, at.proj.bias, s1, rq_rows, A, Nq, x1)
        # MLP
        x1n = self._rows_planes(("b", i, "x1n"), rq_rows, A)
        mean2, rstd2 = ctx.buf(("b", i, "m2"), (rq_rows,)), ctx.buf(("b", i, "r2"), (rq_rows,))
        self._ln_fwd(x1, A, rq_rows, A, blk.norm2, x1n, None, mean2, rstd2)
        yfc1 = self._lin_fwd(("b", i, "yfc1"), blk.mlp.fc1, x1n)
        hidden = blk.mlp.fc1.out_features
        hpl = self._rows_planes(("b", i, "h"), rq_rows, hidden)
        ops.bias_gelu(yfc1, blk.mlp.fc1.bias, rq_rows, hidden, hpl)
        yfc2 = self._lin_fwd(("b", i, "yfc2"), blk.mlp.fc2, hpl)
        x2 = ctx.buf(("x", i + 1), (B, Nq, Do))
        if A != Do:  # channel expansion in the MLP: the residual is proj(norm2(x1)) (attention.py:507-508)
            base, base_bias = self._lin_fwd(("b", i, "ybase"), blk.proj, x1n), blk.proj.bias
        else:
            base, base_bias = x1, None
        ops.residual_add(base, base_bias, yfc2, blk.mlp.fc2.bias, s2, rq_rows, Do, Nq, x2)
        sv = dict(x_in=x_in, thw=list(thw), xn=xn, mean1=mean1, rstd1=rstd1, yqkv=yqkv, pooled=pooled, pl=pl,
                  stats=stats, geo=geo, P=P, tab=tab, Ltp=Ltp, merged=merged, x1=x1, x1n=x1n, mean2=mean2, rstd2=rstd2,
                  yfc1=yfc1, hpl=hpl, amax=amax, pool_skip=pool_skip, q_thw=q_thw, k_thw=k_thw, s1=s1, s2=s2)
        return x2, list(q_thw), sv

    # ================================================================================== backward program
    def _backward_program(self, dlogits: torch.Tensor) -> None:
        ctx = self.ctx
        sv = self._saved
        B = sv["B"]
        dx = self._final_backward(dlogits)
        if dx is None:
            return
        which = "a"
        for i in range(len(self.blocks) - 1, -1, -1):
            which = "b" if which == "a" else "a"
            dx = self._block_backward(i, self.blocks[i], self.specs[i], sv["blocks"][i], dx, B, which)
        # patch embedding
        T, H, W = sv["thw0"]
        Lt = T * H * W
        pe = self.patch_embed.proj
        E = pe.out_channels
        if self.use_abs_pos and not self.sep_pos_embed:
            ops.pos_embed_joint_bwd(dx, B, Lt + self.ncls, E, ctx.grad_of(self.pos_embed))
        elif self.use_abs_pos:
            part = ctx.scratch("pos.part", T * ops.segment_slabs(T, H * W) * E, F32)
            ops.pos_embed_sep_bwd(dx, B, T, H * W, E, ctx.grad_of(self.pos_embed_spatial),
                                  ctx.grad_of(self.pos_embed_temporal), ctx.grad_of(self.pos_embed_class), part)
        dyp, dyf = self._tokens_split_grad(dx, B, Lt, E)
        self._colsum(dyf, B * Lt, E, ctx.grad_of(pe.bias))
        if self.ncls:
            self._colsum(dx, B, E, ctx.grad_of(self.cls_token).view(E), pitch=(Lt + 1) * E)
        if self.patchify:
            xr = sv["xin"]
            gw = ctx.grad_of(pe.weight).view(E, xr.c)
            ops.zero_f32(ops.f32view(gw))
            ops.conv_wgrad(xr, dyp, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (xr.t, xr.h, xr.w)), gw,
                           nsplit=ctx.nsplit)
            return
        taps = math.prod(pe.kernel_size)
        dwm = ctx.scratch("pe.dwm", E * taps * 8, F32).view(E, taps * 8)
        ops.zero_f32(ops.f32view(dwm))
        ops.conv_wgrad(sv["xin"], Planes(dyp.hi, dyp.lo, B, T, H, W, E, 0), sv["geom"], dwm, nsplit=ctx.nsplit)
        ops.filter_unpack_grad(dwm, ctx.grad_of(pe.weight), 8, accumulate=False)

    def _block_backward(self, i, blk: BlockModule, spec, sv, dx2: torch.Tensor, B, which: str) -> torch.Tensor:
        """dx2: gradient w.r.t. the block output [B, Nq, A] (clobbered).  Returns the gradient w.r.t. the block input."""
        ctx = self.ctx
        D, Do, Hn = spec["dim"], spec["dim_out"], spec["heads"]
        A = Do if self.dim_mul_in_att else D
        hd = A // Hn
        T, Hh, W = sv["thw"]
        nc = self.ncls
        N = T * Hh * W + nc
        rows = B * N
        q_thw, k_thw = sv["q_thw"], sv["k_thw"]
        Lq, Lk = math.prod(q_thw), math.prod(k_thw)
        Nq, Nk = Lq + nc, Lk + nc
        Nkp = ops.pad8(Nk)
        BH = B * Hn
        rq_rows = B * Nq
        at = blk.attn
        hidden = blk.mlp.fc1.out_features
        dx2 = dx2.view(rq_rows, Do)
        # ---------------- MLP branch: x2 = base + s2 * (fc2(gelu(fc1(LN2(x1)) + b1)) + b2),  base = x1 | proj(LN2(x1))
        g2 = self._rows_planes("g.small", rq_rows, Do, scratch=True)
        g2f = ctx.scratch("g.small.f", rq_rows * Do, F32)
        ops.scale_split(dx2, sv["s2"], rq_rows, Do, Nq, g2, g2f)
        dH = ctx.scratch("g.hidden.f", rq_rows * hidden, F32).view(rq_rows, hidden)
        self._lin_bwd(blk.mlp.fc2, g2, g2f, sv["hpl"], dH)
        g1 = self._rows_planes("g.hidden", rq_rows, hidden, scratch=True)
        g1f = ctx.scratch("g.hidden.f2", rq_rows * hidden, F32)
        ops.bias_gelu_bwd(dH, sv["yfc1"], blk.mlp.fc1.bias, rq_rows, hidden, g1, g1f)
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
        ops.scale_split(dx1, sv["s1"], rq_rows, A, Nq, gp, gpf)
        dmerged = ctx.scratch("g.small.f2", rq_rows * A, F32).view(rq_rows, A)
        self._lin_bwd(at.proj, gp, gpf, sv["merged"], dmerged)
        dO = self._rows_planes("attn.dO", BH * Nq, hd, scratch=True)
        dq = ctx.scratch("attn.dq", BH * Nq * hd, F32).view(BH, Nq, hd)
        ops.attn_split_grad(dmerged, B, Hn, Nq, hd, self.residual_pooling, dO, dq, cls=bool(nc))
        pl, P = sv["pl"], sv["P"]
        dv = ctx.scratch("attn.dv", BH * Nk * hd, F32).view(BH, Nk, hd)
        ops.gemm_batched(P, (Nkp, Nq * Nkp), True, dO, (hd, Nq * hd), True, Nk, hd, Nq, BH, dv, hd, nsplit=ctx.nsplit)
        dS = self._rows_planes("attn.dS", BH * Nq, Nkp, scratch=True)
        Ltp = sv["Ltp"]
        drq = ctx.scratch("attn.RQ", BH * Lq * Ltp, F32).view(BH * Lq, Ltp) if Ltp else None
        dP = ctx.scratch("attn.S", BH * Nq * Nkp, F32).view(BH, Nq, Nkp)
        ops.gemm_batched(dO, (hd, Nq * hd), False, pl["v"], (hd, Nk * hd), False, Nq, Nk, hd, BH, dP, Nkp,
                         nsplit=ctx.nsplit)
        tabs = self._rel_tables(at)
        ops.softmax_relpos_bwd(P, dP, dS, BH, Nq, Nk, q_thw, k_thw, drq=drq, cls=bool(nc), spatial_only=len(tabs) == 2)
        scale = hd ** -0.5
        # dq += scale * dS k ;  dk = scale * dS^T q
        ops.gemm_batched(dS, (Nkp, Nq * Nkp), False, pl["k"], (hd, Nk * hd), True, Nq, hd, Nk, BH, dq, hd, alpha=scale,
                         accumulate=True, nsplit=ctx.nsplit)
        dk = ctx.scratch("attn.dk", BH * Nk * hd, F32).view(BH, Nk, hd)
        ops.gemm_batched(dS, (Nkp, Nq * Nkp), True, pl["q"], (hd, Nq * hd), True, Nk, hd, Nq, BH, dk, hd, alpha=scale,
                         nsplit=ctx.nsplit)
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
                           (Nq * hd, Nq * hd, Nq * hd, hd), out_offset=nc * hd, accumulate=True, nsplit=ctx.nsplit)
            # d tables = dRQ^T . q_nocls
            dtab = ctx.scratch("attn.dtab", Ltp * hd, F32).view(Ltp, hd)
            ops.zero_f32(ops.f32view(dtab))
            qv = Planes(pl["q"].hi, pl["q"].lo, BH, 1, 1, Nq, hd, 0)
            ops.conv_wgrad(qv, Planes(drq_p.hi, drq_p.lo, BH, 1, 1, Lq, Ltp, 0),
                           ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, nc), (1, 1, Lq)), dtab, nsplit=ctx.nsplit)
            off = 0
            for prm in tabs:
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
            prow = BH * (Lo + nc)
            if has:
                dpool = ctx.scratch("attn.dpool", prow * hd, F32).view(prow, hd)
                m_, r_ = sv["stats"][name]
                self._ln_bwd(grad.view(prow, hd), hd, sv["pooled"][name], hd, prow, hd, getattr(at, f"norm_{name}"), m_,
                             r_, dpool, hd, False)
            else:
                dpool = grad.view(prow, hd)
            w = dw = wp = None
            if has:
                w = getattr(at, f"pool_{name}").weight
                dw = ctx.grad_of(w)
                wp = ctx.scratch("attn.wpart", ops.dwpool_wgrad_blocks(B, Hn, othw) * hd * math.prod(kern), F32)
            ops.dwpool_bwd(sv["yqkv"], j * A, at.qkv.bias, w, B, Hn, hd, sv["thw"], othw, kern, strd, dpool, dyqkv, dw=dw,
                           wpartials=wp, cls=bool(nc))
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
            ops.token_maxpool_bwd(dx1, sv["amax"], B, A, sv["thw"], q_thw, ks, sq, dsrc, cls=bool(nc))
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
