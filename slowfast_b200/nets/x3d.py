"""X3D (video_model_builder.py:664 X3D; resnet_helper.py:122 X3DTransform; stem_helper.py:204 X3DStem;
operators.py:14 SE; head_helper.py:352 X3DHead) on the engine.

Module tree and parameter names mirror the reference (``s1.pathway0_stem.{conv_xy,conv,bn}``,
``s{2..5}.pathway0_res{i}.{branch1,branch1_bn,branch2.{a,a_bn,b,b_bn,se.fc1,se.fc2,c,c_bn}}``,
``head.{conv_5,conv_5_bn,lin_5,projection}``), so checkpoints, the optimizer's parameter grouping and
``build_model`` work unchanged.  Execution:

  stem   : conv_xy 1x3x3 (wgmma implicit GEMM, C_in padded 3->8) -> channelwise 5x1x1 conv with the BatchNorm
           partials in its epilogue -> fused BN+ReLU
  block  : a (1x1x1 GEMM + BN stats) -> BN+ReLU -> channelwise 3x3x3 (+ BN partials per sample tile, which also
           ARE the SE average pool) -> [SE FCs, one block per sample] -> BN*gate -> Swish -> c (1x1x1 GEMM + BN)
           -> relu(shortcut + c_bn) in one pass.  X3D-M's 54- / 108-wide bottlenecks run padded to 56 / 112
           channels; pad channels carry exact zeros.
  head   : conv_5 + BN + ReLU -> global average pool -> lin_5 -> ReLU -> dropout -> Linear

X3D is HBM-bound everywhere (SURVEY.md section 8d: 9.47 GFLOP vs 366 MB per clip): the kernels that matter are the
channelwise convolutions and the fused normalisation passes in csrc/x3d_ops.cu.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn

from .. import lib as L
from .. import ops
from ..config import nsplit_of
from ..engine import Act, ConvBN, Ctx, Namespace, bump_num_batches_tracked
from ..ops import F32
from .resnet import STAGE_DEPTH, _conv, _VideoResNetBase, init_resnet_weights


def round_width(width, multiplier, min_width=1, divisor=1):
    """slowfast/models/utils.py:10 (channel rounding of the X3D expansion)."""
    if not multiplier:
        return width
    width *= multiplier
    min_width = min_width or divisor
    width_out = max(min_width, int(width + divisor / 2) // divisor * divisor)
    if width_out < 0.9 * width:
        width_out += divisor
    return int(width_out)


def se_width(dim_in: int, ratio: float) -> int:
    """operators.py:17 SE._round_width (min_width = divisor = 8)."""
    return round_width(dim_in, ratio, min_width=8, divisor=8)


class X3DStemModule(Namespace):
    """X3DStem parameter container: conv_xy, conv (channelwise temporal), bn."""

    def __init__(self, cin, cout, k, stride, pad, eps=1e-5, mmt=0.1):
        super().__init__()
        self.conv_xy = _conv(cin, cout, (1, k[1], k[2]), (1, stride[1], stride[2]), (0, pad[1], pad[2]))
        self.conv = nn.Conv3d(cout, cout, kernel_size=(k[0], 1, 1), stride=(stride[0], 1, 1), padding=(pad[0], 0, 0),
                              bias=False, groups=cout)
        self.bn = nn.BatchNorm3d(cout, eps=eps, momentum=mmt)
        self.relu = nn.ReLU(True)


class SEModule(Namespace):
    """SE parameter container: fc1, fc2 (1x1x1 Conv3d with bias)."""

    def __init__(self, dim_in, ratio):
        super().__init__()
        self.avg_pool = nn.Identity()
        dim_fc = se_width(dim_in, ratio)
        self.fc1 = nn.Conv3d(dim_in, dim_fc, 1, bias=True)
        self.fc1_act = nn.ReLU()
        self.fc2 = nn.Conv3d(dim_fc, dim_in, 1, bias=True)
        self.fc2_sig = nn.Sigmoid()


class X3DTransformModule(Namespace):
    """X3DTransform parameter container: a, a_bn, b (channelwise), b_bn, [se], c, c_bn."""

    def __init__(self, dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, block_idx, se_ratio=0.0625,
                 swish_inner=True, eps=1e-5, mmt=0.1):
        super().__init__()
        s1, s3 = (stride, 1) if stride_1x1 else (1, stride)
        self.a = _conv(dim_in, dim_inner, (1, 1, 1), (1, s1, s1), (0, 0, 0))
        self.a_bn = nn.BatchNorm3d(dim_inner, eps=eps, momentum=mmt)
        self.a_relu = nn.ReLU(True)
        self.b = nn.Conv3d(dim_inner, dim_inner, [temp_k, 3, 3], stride=[1, s3, s3], padding=[temp_k // 2, 1, 1],
                           groups=dim_inner, bias=False, dilation=[1, 1, 1])
        self.b_bn = nn.BatchNorm3d(dim_inner, eps=eps, momentum=mmt)
        if se_ratio > 0.0 and (block_idx + 1) % 2:
            self.se = SEModule(dim_inner, se_ratio)
        self.b_relu = nn.Identity() if swish_inner else nn.ReLU(True)  # Swish has no parameters
        self.swish = bool(swish_inner)
        self.c = _conv(dim_inner, dim_out, (1, 1, 1), (1, 1, 1), (0, 0, 0))
        self.c_bn = nn.BatchNorm3d(dim_out, eps=eps, momentum=mmt)
        self.c_bn.transform_final_bn = True


class X3DBlockModule(Namespace):
    """ResBlock with an X3DTransform branch (+ engine program)."""

    def __init__(self, name, dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, block_idx, ctx: Ctx,
                 eps=1e-5, mmt=0.1):
        super().__init__()
        if dim_in != dim_out or stride != 1:
            self.branch1 = _conv(dim_in, dim_out, (1, 1, 1), (1, stride, stride), (0, 0, 0))
            self.branch1_bn = nn.BatchNorm3d(dim_out, eps=eps, momentum=mmt)
        self.branch2 = X3DTransformModule(dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, block_idx, eps=eps,
                                          mmt=mmt)
        self.relu = nn.ReLU(True)
        self._n, self._ctx = name, ctx
        self._dim_inner, self._dim_out = dim_inner, dim_out
        object.__setattr__(self, "_units", None)

    def units(self):
        if self._units is None:
            b2, n, ctx = self.branch2, self._n, self._ctx
            u = {"a": ConvBN(n + ".a", b2.a, b2.a_bn, ctx), "c": ConvBN(n + ".c", b2.c, b2.c_bn, ctx)}
            if hasattr(self, "branch1"):
                u["s"] = ConvBN(n + ".branch1", self.branch1, self.branch1_bn, ctx)
            object.__setattr__(self, "_units", u)
        return self._units

    def out_dims(self, t, h, w):
        a, b = self.branch2.a, self.branch2.b
        t, h, w = self.units()["a"].out_dims(t, h, w)
        return tuple(ops.conv_out_size(i, k, s, p) for i, k, s, p in zip((t, h, w), b.kernel_size, b.stride,
                                                                         b.padding))

    # ---------------------------------------------------------------------------------------- forward
    def run_forward(self, x: Act, out: Act) -> None:
        ctx, u, nm, b2 = self._ctx, self.units(), self._n, self.branch2
        n = x.dims[0]
        ya = u["a"].fprop(x.planes)
        # relu(a_bn(ya)) is never written: the channelwise conv applies a's BatchNorm + ReLU while reading ya, and
        # the backward kernels recompute it the same way; xa only owns the fp32 gradient
        xa = Act(ctx.storage((nm, "xa"), *ya.shape, planes=False))
        a_affine = (u["a"].scale, u["a"].shift, True)
        # ---- b: channelwise conv + BN partials
        c, cp = self._dim_inner, ya.shape[-1]
        g = ops.DwGeom(n, *xa.dims[1:], tuple(b2.b.kernel_size), tuple(b2.b.stride), tuple(b2.b.padding))
        ot, oh, ow = g.out
        rps = ot * oh * ow
        yb = ctx.buf((nm, "yb"), (n, ot, oh, ow, cp))
        m_tiles, tps = ops.dwconv_tiles(g, cp, True)
        stats = ctx.buf((nm, "b.stats"), (2, c, m_tiles))
        ops.dwconv_fwd(g, cp, c, b2.b.weight, ops.f32view(yb), stats, x_f32=ops.f32view(ya), in_affine=a_affine)
        bb = {k: ctx.buf((nm, "b." + k), (cp,), zero=True) for k in ("scale", "shift", "mean", "invstd")}
        bn = b2.b_bn
        ops.bn_finalize(stats, m_tiles, c, n * rps, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                        bn.momentum if bn.momentum is not None else 0.1, bn.eps, ctx.training, bb["scale"],
                        bb["shift"], bb["mean"], bb["invstd"])
        # ---- SE gate
        gate = None
        se = getattr(b2, "se", None)
        sed = None
        if se is not None:
            f = se.fc1.out_channels
            sed = L.SeDesc()
            sed.n, sed.c, sed.c_pad, sed.f, sed.rows_per_sample = n, c, cp, f, rps
            sed.tiles_per_sample, sed.m_tiles = tps, m_tiles
            sed.stats, sed.scale, sed.shift = stats.data_ptr(), bb["scale"].data_ptr(), bb["shift"].data_ptr()
            sed.mean, sed.invstd = bb["mean"].data_ptr(), bb["invstd"].data_ptr()
            sed.w1, sed.b1 = se.fc1.weight.data_ptr(), se.fc1.bias.data_ptr()
            sed.w2, sed.b2 = se.fc2.weight.data_ptr(), se.fc2.bias.data_ptr()
            sv = {k: ctx.buf((nm, "se." + k), (n, cp)) for k in ("ymean", "avg", "gate")}
            sv["hid"] = ctx.buf((nm, "se.hid"), (n, f))
            sed.ymean, sed.avg, sed.hid, sed.gate = (sv[k].data_ptr() for k in ("ymean", "avg", "hid", "gate"))
            ops.se_fwd(sed)
            gate = sv["gate"]
        act = ops.ACT_SWISH if b2.swish else ops.ACT_RELU
        xb = Act(ctx.storage((nm, "xb"), n, ot, oh, ow, cp))
        ops.bnact_fwd(ops.f32view(yb), bb["scale"], bb["shift"], gate, act, rps, xb.planes)
        # ---- c + shortcut
        yc = u["c"].fprop(xb.planes)
        if "s" in u:
            ys = u["s"].fprop(x.planes)
            ops.bn_apply(ops.f32view(yc), u["c"].scale, u["c"].shift, out.planes, relu=True, y2=ops.f32view(ys),
                         scale2=u["s"].scale, shift2=u["s"].shift)
        else:
            ops.bn_apply(ops.f32view(yc), u["c"].scale, u["c"].shift, out.planes, relu=True, res=x.planes)
        object.__setattr__(self, "_saved", (x, xa, xb, out, g, yb, bb, gate, sed, act, ya, a_affine))

    # ---------------------------------------------------------------------------------------- backward
    def run_backward(self) -> None:
        ctx, u, b2 = self._ctx, self.units(), self.branch2
        x, xa, xb, out, g, yb, bb, gate, sed, act, ya, a_affine = self._saved
        dout = out.grad_view()
        if "s" in u:
            u["s"].bwd(dout, out.planes, x)
            u["c"].bwd(dout, out.planes, xb)
        else:
            acc = x.s.grad_written
            u["c"].bwd(dout, out.planes, xb, dres=x.grad_view(), dres_accumulate=acc)
            x.s.grad_written = True
        dyb = bn_gate_act_backward(ctx, ops.f32view(yb), bb, gate, sed, act, g.n, self._dim_inner, xb.grad_view(),
                                   b2.b_bn, getattr(b2, "se", None))
        ops.dwconv_bwd(g, yb.shape[-1], self._dim_inner, b2.b.weight, dyb, ctx.grad_of(b2.b.weight), None,
                       x_f32=ops.f32view(ya), in_affine=a_affine, dx=xa.grad_view(), dx_accumulate=False)
        xa.s.grad_written = True
        u["a"].bwd(xa.grad_view(), None, x, mask_from_y=True)


def bn_gate_act_backward(ctx: Ctx, y: ops.F32View, bb, gate, sed: Optional["L.SeDesc"], act: int, n: int, c: int,
                         dout: ops.F32View, bn: nn.BatchNorm3d, se) -> ops.F32View:
    """Backward of  act( BN(y) * gate )  (+ the SE branch feeding ``gate``): returns dL/dy as an fp32 view of a
    scratch tensor, and writes dgamma / dbeta (and the SE parameter gradients) into their gradient slots."""
    cp = y.c
    rps = y.rows // n
    tps2 = ops.bnact_tiles_per_sample(y.rows, rps)
    partials = ctx.scratch("x3d.partials", n * tps2 * 2 * cp, F32)
    ops.bnact_bwd_reduce(y, bb["scale"], bb["shift"], bb["mean"], bb["invstd"], gate, act, rps, dout, partials)
    d = L.SeDesc()
    if sed is not None:  # forward pointers (stats are not needed again)
        for k, _ in L.SeDesc._fields_:
            setattr(d, k, getattr(sed, k))
    d.n, d.c, d.c_pad, d.rows_per_sample = n, c, cp, rps
    d.mean, d.invstd = bb["mean"].data_ptr(), bb["invstd"].data_ptr()
    d.partials, d.tiles2_per_sample = partials.data_ptr(), tps2
    d.a12 = ctx.scratch("x3d.a12", n * 2 * cp, F32).data_ptr()
    coef = ctx.scratch("x3d.coef", 3 * cp, F32)
    d.coef = coef.data_ptr()
    d.gamma, d.beta = bn.weight.data_ptr(), bn.bias.data_ptr()
    d.dgamma, d.dbeta = ctx.grad_of(bn.weight).data_ptr(), ctx.grad_of(bn.bias).data_ptr()
    d.training = 1 if ctx.training else 0
    davg = None
    if se is not None:
        f = se.fc1.out_channels
        d.has_se = 1
        d.do2 = ctx.scratch("x3d.do2", n * cp, F32).data_ptr()
        d.dhid = ctx.scratch("x3d.dhid", n * f, F32).data_ptr()
        davg = ctx.scratch("x3d.davg", n * cp, F32)
        d.davg = davg.data_ptr()
        d.dw1, d.db1 = ctx.grad_of(se.fc1.weight).data_ptr(), ctx.grad_of(se.fc1.bias).data_ptr()
        d.dw2, d.db2 = ctx.grad_of(se.fc2.weight).data_ptr(), ctx.grad_of(se.fc2.bias).data_ptr()
    else:
        d.has_se, d.f = 0, 0
    ops.se_bwd(d)
    dy_t = ctx.scratch("x3d.dy", y.rows * cp, F32).view(y.rows, cp)
    dy = ops.f32view(dy_t)
    ops.bnact_bwd_apply(y, bb["scale"], bb["shift"], bb["mean"], bb["invstd"], gate, act, rps, dout, davg, coef, dy)
    return dy


class X3DStageModule(Namespace):
    """ResStage container of X3D blocks: pathway0_res{i}."""

    def __init__(self, name, dim_in, dim_out, dim_inner, temp_k, stride, num_blocks, stride_1x1, ctx: Ctx):
        super().__init__()
        self.num_blocks = num_blocks
        for i in range(num_blocks):
            blk = X3DBlockModule(f"{name}.pathway0_res{i}", dim_in if i == 0 else dim_out, dim_out, temp_k,
                                 stride if i == 0 else 1, dim_inner, stride_1x1, i, ctx)
            self.add_module(f"pathway0_res{i}", blk)

    def blocks(self) -> List[X3DBlockModule]:
        return [getattr(self, f"pathway0_res{i}") for i in range(self.num_blocks)]


class X3DHeadModule(Namespace):
    """X3DHead parameter container: conv_5, conv_5_bn, lin_5, projection."""

    def __init__(self, dim_in, dim_inner, dim_out, num_classes, dropout_rate, act_func, bn_lin5_on, eps=1e-5,
                 mmt=0.1):
        super().__init__()
        assert not bn_lin5_on, "X3D.BN_LIN5 is not on the engine path"
        self.conv_5 = _conv(dim_in, dim_inner, (1, 1, 1), (1, 1, 1), (0, 0, 0))
        self.conv_5_bn = nn.BatchNorm3d(dim_inner, eps=eps, momentum=mmt)
        self.conv_5_relu = nn.ReLU(True)
        self.avg_pool = nn.Identity()
        self.lin_5 = _conv(dim_inner, dim_out, (1, 1, 1), (1, 1, 1), (0, 0, 0))
        self.lin_5_relu = nn.ReLU(True)
        if dropout_rate > 0.0:
            self.dropout = nn.Dropout(dropout_rate)
        self.projection = nn.Linear(dim_out, num_classes, bias=True)
        if act_func not in ("softmax", "none"):
            raise NotImplementedError(f"head activation {act_func!r} is not on the engine path")
        self.act_func = act_func
        self.dropout_rate = dropout_rate


class B200X3D(_VideoResNetBase):
    """X3D network (video_model_builder.py:664) on the engine."""

    num_pathways = 1

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        assert cfg.BN.NORM_TYPE == "batchnorm", "only BN.NORM_TYPE=batchnorm is on the engine path"
        assert cfg.RESNET.TRANS_FUNC == "x3d_transform" and cfg.MODEL.ARCH == "x3d"
        assert cfg.X3D.CHANNELWISE_3x3x3, "X3D with dense 3x3x3 convolutions is not on the engine path"
        assert not cfg.DETECTION.ENABLE
        assert float(cfg.MODEL.DROPCONNECT_RATE) == 0.0, "drop-connect is not on the engine path (0.0 in X3D yamls)"
        assert all(len(l) == 0 for st in cfg.NONLOCAL.LOCATION for l in st)
        self.ctx = Ctx(nsplit_of(cfg))
        ctx = self.ctx
        exp_stage = 2.0
        dim_c1 = cfg.X3D.DIM_C1
        dim_res2 = round_width(dim_c1, exp_stage, divisor=8) if cfg.X3D.SCALE_RES2 else dim_c1
        dim_res3 = round_width(dim_res2, exp_stage, divisor=8)
        dim_res4 = round_width(dim_res3, exp_stage, divisor=8)
        dim_res5 = round_width(dim_res4, exp_stage, divisor=8)
        block_basis = [[1, dim_res2, 2], [2, dim_res3, 2], [5, dim_res4, 2], [3, dim_res5, 2]]
        assert cfg.RESNET.DEPTH in STAGE_DEPTH
        w_mul, d_mul = cfg.X3D.WIDTH_FACTOR, cfg.X3D.DEPTH_FACTOR
        dim_res1 = round_width(dim_c1, w_mul)
        # temporal kernels (video_model_builder.py:91-97): conv1 5, res2..res5 3
        self.s1 = Namespace()
        self.s1.add_module("pathway0_stem", X3DStemModule(cfg.DATA.INPUT_CHANNEL_NUM[0], dim_res1, (5, 3, 3),
                                                          (1, 2, 2), (2, 1, 1)))
        dim_in = dim_res1
        dim_out = dim_inner = None
        for stage, (reps, width, stride) in enumerate(block_basis):
            dim_out = round_width(width, w_mul)
            dim_inner = int(cfg.X3D.BOTTLENECK_FACTOR * dim_out)
            n_rep = int(math.ceil(d_mul * reps)) if d_mul else reps
            self.add_module(f"s{stage + 2}", X3DStageModule(f"s{stage + 2}", dim_in, dim_out, dim_inner, 3, stride,
                                                            n_rep, cfg.RESNET.STRIDE_1X1, ctx))
            dim_in = dim_out
        self.head = X3DHeadModule(dim_out, dim_inner, cfg.X3D.DIM_C5, cfg.MODEL.NUM_CLASSES, cfg.MODEL.DROPOUT_RATE,
                                  cfg.MODEL.HEAD_ACT, cfg.X3D.BN_LIN5)
        init_resnet_weights(self, cfg.MODEL.FC_INIT_STD, cfg.RESNET.ZERO_INIT_FINAL_BN, False)
        for m in self.modules():  # c2_msra_fill zeroes conv biases (the SE FCs)
            if isinstance(m, nn.Conv3d) and m.bias is not None:
                nn.init.constant_(m.bias, 0)
        self._init_graph_state()
        b200 = getattr(cfg, "B200", None)
        if b200 is not None and "CUDA_GRAPH" in b200:
            self.cuda_graphs = bool(b200["CUDA_GRAPH"])
        self._drop_seed = int(getattr(cfg, "RNG_SEED", 0))
        self._drop_counter = None
        object.__setattr__(self, "_units", None)

    def _engine_units(self):
        if self._units is None:
            stem, head, ctx = self.s1.pathway0_stem, self.head, self.ctx
            u = {"xy": ConvBN("s1.conv_xy", stem.conv_xy, None, ctx),
                 "c5": ConvBN("head.conv_5", head.conv_5, head.conv_5_bn, ctx)}
            object.__setattr__(self, "_units", u)
        return self._units

    # ------------------------------------------------------------------ forward program
    def _engine_forward(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
        ctx.device = inputs[0].device
        ctx.training = self.training
        ctx.begin_phase("fwd")
        if inputs[0].device.type != "cuda":
            raise L.NativeLibraryError("slowfast_b200 runs on CUDA devices only (no CPU fallback)")
        u = self._engine_units()
        (x,) = inputs
        n, _, t, h, w = x.shape
        stem = self.s1.pathway0_stem
        # ---- stem
        xin = Act(ctx.storage(("in", 0), n, t, h, w, u["xy"].cin_pad))
        ops.input_pack(x.contiguous().float(), xin.planes)
        y0 = u["xy"].fprop(xin.planes)
        c1 = stem.conv.out_channels
        assert y0.shape[-1] == c1 and c1 % 8 == 0, "stem width must be a multiple of 8"
        g = ops.DwGeom(n, *y0.shape[1:4], tuple(stem.conv.kernel_size), tuple(stem.conv.stride),
                       tuple(stem.conv.padding))
        ot, oh, ow = g.out
        y1 = ctx.buf(("s1", "y1"), (n, ot, oh, ow, c1))
        m_tiles, _ = ops.dwconv_tiles(g, c1, True)
        stats = ctx.buf(("s1", "stats"), (2, c1, m_tiles))
        ops.dwconv_fwd(g, c1, c1, stem.conv.weight, ops.f32view(y1), stats, x_f32=ops.f32view(y0))
        bb = {k: ctx.buf(("s1", k), (c1,), zero=True) for k in ("scale", "shift", "mean", "invstd")}
        bn = stem.bn
        ops.bn_finalize(stats, m_tiles, c1, n * ot * oh * ow, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                        bn.momentum if bn.momentum is not None else 0.1, bn.eps, ctx.training, bb["scale"],
                        bb["shift"], bb["mean"], bb["invstd"])
        cur = Act(ctx.storage(("s1", "out"), n, ot, oh, ow, c1))
        ops.bnact_fwd(ops.f32view(y1), bb["scale"], bb["shift"], None, ops.ACT_RELU, ot * oh * ow, cur.planes)
        self._stem_saved = (g, y0, y1, bb, cur)
        # ---- stages
        for i in range(2, 6):
            for bi, blk in enumerate(getattr(self, f"s{i}").blocks()):
                tt, hh, ww = blk.out_dims(*cur.dims[1:])
                out = Act(ctx.storage((f"s{i}", bi), n, tt, hh, ww, blk._dim_out))
                blk.run_forward(cur, out)
                cur = out
        if ctx.training:
            bump_num_batches_tracked(self._all_bns())
        out = self._x3d_head_forward(cur)
        ctx.end_phase()
        return out

    def _x3d_head_forward(self, feat: Act) -> torch.Tensor:
        ctx, head, u = self.ctx, self.head, self._engine_units()
        n, t, h, w = feat.dims
        ps = head_pool_size(self.cfg)
        assert (t, h, w) == ps or ps is None, \
            f"X3DHead on the engine pools the whole {ps} extent to 1x1x1; got features {t, h, w}"
        y5 = u["c5"].fprop(feat.planes)
        x5 = Act(ctx.storage(("head", "x5"), *y5.shape))
        ops.bn_apply(ops.f32view(y5), u["c5"].scale, u["c5"].shift, x5.planes, relu=True)
        ci, co = head.lin_5.in_channels, head.lin_5.out_channels
        pooled = ctx.buf(("head", "pooled"), (n, x5.c))
        ops.global_avgpool_fwd(x5.planes, pooled, 0)
        assert x5.c == ci
        l5 = ctx.buf(("head", "l5"), (n, co))
        ops.small_linear_fwd(pooled, head.lin_5.weight.view(co, ci), None, l5)
        ops.relu_fwd(l5)
        p = head.dropout_rate
        self._drop_mask = None
        if ctx.training and p > 0.0:
            self._drop_mask = ctx.buf(("head", "mask"), (n, co), torch.uint8)
            if self._drop_counter is None or self._drop_counter.device != ctx.device:
                self._drop_counter = torch.zeros(1, dtype=torch.int64, device=ctx.device)
            ops.dropout_fwd(l5, self._drop_mask, p, self._drop_seed, self._drop_counter)
        logits = torch.empty((n, head.projection.out_features), dtype=torch.float32, device=ctx.device)
        ops.small_linear_fwd(l5, head.projection.weight, head.projection.bias, logits)
        if not ctx.training and head.act_func == "softmax":
            ops.row_softmax(logits)
        self._head_saved = (feat, x5, pooled, l5)
        return logits

    # ------------------------------------------------------------------ backward program
    def _engine_backward(self, dlogits: torch.Tensor):
        ctx = self.ctx
        params = [p for p in self.parameters()]
        ctx.begin_backward(params)
        ctx.begin_phase("bwd")
        u, head = self._engine_units(), self.head
        feat, x5, pooled, l5 = self._head_saved
        n, co = l5.shape
        ci = pooled.shape[1]
        proj = head.projection
        dl5 = ctx.buf(("head", "dl5"), (n, co))
        ops.small_linear_bwd(dlogits, l5, proj.weight, ctx.grad_of(proj.weight), ctx.grad_of(proj.bias), dl5)
        if self._drop_mask is not None:
            ops.dropout_bwd(dl5, self._drop_mask, head.dropout_rate)
        ops.relu_bwd(dl5, l5)  # (dropped entries are already zero in dl5, kept ones are positive iff ReLU passed)
        dpooled = ctx.buf(("head", "dpooled"), (n, ci))
        ops.small_linear_bwd(dl5, pooled, head.lin_5.weight.view(co, ci), ctx.grad_of(head.lin_5.weight), None, dpooled)
        _, t, h, w = x5.dims
        ops.global_avgpool_bwd(dpooled, 0, n, t * h * w, ci, x5.grad_view())
        x5.s.grad_written = True
        u["c5"].bwd(x5.grad_view(), x5.planes, feat)
        for i in range(5, 1, -1):
            for blk in reversed(getattr(self, f"s{i}").blocks()):
                blk.run_backward()
        # ---- stem
        stem = self.s1.pathway0_stem
        g, y0, y1, bb, out = self._stem_saved
        c1 = y1.shape[-1]
        dy1 = bn_gate_act_backward(ctx, ops.f32view(y1), bb, None, None, ops.ACT_RELU, g.n, c1, out.grad_view(),
                                   stem.bn, None)
        dy0 = ctx.scratch_planes("dy", *y0.shape)
        ops.dwconv_bwd(g, c1, c1, stem.conv.weight, dy1, ctx.grad_of(stem.conv.weight), None, x_f32=ops.f32view(y0),
                       dx_planes=dy0)
        u["xy"].wgrad(dy0)
        ctx.end_phase()
        return [ctx.grad_of(p) for p in params]


def head_pool_size(cfg):
    """pool_size handed to X3DHead (video_model_builder.py:783-789)."""
    spat = int(math.ceil(cfg.DATA.TRAIN_CROP_SIZE / 32.0))
    return (cfg.DATA.NUM_FRAMES, spat, spat)
