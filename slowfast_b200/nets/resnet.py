"""SlowFast / ResNet (C2D, I3D, Slow) video backbones on the engine.

Mirrors the reference's module tree and parameter names (slowfast/models/video_model_builder.py:173 SlowFast,
:445 ResNet; resnet_helper.py:259 BottleneckTransform, :395 ResBlock, :524 ResStage; stem_helper.py:20,127;
head_helper.py:198) so that checkpoints, the optimizer's parameter grouping and ``build_model`` work unchanged,
but executes with the library's kernels:

  stem    : conv (implicit GEMM, C_in padded 3->8) -> BN stats in the epilogue -> fused BN+ReLU+MaxPool
  block   : three conv+BN units; BN-apply/ReLU/residual-add fused into one pass that emits the split-bf16 operand
            planes of the next conv; the block tail is relu(x + c_bn) or relu(branch1_bn + c_bn) in ONE kernel
  lateral : FuseFastToSlow's conv+BN+ReLU writes straight into the channel slice of the slow pathway's next input
            (torch.cat never happens)
  head    : global average pools -> dropout -> Linear
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from .. import ops
from ..config import nsplit_of
from ..engine import Act, ConvBN, Ctx, ModelFunction, Namespace, StemConvBN, bump_num_batches_tracked

# depth -> blocks per stage (video_model_builder.py:38)
STAGE_DEPTH = {18: (2, 2, 2, 2), 50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}

# temporal kernel of [conv1, res2, res3, res4, res5] per pathway (video_model_builder.py:41-98); "a_b" = first
# block(s) use a, the pattern then repeats over the stage (ResStage :631-635)
TEMPORAL_KERNELS = {
    "2d": [[[1]], [[1]], [[1]], [[1]], [[1]]],
    "c2d": [[[1]], [[1]], [[1]], [[1]], [[1]]],
    "slow_c2d": [[[1]], [[1]], [[1]], [[1]], [[1]]],
    "i3d": [[[5]], [[3]], [[3, 1]], [[3, 1]], [[1, 3]]],
    "slow_i3d": [[[5]], [[3]], [[3, 1]], [[3, 1]], [[1, 3]]],
    "slow": [[[1]], [[1]], [[1]], [[3]], [[3]]],
    "slowfast": [[[1], [5]], [[1], [3]], [[1], [3]], [[3], [3]], [[3], [3]]],
}
# temporal max-pool after res2 per pathway (video_model_builder.py:100-109)
POOL1 = {"2d": [[1, 1, 1]], "c2d": [[2, 1, 1]], "slow_c2d": [[1, 1, 1]], "i3d": [[2, 1, 1]], "slow_i3d": [[1, 1, 1]],
         "slow": [[1, 1, 1]], "slowfast": [[1, 1, 1], [1, 1, 1]]}


def _conv(cin, cout, k, stride, pad):
    return nn.Conv3d(cin, cout, kernel_size=list(k), stride=list(stride), padding=list(pad), bias=False)


class StemModule(Namespace):
    """ResNetBasicStem parameter container: conv, bn (+ inert relu / pool_layer)."""

    def __init__(self, cin, cout, k, stride, pad, eps, mmt):
        super().__init__()
        self.conv = _conv(cin, cout, k, stride, pad)
        self.bn = nn.BatchNorm3d(cout, eps=eps, momentum=mmt)
        self.relu = nn.ReLU(True)
        self.pool_layer = nn.MaxPool3d(kernel_size=[1, 3, 3], stride=[1, 2, 2], padding=[0, 1, 1])


class FuseModule(Namespace):
    """FuseFastToSlow parameter container: conv_f2s, bn."""

    def __init__(self, dim_in, ratio, kernel, alpha, eps=1e-5, mmt=0.1):
        super().__init__()
        self.conv_f2s = _conv(dim_in, dim_in * ratio, (kernel, 1, 1), (alpha, 1, 1), (kernel // 2, 0, 0))
        self.bn = nn.BatchNorm3d(dim_in * ratio, eps=eps, momentum=mmt)
        self.relu = nn.ReLU(True)


class BottleneckModule(Namespace):
    """BottleneckTransform parameter container: a, a_bn, b, b_bn, c, c_bn."""

    def __init__(self, dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, eps, mmt):
        super().__init__()
        s1, s3 = (stride, 1) if stride_1x1 else (1, stride)
        self.a = _conv(dim_in, dim_inner, (temp_k, 1, 1), (1, s1, s1), (temp_k // 2, 0, 0))
        self.a_bn = nn.BatchNorm3d(dim_inner, eps=eps, momentum=mmt)
        self.a_relu = nn.ReLU(True)
        self.b = _conv(dim_inner, dim_inner, (1, 3, 3), (1, s3, s3), (0, 1, 1))
        self.b_bn = nn.BatchNorm3d(dim_inner, eps=eps, momentum=mmt)
        self.b_relu = nn.ReLU(True)
        self.c = _conv(dim_inner, dim_out, (1, 1, 1), (1, 1, 1), (0, 0, 0))
        self.c.final_conv = True
        self.c_bn = nn.BatchNorm3d(dim_out, eps=eps, momentum=mmt)
        self.c_bn.transform_final_bn = True


class ResBlockModule(Namespace):
    """ResBlock parameter container (+ engine program of one bottleneck block)."""

    def __init__(self, name, dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, ctx: Ctx, eps=1e-5, mmt=0.1):
        super().__init__()
        if dim_in != dim_out or stride != 1:
            self.branch1 = _conv(dim_in, dim_out, (1, 1, 1), (1, stride, stride), (0, 0, 0))
            self.branch1_bn = nn.BatchNorm3d(dim_out, eps=eps, momentum=mmt)
        self.branch2 = BottleneckModule(dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, eps, mmt)
        self.relu = nn.ReLU(True)
        self._n = name
        self._ctx = ctx
        self._dim_inner, self._dim_out = dim_inner, dim_out
        object.__setattr__(self, "_units", None)

    def units(self):
        if self._units is None:
            b2, n, ctx = self.branch2, self._n, self._ctx
            u = {"a": ConvBN(n + ".a", b2.a, b2.a_bn, ctx), "b": ConvBN(n + ".b", b2.b, b2.b_bn, ctx),
                 "c": ConvBN(n + ".c", b2.c, b2.c_bn, ctx)}
            if hasattr(self, "branch1"):
                u["s"] = ConvBN(n + ".branch1", self.branch1, self.branch1_bn, ctx)
            object.__setattr__(self, "_units", u)
        return self._units

    def out_dims(self, t, h, w):
        u = self.units()
        return u["b"].out_dims(*u["a"].out_dims(t, h, w))

    def bns(self):
        return [u.bn for u in self.units().values()]

    def run_forward(self, x: Act, out: Act) -> None:
        ctx, u, nm = self._ctx, self.units(), self._n
        n, t, h, w = x.dims
        ya = u["a"].fprop(x.planes)
        xa = Act(ctx.storage((nm, "xa"), *ya.shape))
        ops.bn_apply(ops.f32view(ya), u["a"].scale, u["a"].shift, xa.planes, relu=True)
        yb = u["b"].fprop(xa.planes)
        xb = Act(ctx.storage((nm, "xb"), *yb.shape))
        ops.bn_apply(ops.f32view(yb), u["b"].scale, u["b"].shift, xb.planes, relu=True)
        yc = u["c"].fprop(xb.planes)
        if "s" in u:
            ys = u["s"].fprop(x.planes)
            ops.bn_apply(ops.f32view(yc), u["c"].scale, u["c"].shift, out.planes, relu=True, y2=ops.f32view(ys),
                         scale2=u["s"].scale, shift2=u["s"].shift)
        else:
            ops.bn_apply(ops.f32view(yc), u["c"].scale, u["c"].shift, out.planes, relu=True, res=x.planes)
        object.__setattr__(self, "_saved", (x, xa, xb, out))

    def run_backward(self) -> None:
        """Consumes out.grad, produces (accumulates into) x.grad and all parameter gradients of the block."""
        u = self.units()
        x, xa, xb, out = self._saved
        dout = out.grad_view()
        if "s" in u:
            u["s"].bwd(dout, out.planes, x)
            u["c"].bwd(dout, out.planes, xb)
        else:
            # identity shortcut: dz = dout * relu' flows into x.grad as well (emitted by the same BN-backward pass)
            acc = x.s.grad_written
            u["c"].bwd(dout, out.planes, xb, dres=x.grad_view(), dres_accumulate=acc)
            x.s.grad_written = True
        u["b"].bwd(xb.grad_view(), xb.planes, xa)
        u["a"].bwd(xa.grad_view(), xa.planes, x)


class StageModule(Namespace):
    """ResStage container: pathway{p}_res{i} blocks."""

    def __init__(self, name, dim_in, dim_out, dim_inner, temp_kernel_sizes, stride, num_blocks, num_block_temp_kernel,
                 stride_1x1, ctx: Ctx):
        super().__init__()
        self.num_pathways = len(num_blocks)
        self.num_blocks = list(num_blocks)
        for p in range(self.num_pathways):
            tks = (temp_kernel_sizes[p] * num_blocks[p])[:num_block_temp_kernel[p]] + \
                [1] * (num_blocks[p] - num_block_temp_kernel[p])
            for i in range(num_blocks[p]):
                blk = ResBlockModule(f"{name}.pathway{p}_res{i}", dim_in[p] if i == 0 else dim_out[p], dim_out[p],
                                     tks[i], stride[p] if i == 0 else 1, dim_inner[p], stride_1x1, ctx)
                self.add_module(f"pathway{p}_res{i}", blk)

    def blocks(self, p) -> List[ResBlockModule]:
        return [getattr(self, f"pathway{p}_res{i}") for i in range(self.num_blocks[p])]


class BasicHeadModule(Namespace):
    """ResNetBasicHead container: projection (+ inert pools / dropout / act)."""

    def __init__(self, dim_in, num_classes, dropout_rate, act_func, pool_size=None):
        super().__init__()
        # AvgPool3d(pool_size, stride=1) per pathway (None = adaptive 1x1x1, video_model_builder.py:398-416)
        self.pool_size = [None] * len(dim_in) if pool_size is None else [None if p is None else tuple(p) for p in pool_size]
        for p in range(len(dim_in)):
            self.add_module(f"pathway{p}_avgpool", nn.Identity())
        if dropout_rate > 0.0:
            self.dropout = nn.Dropout(dropout_rate)
        self.projection = nn.Linear(sum(dim_in), num_classes, bias=True)
        if act_func not in ("softmax", "none"):
            raise NotImplementedError(f"head activation {act_func!r} is not on the engine path")
        self.act_func = act_func
        self.dropout_rate = dropout_rate
        self.dim_in = list(dim_in)


def init_resnet_weights(model: nn.Module, fc_init_std, zero_init_final_bn, zero_init_final_conv) -> None:
    """ResNet-style initialisation, same draws in the same module order as the reference
    (utils/weight_init_helper.py:10-45; c2_msra_fill = kaiming_normal_(fan_out, relu))."""
    for m in model.modules():
        if isinstance(m, nn.Conv3d):
            if getattr(m, "final_conv", False) and zero_init_final_conv:
                m.weight.data.zero_()
            else:
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        elif isinstance(m, (nn.BatchNorm3d, nn.BatchNorm2d, nn.BatchNorm1d)):
            zero = getattr(m, "transform_final_bn", False) and zero_init_final_bn
            if m.weight is not None:
                m.weight.data.fill_(0.0 if zero else 1.0)
            if m.bias is not None:
                m.bias.data.zero_()
        if isinstance(m, nn.Linear):
            m.weight.data.normal_(mean=0.0, std=fc_init_std)
            if m.bias is not None:
                m.bias.data.zero_()


class _VideoResNetBase(nn.Module):
    """Shared engine driver of the ResNet-family models."""

    num_pathways = 1
    # CUDA-graph execution of the forward / backward programs (set False to run every launch eagerly)
    cuda_graphs = True
    graph_warmup = 2
    # W-shift stem kernels (csrc/conv_stem.cu); False = generic im2col path (kept for A/B checks)
    wshift_stem = True

    def _init_graph_state(self):
        object.__setattr__(self, "_graphs", {})
        object.__setattr__(self, "_graph_seen", {})

    def _check_cfg(self, cfg):
        assert cfg.BN.NORM_TYPE == "batchnorm", "only BN.NORM_TYPE=batchnorm is on the engine path (SURVEY §2 #9)"
        assert cfg.RESNET.TRANS_FUNC == "bottleneck_transform"
        assert cfg.RESNET.NUM_GROUPS == 1
        assert not cfg.DETECTION.ENABLE, "RoI head is out of scope"
        assert all(len(l) == 0 for st in cfg.NONLOCAL.LOCATION for l in st), "Nonlocal blocks are out of scope"
        assert all(d == 1 for st in cfg.RESNET.SPATIAL_DILATIONS for d in st)
        assert float(cfg.MODEL.DROPCONNECT_RATE) == 0.0 or True  # drop-connect is a no-op in the reference (§3.3)

    # ------------------------------------------------------------------ public nn.Module API
    def forward(self, x, bboxes=None):
        assert bboxes is None, "detection is out of scope of the engine"
        x = list(x[:])
        assert len(x) == self.num_pathways, f"Input tensor does not contain {self.num_pathways} pathway"
        params = [p for p in self.parameters()]
        return ModelFunction.apply(self, len(x), *x, *params)

    def _all_bns(self):
        return [m for m in self.modules() if isinstance(m, nn.BatchNorm3d)]

    def allreduce_gradients(self, group=None) -> None:
        """Data-parallel exchange step (SURVEY.md §8e): ONE NCCL all-reduce (average) over the flat gradient
        bucket the last backward filled; ``param.grad`` is re-pointed at the bucket slices where autograd made a
        private copy.  (Under the reference's build_model the DDP wrapper does its own bucketing instead.)"""
        from ..engine import allreduce_flat_gradients
        assert self.ctx.flat_grad is not None, "call after backward()"
        allreduce_flat_gradients(self.ctx.flat_grad, list(self.parameters()), group,
                                 repoint=not getattr(self, "flat_grad_only", False))

    # ------------------------------------------------------------------ helpers
    def _stem_forward(self, p: int, x: torch.Tensor, stem: StemModule, unit: ConvBN, out: Act) -> None:
        ctx = self.ctx
        n, c, t, h, w = x.shape
        if isinstance(unit, StemConvBN):
            xin = unit.pack_input(x, ("in", p))
        else:
            xin = Act(ctx.storage(("in", p), n, t, h, w, unit.cin_pad))
            ops.input_pack(x.contiguous().float(), xin.planes)
        y = unit.fprop(xin.planes)
        _, ot, oh, ow, co = y.shape
        argmax = ctx.buf(("stem.argmax", p), (n, ot, out.dims[2], out.dims[3], co), torch.uint8)
        ops.bn_relu_maxpool_fwd(y, unit.scale, unit.shift, out.planes, argmax, (3, 3), (2, 2), (1, 1))
        self._stem_saved[p] = (xin, argmax, out)

    def _stem_backward(self, p: int, unit: ConvBN) -> None:
        ctx = self.ctx
        xin, argmax, out = self._stem_saved[p]
        dz = ctx.scratch("stem.dz", unit.y.numel(), torch.float32).view(unit.y.shape)
        ops.bn_relu_maxpool_bwd(out.grad_view(), argmax, dz, out.dims[2], out.dims[3], (3, 3), (2, 2), (1, 1))
        unit.bwd(ops.f32view(dz), None, None)

    def _head_forward(self, feats: List[Act]) -> torch.Tensor:
        ctx, head = self.ctx, self.head
        n = feats[0].dims[0]
        dim = sum(head.dim_in)
        # AvgPool3d(pool_size, stride=1): the train-time extent gives a 1x1x1 map (global mean); a larger map (test crop
        # 256 -> 8x8 against a 7x7 pool) gives several windows, projected and soft-maxed per location and then
        # averaged - the reference's fully-convolutional inference (head_helper.py:305-350)
        windows = []
        for f, ps in zip(feats, head.pool_size):
            t, h, w = f.dims[1:]
            if ps is None or tuple(ps) == (t, h, w):
                windows.append((1, 1, 1))
            else:
                assert all(k <= d for k, d in zip(ps, (t, h, w))), f"head pool {ps} larger than the feature map {(t, h, w)}"
                windows.append((t - ps[0] + 1, h - ps[1] + 1, w - ps[2] + 1))
        assert len(set(windows)) == 1, f"pathway pool outputs differ: {windows}"
        g = windows[0][0] * windows[0][1] * windows[0][2]
        if g > 1:
            if ctx.training:
                raise RuntimeError("ResNetBasicHead: input larger than the train-time pool size in training mode "
                                   "(the reference's view(N, -1) would produce N x (locations*classes) here)")
            pooled = ctx.buf(("head.pooled.win",), (n * g, dim))
            col = 0
            for f, ps in zip(feats, head.pool_size):
                ops.window_avgpool_fwd(f.planes, ps, pooled, col)
                col += f.c
            proj = ctx.buf(("head.proj.win",), (n * g, head.projection.out_features))
            ops.small_linear_fwd(pooled, head.projection.weight, head.projection.bias, proj)
            if head.act_func == "softmax":
                ops.row_softmax(proj)
            logits = torch.empty((n, head.projection.out_features), dtype=torch.float32, device=ctx.device)
            ops.rows_group_mean(proj, logits, g)
            self._head_saved = None
            return logits
        pooled = ctx.buf(("head.pooled",), (n, dim))
        col = 0
        for f in feats:
            ops.global_avgpool_fwd(f.planes, pooled, col)
            col += f.c
        p = head.dropout_rate
        self._drop_mask = None
        if ctx.training and p > 0.0:
            self._drop_mask = ctx.buf(("head.mask",), (n, dim), torch.uint8)
            if getattr(self, "_drop_counter", None) is None or self._drop_counter.device != ctx.device:
                self._drop_counter = torch.zeros(1, dtype=torch.int64, device=ctx.device)
            ops.dropout_fwd(pooled, self._drop_mask, p, self._drop_seed, self._drop_counter)
        logits = torch.empty((n, head.projection.out_features), dtype=torch.float32, device=ctx.device)
        ops.small_linear_fwd(pooled, head.projection.weight, head.projection.bias, logits)
        if not ctx.training and head.act_func == "softmax":
            ops.row_softmax(logits)
        self._head_saved = (feats, pooled)
        return logits

    def _head_backward(self, dlogits: torch.Tensor) -> None:
        ctx, head = self.ctx, self.head
        feats, pooled = self._head_saved
        n, dim = pooled.shape
        dpooled = ctx.buf(("head.dpooled",), (n, dim))
        proj = head.projection
        ops.small_linear_bwd(dlogits, pooled, proj.weight, ctx.grad_of(proj.weight), ctx.grad_of(proj.bias), dpooled)
        if self._drop_mask is not None:
            ops.dropout_bwd(dpooled, self._drop_mask, head.dropout_rate)
        col = 0
        for f in feats:
            nn_, t, h, w = f.dims
            assert not f.s.grad_written
            ops.global_avgpool_bwd(dpooled, col, nn_, t * h * w, f.c, f.grad_view())
            f.s.grad_written = True
            col += f.c


class B200SlowFast(_VideoResNetBase):
    """Two-pathway SlowFast network (video_model_builder.py:173) on the engine."""

    num_pathways = 2

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self._check_cfg(cfg)
        self.ctx = Ctx(nsplit_of(cfg))
        ctx = self.ctx
        d2, d3, d4, d5 = STAGE_DEPTH[cfg.RESNET.DEPTH]
        wpg = cfg.RESNET.WIDTH_PER_GROUP
        dim_inner = cfg.RESNET.NUM_GROUPS * wpg
        beta_inv, ratio = cfg.SLOWFAST.BETA_INV, cfg.SLOWFAST.FUSION_CONV_CHANNEL_RATIO
        fk, alpha = cfg.SLOWFAST.FUSION_KERNEL_SZ, cfg.SLOWFAST.ALPHA
        out_dim_ratio = beta_inv // ratio
        tk = TEMPORAL_KERNELS[cfg.MODEL.ARCH]
        assert POOL1[cfg.MODEL.ARCH] == [[1, 1, 1], [1, 1, 1]]
        cin = cfg.DATA.INPUT_CHANNEL_NUM

        self.s1 = Namespace()
        self.s1.add_module("pathway0_stem", StemModule(cin[0], wpg, tk[0][0] + [7, 7], (1, 2, 2),
                                                       (tk[0][0][0] // 2, 3, 3), 1e-5, 0.1))
        self.s1.add_module("pathway1_stem", StemModule(cin[1], wpg // beta_inv, tk[0][1] + [7, 7], (1, 2, 2),
                                                       (tk[0][1][0] // 2, 3, 3), 1e-5, 0.1))
        self.s1_fuse = FuseModule(wpg // beta_inv, ratio, fk, alpha)
        widths = [wpg * 4, wpg * 8, wpg * 16, wpg * 32]
        depths = [d2, d3, d4, d5]
        prev = wpg
        for i, (wd, dp) in enumerate(zip(widths, depths)):
            st = StageModule(
                f"s{i + 2}", dim_in=[prev + prev // out_dim_ratio, prev // beta_inv], dim_out=[wd, wd // beta_inv],
                dim_inner=[dim_inner * (2 ** i), dim_inner * (2 ** i) // beta_inv], temp_kernel_sizes=tk[i + 1],
                stride=cfg.RESNET.SPATIAL_STRIDES[i], num_blocks=[dp] * 2,
                num_block_temp_kernel=cfg.RESNET.NUM_BLOCK_TEMP_KERNEL[i], stride_1x1=cfg.RESNET.STRIDE_1X1, ctx=ctx)
            self.add_module(f"s{i + 2}", st)
            if i < 3:
                self.add_module(f"s{i + 2}_fuse", FuseModule(wd // beta_inv, ratio, fk, alpha))
            if i == 0:
                for p in range(2):
                    self.add_module(f"pathway{p}_pool", nn.Identity())
            prev = wd
        crop32 = cfg.DATA.TRAIN_CROP_SIZE // 32
        pools = None if cfg.MULTIGRID.SHORT_CYCLE else [[cfg.DATA.NUM_FRAMES // alpha, crop32, crop32],
                                                         [cfg.DATA.NUM_FRAMES, crop32, crop32]]
        self.head = BasicHeadModule([wpg * 32, wpg * 32 // beta_inv], cfg.MODEL.NUM_CLASSES, cfg.MODEL.DROPOUT_RATE,
                                    cfg.MODEL.HEAD_ACT, pool_size=pools)
        init_resnet_weights(self, cfg.MODEL.FC_INIT_STD, cfg.RESNET.ZERO_INIT_FINAL_BN,
                            cfg.RESNET.ZERO_INIT_FINAL_CONV)
        self._ratio = ratio
        self._init_graph_state()
        b200 = getattr(cfg, "B200", None)
        if b200 is not None and "CUDA_GRAPH" in b200:
            self.cuda_graphs = bool(b200["CUDA_GRAPH"])
        self._stem_saved = {}
        self._drop_seed = int(getattr(cfg, "RNG_SEED", 0))
        self._drop_step = 0
        object.__setattr__(self, "_units", None)

    def _engine_units(self):
        if self._units is None:
            ctx = self.ctx
            crop = int(self.cfg.DATA.TRAIN_CROP_SIZE)
            u = {}
            for p, stem in enumerate((self.s1.pathway0_stem, self.s1.pathway1_stem)):
                cls = StemConvBN if (self.wshift_stem and StemConvBN.supported(stem.conv, crop)) else ConvBN
                u[f"stem{p}"] = cls(f"s1.p{p}", stem.conv, stem.bn, ctx)
            for i in range(1, 5):
                f = getattr(self, f"s{i}_fuse")
                u[f"fuse{i}"] = ConvBN(f"s{i}_fuse", f.conv_f2s, f.bn, ctx)
            object.__setattr__(self, "_units", u)
        return self._units

    # ------------------------------------------------------------------ forward program
    def _engine_forward(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
        ctx.device = inputs[0].device
        ctx.training = self.training
        ctx.begin_phase("fwd")
        if inputs[0].device.type != "cuda":
            raise ops.L.NativeLibraryError("slowfast_b200 runs on CUDA devices only (no CPU fallback)")
        u = self._engine_units()
        xs, xf = inputs
        n = xs.shape[0]
        ratio = self._ratio
        # ---- s1: stems.  The slow stem's pooled output is written into the first slice of the concat storage.
        cs, cf = u["stem0"].cout, u["stem1"].cout
        ts, hs, ws = u["stem0"].out_dims(*xs.shape[2:])
        tf, hf, wf = u["stem1"].out_dims(*xf.shape[2:])
        ph, pw = ops.conv_out_size(hs, 3, 2, 1), ops.conv_out_size(ws, 3, 2, 1)
        slow = Act(ctx.storage(("cat", 1), n, ts, ph, pw, cs + ratio * cf))
        fast = Act(ctx.storage(("fast", 1), n, tf, ph, pw, cf))
        self._stem_forward(0, xs, self.s1.pathway0_stem, u["stem0"], slow.slice(0, cs))
        self._stem_forward(1, xf, self.s1.pathway1_stem, u["stem1"], fast)
        self._fuse_forward(1, fast, slow.slice(cs, ratio * cf))
        trace = [(slow, fast, cs)]
        for i in range(2, 6):
            stage: StageModule = getattr(self, f"s{i}")
            outs = []
            for p, x in enumerate((slow, fast)):
                blocks = stage.blocks(p)
                for bi, blk in enumerate(blocks):
                    t, h, w = blk.out_dims(*x.dims[1:])
                    last = bi == len(blocks) - 1
                    cout = blk._dim_out
                    if last and p == 0 and i < 5:
                        cf_next = stage.blocks(1)[-1]._dim_out
                        full = Act(ctx.storage(("cat", i), n, t, h, w, cout + ratio * cf_next))
                        out = full.slice(0, cout)
                    else:
                        full = None
                        out = Act(ctx.storage((f"s{i}", p, bi), n, t, h, w, cout))
                    blk.run_forward(x, out)
                    x = full if full is not None else out
                outs.append(x)
            slow, fast = outs
            if i < 5:
                cs = stage.blocks(0)[-1]._dim_out
                self._fuse_forward(i, fast, slow.slice(cs, slow.c - cs))
            trace.append((slow, fast, cs))
        self._trace = trace
        if ctx.training:
            bump_num_batches_tracked(self._all_bns())
        out = self._head_forward([slow, fast])
        ctx.end_phase()
        return out

    def _fuse_forward(self, i: int, fast: Act, out: Act) -> None:
        unit = self._engine_units()[f"fuse{i}"]
        y = unit.fprop(fast.planes)
        ops.bn_apply(ops.f32view(y), unit.scale, unit.shift, out.planes, relu=True)
        self.__dict__.setdefault("_fuse_saved", {})[i] = (fast, out)

    # ------------------------------------------------------------------ backward program
    def _engine_backward(self, dlogits: torch.Tensor):
        ctx = self.ctx
        params = [p for p in self.parameters()]
        ctx.begin_backward(params)
        ctx.begin_phase("bwd")
        u = self._engine_units()
        self._head_backward(dlogits)
        for i in range(5, 1, -1):
            stage: StageModule = getattr(self, f"s{i}")
            if i < 5:
                fast, out = self._fuse_saved[i]
                u[f"fuse{i}"].bwd(out.grad_view(), out.planes, fast)
            for p in (0, 1):
                for blk in reversed(stage.blocks(p)):
                    blk.run_backward()
        fast, out = self._fuse_saved[1]
        u["fuse1"].bwd(out.grad_view(), out.planes, fast)
        self._stem_backward(0, u["stem0"])
        self._stem_backward(1, u["stem1"])
        ctx.end_phase()
        return [ctx.grad_of(p) for p in params]
