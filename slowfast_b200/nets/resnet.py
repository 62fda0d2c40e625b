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
  head    : global average pools -> dropout -> Linear, or the MLPHead of CONTRASTIVE.NUM_MLP_LAYERS > 1
            (Linear -> ReLU -> ... -> Linear; bias + ReLU fused into each hidden layer's kernel)
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from .. import ops
from ..engine import Act, ConvBN, Ctx, EngineModel, Namespace, StemConvBN, check_head_act
from ..ops import F32, Planes
from ..subbn import norm_factory, num_splits_of

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
    """ResNetBasicStem parameter container: conv, bn (+ inert relu / pool_layer).

    ``norm`` (here and in every container below) builds the BN modules: nn.BatchNorm3d, or the sub-batch BN container
    of ``subbn.norm_factory``."""

    def __init__(self, cin, cout, k, stride, pad, eps, mmt, norm=nn.BatchNorm3d):
        super().__init__()
        self.conv = _conv(cin, cout, k, stride, pad)
        self.bn = norm(num_features=cout, eps=eps, momentum=mmt)
        self.relu = nn.ReLU(True)
        self.pool_layer = nn.MaxPool3d(kernel_size=[1, 3, 3], stride=[1, 2, 2], padding=[0, 1, 1])


class FuseModule(Namespace):
    """FuseFastToSlow parameter container: conv_f2s, bn."""

    def __init__(self, dim_in, ratio, kernel, alpha, eps=1e-5, mmt=0.1, norm=nn.BatchNorm3d):
        super().__init__()
        self.conv_f2s = _conv(dim_in, dim_in * ratio, (kernel, 1, 1), (alpha, 1, 1), (kernel // 2, 0, 0))
        self.bn = norm(num_features=dim_in * ratio, eps=eps, momentum=mmt)
        self.relu = nn.ReLU(True)


class BottleneckModule(Namespace):
    """BottleneckTransform parameter container: a, a_bn, b, b_bn, c, c_bn."""

    def __init__(self, dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, eps, mmt, norm=nn.BatchNorm3d):
        super().__init__()
        s1, s3 = (stride, 1) if stride_1x1 else (1, stride)
        self.a = _conv(dim_in, dim_inner, (temp_k, 1, 1), (1, s1, s1), (temp_k // 2, 0, 0))
        self.a_bn = norm(num_features=dim_inner, eps=eps, momentum=mmt)
        self.a_relu = nn.ReLU(True)
        self.b = _conv(dim_inner, dim_inner, (1, 3, 3), (1, s3, s3), (0, 1, 1))
        self.b_bn = norm(num_features=dim_inner, eps=eps, momentum=mmt)
        self.b_relu = nn.ReLU(True)
        self.c = _conv(dim_inner, dim_out, (1, 1, 1), (1, 1, 1), (0, 0, 0))
        self.c.final_conv = True
        self.c_bn = norm(num_features=dim_out, eps=eps, momentum=mmt)
        self.c_bn.transform_final_bn = True


class ResBlockModule(Namespace):
    """ResBlock parameter container (+ engine program of one bottleneck block)."""

    def __init__(self, name, dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, ctx: Ctx, eps=1e-5, mmt=0.1,
                 norm=nn.BatchNorm3d):
        super().__init__()
        if dim_in != dim_out or stride != 1:
            self.branch1 = _conv(dim_in, dim_out, (1, 1, 1), (1, stride, stride), (0, 0, 0))
            self.branch1_bn = norm(num_features=dim_out, eps=eps, momentum=mmt)
        self.branch2 = BottleneckModule(dim_in, dim_out, temp_k, stride, dim_inner, stride_1x1, eps, mmt, norm)
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
        ops.bn_apply(ops.f32view(ya), u["a"].scale, u["a"].shift, xa.planes, relu=True, **u["a"].split_kw)
        yb = u["b"].fprop(xa.planes)
        xb = Act(ctx.storage((nm, "xb"), *yb.shape))
        ops.bn_apply(ops.f32view(yb), u["b"].scale, u["b"].shift, xb.planes, relu=True, **u["b"].split_kw)
        yc = u["c"].fprop(xb.planes)
        if "s" in u:
            ys = u["s"].fprop(x.planes)
            ops.bn_apply(ops.f32view(yc), u["c"].scale, u["c"].shift, out.planes, relu=True, y2=ops.f32view(ys),
                         scale2=u["s"].scale, shift2=u["s"].shift, **u["c"].split_kw)
        else:
            ops.bn_apply(ops.f32view(yc), u["c"].scale, u["c"].shift, out.planes, relu=True, res=x.planes,
                         **u["c"].split_kw)
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


NONLOCAL_INSTANTIATIONS = ("softmax", "dot_product")


class NonlocalModule(Namespace):
    """Non-local block (nonlocal_helper.py:10-144): conv_theta, conv_phi, conv_g, conv_out (1x1x1, bias=True), bn (+ pool)
    and the engine program of one block, including the temporal group fold of resnet_helper.py:704-722.

      theta = conv_theta(x);  xp = maxpool(x);  phi, g = conv_phi(xp), conv_g(xp)        (biases added while packing)
      softmax     : O = softmax(d^-0.5 theta phi^T) g    S / P: [n*G, Nq, pad8(Nk)], kept for the backward
      dot_product : O = (1/Nk) theta (phi^T g)           reassociated: the Nq x Nk matrix is never formed
      out = x + bn(conv_out(O))                           no ReLU; one BN-apply pass with the residual

    Channels-last, the fold of T into the batch ([n, T, ...] -> [n*G, T/G, ...]) is the same memory, so every kernel
    simply runs on that view."""

    def __init__(self, name, dim, dim_inner, pool_size, instantiation, group, ctx: Ctx, eps=1e-5, mmt=0.1,
                 norm=nn.BatchNorm3d):
        super().__init__()
        if instantiation not in NONLOCAL_INSTANTIATIONS:
            raise NotImplementedError(f"Unknown norm type {instantiation}")
        self.conv_theta = nn.Conv3d(dim, dim_inner, kernel_size=1, stride=1, padding=0)
        self.conv_phi = nn.Conv3d(dim, dim_inner, kernel_size=1, stride=1, padding=0)
        self.conv_g = nn.Conv3d(dim, dim_inner, kernel_size=1, stride=1, padding=0)
        self.conv_out = nn.Conv3d(dim_inner, dim, kernel_size=1, stride=1, padding=0)
        self.conv_out.zero_init = False
        self.bn = norm(num_features=dim, eps=eps, momentum=mmt)
        self.bn.transform_final_bn = True
        self.use_pool = pool_size is not None and any(s > 1 for s in pool_size)
        self.pool_size = tuple(int(s) for s in pool_size) if pool_size is not None else None
        if self.use_pool:
            self.pool = nn.MaxPool3d(kernel_size=list(pool_size), stride=list(pool_size), padding=[0, 0, 0])
        assert dim % 8 == 0 and dim_inner % 8 == 0, "Non-local widths must be multiples of 8"
        self.instantiation = instantiation
        self.dim, self.dim_inner, self.group = dim, dim_inner, int(group)
        self._n = name
        self._ctx = ctx
        object.__setattr__(self, "_units", None)

    def units(self):
        if self._units is None:
            n, ctx = self._n, self._ctx
            u = {"theta": ConvBN(n + ".theta", self.conv_theta, None, ctx),
                 "phi": ConvBN(n + ".phi", self.conv_phi, None, ctx),
                 "g": ConvBN(n + ".g", self.conv_g, None, ctx),
                 "out": ConvBN(n + ".out", self.conv_out, self.bn, ctx)}
            object.__setattr__(self, "_units", u)
        return self._units

    def run_forward(self, x: Act, out: Act) -> None:
        ctx, u, nm = self._ctx, self.units(), self._n
        n, t, h, w = x.dims
        c, d, grp = x.c, self.dim_inner, self.group
        if t % grp:
            raise ValueError(f"{nm}: NONLOCAL.GROUP {grp} does not divide the {t} frames of the block's input")
        ng, tg = n * grp, t // grp
        nq = tg * h * w
        xg = Planes(x.s.hi, x.s.lo, ng, tg, h, w, c, x.c0)  # the group fold: a view of the same memory
        th = Act(ctx.storage((nm, "theta"), n, t, h, w, d))
        ops.bias_split(ops.f32view(u["theta"].fprop(x.planes)), self.conv_theta.bias, th.planes)
        argmax = None
        if self.use_pool:
            k = self.pool_size
            od = (tg // k[0], h // k[1], w // k[2])
            if min(od) < 1:
                raise ValueError(f"{nm}: pool {k} larger than the (grouped) input {(tg, h, w)}")
            src = Act(ctx.storage((nm, "xp"), ng, *od, c))
            argmax = ctx.buf((nm, "argmax"), (ng, *od, c), torch.uint8)
            ops.maxpool3d_fwd(xg, src.planes, argmax, k, k, (0, 0, 0))
        else:
            src = x
        sn, st, sh, sw = src.dims
        nk = sn * st * sh * sw // ng
        ph = Act(ctx.storage((nm, "phi"), sn, st, sh, sw, d))
        gg = Act(ctx.storage((nm, "g"), sn, st, sh, sw, d))
        ops.bias_split(ops.f32view(u["phi"].fprop(src.planes)), self.conv_phi.bias, ph.planes)
        ops.bias_split(ops.f32view(u["g"].fprop(src.planes)), self.conv_g.bias, gg.planes)
        o = ctx.scratch("nl.O", ng * nq * d, F32).view(ng * nq, d)
        nsplit = ctx.nsplit
        if self.instantiation == "softmax":
            nkp = ops.pad8(nk)
            s = ctx.scratch("nl.S", ng * nq * nkp, F32).view(ng * nq, nkp)
            ops.gemm_batched(th.planes, (d, nq * d), False, ph.planes, (d, nk * d), False, nq, nk, d, ng, s, nkp,
                             alpha=d ** -0.5, nsplit=nsplit)
            ps = ctx.storage((nm, "P"), 1, 1, 1, ng * nq, nkp)
            aux = Planes(ps.hi, ps.lo, 1, 1, 1, ng * nq, nkp, 0)
            ops.softmax_relpos_fwd(s, aux, ng, nq, nk)
            # O = P g   (g MN-major: memory [n*G][Nk][d])
            ops.gemm_batched(aux, (nkp, nq * nkp), False, gg.planes, (d, nk * d), True, nq, d, nk, ng, o, d, nsplit=nsplit)
        else:
            # M = phi^T g (d x d per batch entry), O = (1/Nk) theta M
            mf = ctx.scratch("nl.M", ng * d * d, F32).view(ng * d, d)
            ops.gemm_batched(ph.planes, (d, nk * d), True, gg.planes, (d, nk * d), True, d, d, nk, ng, mf, d,
                             nsplit=nsplit)
            ms = ctx.storage((nm, "M"), 1, 1, 1, ng * d, d)
            aux = Planes(ms.hi, ms.lo, 1, 1, 1, ng * d, d, 0)
            ops.bias_split(ops.f32view(mf), None, aux)
            ops.gemm_batched(th.planes, (d, nq * d), False, aux, (d, d * d), True, nq, d, d, ng, o, d, alpha=1.0 / nk,
                             nsplit=nsplit)
        oa = Act(ctx.storage((nm, "O"), n, t, h, w, d))
        ops.bias_split(ops.f32view(o), None, oa.planes)
        yo = u["out"].fprop(oa.planes)
        ops.bn_apply(ops.f32view(yo), u["out"].scale, u["out"].shift, out.planes, relu=False, res=x.planes,
                     **u["out"].split_kw)
        object.__setattr__(self, "_saved", (x, out, xg, th, src, argmax, ph, gg, aux, oa, ng, nq, nk))

    def run_backward(self) -> None:
        """Consumes out.grad, accumulates into x.grad and writes every parameter gradient of the block."""
        ctx, u = self._ctx, self.units()
        x, out, xg, th, src, argmax, ph, gg, aux, oa, ng, nq, nk = self._saved
        d, nsplit = self.dim_inner, ctx.nsplit
        # identity path + conv_out: dres = dout (no ReLU), dO = conv_out dgrad of the BN-input gradient
        acc = x.s.grad_written
        u["out"].bwd(out.grad_view(), None, oa, dres=x.grad_view(), dres_accumulate=acc)
        x.s.grad_written = True
        do = ctx.scratch_planes("nl.dO", 1, 1, 1, ng * nq, d)
        ops.bias_split(ops.f32view(oa.s.grad.view(ng * nq, d)), None, do)
        dth = ctx.scratch("nl.dth", ng * nq * d, F32).view(ng * nq, d)
        dph = ctx.scratch("nl.dphi", ng * nk * d, F32).view(ng * nk, d)
        dg = ctx.scratch("nl.dg", ng * nk * d, F32).view(ng * nk, d)
        if self.instantiation == "softmax":
            nkp = aux.pitch
            dp = ctx.scratch("nl.S", ng * nq * nkp, F32).view(ng * nq, nkp)
            ops.gemm_batched(do, (d, nq * d), False, gg.planes, (d, nk * d), False, nq, nk, d, ng, dp, nkp, nsplit=nsplit)
            ds = ctx.scratch_planes("nl.dS", 1, 1, 1, ng * nq, nkp)
            ops.softmax_relpos_bwd(aux, dp, ds, ng, nq, nk)
            a = d ** -0.5
            # d theta = a dS phi;  d phi = a dS^T theta;  dg = P^T dO
            ops.gemm_batched(ds, (nkp, nq * nkp), False, ph.planes, (d, nk * d), True, nq, d, nk, ng, dth, d, alpha=a,
                             nsplit=nsplit)
            ops.gemm_batched(ds, (nkp, nq * nkp), True, th.planes, (d, nq * d), True, nk, d, nq, ng, dph, d, alpha=a,
                             nsplit=nsplit)
            ops.gemm_batched(aux, (nkp, nq * nkp), True, do, (d, nq * d), True, nk, d, nq, ng, dg, d, nsplit=nsplit)
        else:
            s = 1.0 / nk
            # d theta = s dO M^T;  dM = s theta^T dO;  d phi = g dM^T;  dg = phi dM
            ops.gemm_batched(do, (d, nq * d), False, aux, (d, d * d), False, nq, d, d, ng, dth, d, alpha=s, nsplit=nsplit)
            dmf = ctx.scratch("nl.M", ng * d * d, F32).view(ng * d, d)
            ops.gemm_batched(th.planes, (d, nq * d), True, do, (d, nq * d), True, d, d, nq, ng, dmf, d, alpha=s,
                             nsplit=nsplit)
            dm = ctx.scratch_planes("nl.dM", 1, 1, 1, ng * d, d)
            ops.bias_split(ops.f32view(dmf), None, dm)
            ops.gemm_batched(gg.planes, (d, nk * d), False, dm, (d, d * d), False, nk, d, d, ng, dph, d, nsplit=nsplit)
            ops.gemm_batched(ph.planes, (d, nk * d), False, dm, (d, d * d), True, nk, d, d, ng, dg, d, nsplit=nsplit)
        for conv, gm in ((self.conv_theta, dth), (self.conv_phi, dph), (self.conv_g, dg)):
            part = ctx.scratch("colsum.part", ops.colsum_blocks(gm.shape[0]) * d, F32)
            ops.colsum(gm, gm.shape[0], d, ctx.grad_of(conv.bias), part)
        n, t, h, w = x.dims
        dthp = ctx.scratch_planes("nl.dthp", n, t, h, w, d)
        dphp = ctx.scratch_planes("nl.dphip", *src.dims, d)
        dgp = ctx.scratch_planes("nl.dgp", *src.dims, d)
        ops.bias_split(ops.f32view(dth), None, dthp)
        ops.bias_split(ops.f32view(dph), None, dphp)
        ops.bias_split(ops.f32view(dg), None, dgp)
        u["theta"].wgrad(dthp)
        u["theta"].dgrad(dthp, x)
        u["phi"].wgrad(dphp)
        u["g"].wgrad(dgp)
        u["phi"].dgrad(dphp, src)
        u["g"].dgrad(dgp, src)
        if self.use_pool:
            k = self.pool_size
            ops.maxpool3d_bwd(src.grad_view(), argmax, xg, src.dims[1:], x.grad_view(), k, k, (0, 0, 0), accumulate=True)


class StageModule(Namespace):
    """ResStage container: pathway{p}_res{i} blocks, each optionally followed by pathway{p}_nonlocal{i}
    (resnet_helper.py:666-695)."""

    def __init__(self, name, dim_in, dim_out, dim_inner, temp_kernel_sizes, stride, num_blocks, num_block_temp_kernel,
                 stride_1x1, ctx: Ctx, nonlocal_inds=None, nonlocal_pool=None, nonlocal_group=None,
                 instantiation="softmax", norm=nn.BatchNorm3d):
        super().__init__()
        self.num_pathways = len(num_blocks)
        self.num_blocks = list(num_blocks)
        nonlocal_inds = nonlocal_inds or [[] for _ in num_blocks]
        for p in range(self.num_pathways):
            tks = (temp_kernel_sizes[p] * num_blocks[p])[:num_block_temp_kernel[p]] + \
                [1] * (num_blocks[p] - num_block_temp_kernel[p])
            for i in range(num_blocks[p]):
                blk = ResBlockModule(f"{name}.pathway{p}_res{i}", dim_in[p] if i == 0 else dim_out[p], dim_out[p],
                                     tks[i], stride[p] if i == 0 else 1, dim_inner[p], stride_1x1, ctx, norm=norm)
                self.add_module(f"pathway{p}_res{i}", blk)
                if i in nonlocal_inds[p]:
                    nln = NonlocalModule(f"{name}.pathway{p}_nonlocal{i}", dim_out[p], dim_out[p] // 2, nonlocal_pool[p],
                                         instantiation, nonlocal_group[p], ctx, norm=norm)
                    self.add_module(f"pathway{p}_nonlocal{i}", nln)

    def blocks(self, p) -> List[ResBlockModule]:
        return [getattr(self, f"pathway{p}_res{i}") for i in range(self.num_blocks[p])]

    def nonlocal_after(self, p, i) -> Optional[NonlocalModule]:
        return getattr(self, f"pathway{p}_nonlocal{i}", None)

    def run_block_forward(self, p, i, x: Act, out: Act, key) -> None:
        """pathway{p}_res{i} (+ its Non-local block) from x into out; ``key`` names the intermediate storage."""
        blk, nln = self.blocks(p)[i], self.nonlocal_after(p, i)
        if nln is None:
            blk.run_forward(x, out)
            return
        n, t, h, w = out.dims
        mid = Act(blk._ctx.storage(key + ("nl_in",), n, t, h, w, out.c))
        blk.run_forward(x, mid)
        nln.run_forward(mid, out)

    def run_block_backward(self, p, i) -> None:
        nln = self.nonlocal_after(p, i)
        if nln is not None:
            nln.run_backward()
        self.blocks(p)[i].run_backward()


class MLPHeadModule(Namespace):
    """MLPHead container (head_helper.py:147-196) without BN: projection = Sequential(Linear, ReLU, ..., Linear), every
    Linear with a bias and ``xavier_init`` (c2_xavier_fill in init_resnet_weights)."""

    def __init__(self, dim_in, dim_out, mlp_dim, num_layers):
        super().__init__()
        layers = [nn.Linear(dim_in, mlp_dim, bias=True)]
        for i in range(1, num_layers):
            layers.append(nn.ReLU(inplace=True))
            layers.append(nn.Linear(mlp_dim, dim_out if i == num_layers - 1 else mlp_dim, bias=True))
        for m in layers:
            if isinstance(m, nn.Linear):
                m.xavier_init = True
        self.projection = nn.Sequential(*layers)


def _check_contrastive_head(contrastive) -> int:
    """NUM_MLP_LAYERS of the head; the BN variants of MLPHead and the predictor heads are rejected by name."""
    if contrastive is None:
        return 1
    if list(contrastive.get("PREDICTOR_DEPTHS", [])):
        raise NotImplementedError("CONTRASTIVE.PREDICTOR_DEPTHS (predictor MLP heads) is not on the engine path")
    layers = int(contrastive.get("NUM_MLP_LAYERS", 1))
    if layers > 1:
        for opt in ("BN_MLP", "BN_SYNC_MLP"):
            if contrastive.get(opt, False):
                raise NotImplementedError(f"CONTRASTIVE.{opt} (BatchNorm inside the MLP head) is not on the engine path")
    return layers


class BasicHeadModule(Namespace):
    """ResNetBasicHead container: projection (+ inert pools / dropout / act).  ``contrastive`` (cfg.CONTRASTIVE)
    selects the MLPHead projection when NUM_MLP_LAYERS > 1.  ``detach_final_fc`` (MODEL.DETACH_FINAL_FC, linear
    evaluation, head_helper.py:319-320): the pooled features are detached after the dropout, so the backward runs the
    projection's Linear layers only."""

    def __init__(self, dim_in, num_classes, dropout_rate, act_func, pool_size=None, contrastive=None,
                 detach_final_fc=False):
        super().__init__()
        mlp_layers = _check_contrastive_head(contrastive)
        # AvgPool3d(pool_size, stride=1) per pathway (None = adaptive 1x1x1, video_model_builder.py:398-416)
        self.pool_size = [None] * len(dim_in) if pool_size is None else [None if p is None else tuple(p) for p in pool_size]
        for p in range(len(dim_in)):
            self.add_module(f"pathway{p}_avgpool", nn.Identity())
        if dropout_rate > 0.0:
            self.dropout = nn.Dropout(dropout_rate)
        if mlp_layers == 1:
            self.projection = nn.Linear(sum(dim_in), num_classes, bias=True)
        else:
            self.projection = MLPHeadModule(sum(dim_in), num_classes, int(contrastive.MLP_DIM), mlp_layers)
        check_head_act(act_func)
        self.act_func = act_func
        self.dropout_rate = dropout_rate
        self.detach_final_fc = bool(detach_final_fc)
        self.dim_in = list(dim_in)

    def linears(self) -> List[nn.Linear]:
        """The projection's Linear layers in order; a ReLU sits between consecutive ones."""
        if isinstance(self.projection, nn.Linear):
            return [self.projection]
        return [m for m in self.projection.projection if isinstance(m, nn.Linear)]

    def params_after_detach(self) -> List[nn.Parameter]:
        """The parameters behind the detach: every Linear layer's weight and bias."""
        return [p for lin in self.linears() for p in (lin.weight, lin.bias)]


def init_resnet_weights(model: nn.Module, fc_init_std, zero_init_final_bn, zero_init_final_conv) -> None:
    """ResNet-style initialisation, same draws in the same module order as the reference
    (utils/weight_init_helper.py:10-45; c2_msra_fill = kaiming_normal_(fan_out, relu))."""
    for m in model.modules():
        if isinstance(m, nn.Conv3d):
            if getattr(m, "final_conv", False) and zero_init_final_conv:
                m.weight.data.zero_()
            else:
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                if m.bias is not None:  # (the Non-local convs; c2_msra_fill zeroes the bias)
                    m.bias.data.zero_()
        elif isinstance(m, (nn.BatchNorm3d, nn.BatchNorm2d, nn.BatchNorm1d)):
            zero = getattr(m, "transform_final_bn", False) and zero_init_final_bn
            if m.weight is not None:
                m.weight.data.fill_(0.0 if zero else 1.0)
            if m.bias is not None:
                m.bias.data.zero_()
        if isinstance(m, nn.Linear):
            if getattr(m, "xavier_init", False):
                nn.init.kaiming_uniform_(m.weight, a=1)  # c2_xavier_fill (MLPHead layers)
            else:
                m.weight.data.normal_(mean=0.0, std=fc_init_std)
            if m.bias is not None:
                m.bias.data.zero_()


class _VideoResNetBase(EngineModel):
    """Config checks, stem, head and MLP of the ResNet-family models."""

    num_pathways = 1
    # splits of the training batch (BN.NUM_SPLITS under sub_batchnorm; set by _check_cfg)
    _bn_splits = 1

    def _check_cfg(self, cfg):
        # BN.NORM_TYPE: batchnorm or sub_batchnorm (multigrid's long cycle); norm_factory rejects the others
        self._norm = norm_factory(cfg)
        self._bn_splits = num_splits_of(cfg)
        if cfg.MODEL.FROZEN_BN and cfg.BN.NORM_TYPE == "sub_batchnorm":
            raise NotImplementedError("MODEL.FROZEN_BN with BN.NORM_TYPE sub_batchnorm (frozen sub-batch BN statistics) "
                                      "is not on the engine path")
        assert cfg.RESNET.TRANS_FUNC == "bottleneck_transform"
        assert cfg.RESNET.NUM_GROUPS == 1
        assert not cfg.DETECTION.ENABLE, "RoI head is out of scope"
        assert all(d == 1 for st in cfg.RESNET.SPATIAL_DILATIONS for d in st)

    # ------------------------------------------------------------------ public nn.Module API
    def forward(self, x, bboxes=None):
        assert bboxes is None, "detection is out of scope of the engine"
        x = list(x[:])
        assert len(x) == self.num_pathways, f"Input tensor does not contain {self.num_pathways} pathway"
        if self.training and self._bn_splits > 1 and x[0].shape[0] % self._bn_splits:
            raise ValueError(f"sub_batchnorm: BN.NUM_SPLITS {self._bn_splits} does not divide the batch size "
                             f"{x[0].shape[0]} (every split takes batch / NUM_SPLITS clips)")
        return self._run(x)

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
        ops.bn_relu_maxpool_fwd(y, unit.scale, unit.shift, out.planes, argmax, (3, 3), (2, 2), (1, 1),
                                splits=unit.splits)
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
            proj = self._head_mlp_forward(pooled, ("head.proj.win",))[-1]
            ops.head_act(proj, head.act_func)
            logits = torch.empty((n, proj.shape[1]), dtype=torch.float32, device=ctx.device)
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
            ops.dropout_fwd(pooled, self._drop_mask, p, self._seed, self._head_drop_counter())
        acts = self._head_mlp_forward(pooled, None)
        logits = acts[-1]
        if not ctx.training:
            ops.head_act(logits, head.act_func)
        self._head_saved = (feats, acts[:-1])
        return logits

    def _head_mlp_forward(self, x: torch.Tensor, key) -> List[torch.Tensor]:
        """[x, hidden activations..., output] of the projection; the output is a fresh tensor when ``key`` is None
        (the logits handed to autograd), else a buffer named by ``key``."""
        ctx, lins = self.ctx, self.head.linears()
        acts = [x]
        for i, lin in enumerate(lins):
            last = i == len(lins) - 1
            shape = (x.shape[0], lin.out_features)
            if not last:
                y = ctx.buf(("head.mlp", i, key is not None), shape)
            elif key is None:
                y = torch.empty(shape, dtype=torch.float32, device=ctx.device)
            else:
                y = ctx.buf(key, shape)
            ops.small_linear_fwd(acts[-1], lin.weight, lin.bias, y, relu=not last)
            acts.append(y)
        return acts

    def _head_backward(self, dlogits: torch.Tensor) -> bool:
        """The head's backward into the feature gradients; False under MODEL.DETACH_FINAL_FC, where it stops at the
        projection's first Linear and nothing before the detach has a gradient."""
        ctx, head = self.ctx, self.head
        feats, acts = self._head_saved
        dy = dlogits
        for i in reversed(range(len(acts))):
            lin, x = head.linears()[i], acts[i]
            if i == 0 and head.detach_final_fc:
                dx = None
            else:
                dx = ctx.buf(("head.dpooled",) if i == 0 else ("head.dmlp", i), x.shape)
            ops.small_linear_bwd(dy, x, lin.weight, ctx.grad_of(lin.weight), ctx.grad_of(lin.bias), dx, relu_mask=i > 0)
            dy = dx
        if head.detach_final_fc:
            return False
        dpooled = dy
        if self._drop_mask is not None:
            ops.dropout_bwd(dpooled, self._drop_mask, head.dropout_rate)
        col = 0
        for f in feats:
            nn_, t, h, w = f.dims
            assert not f.s.grad_written
            ops.global_avgpool_bwd(dpooled, col, nn_, t * h * w, f.c, f.grad_view())
            f.s.grad_written = True
            col += f.c
        return True


class B200SlowFast(_VideoResNetBase):
    """Two-pathway SlowFast network (video_model_builder.py:173) on the engine."""

    num_pathways = 2

    def __init__(self, cfg):
        super().__init__(cfg)
        self._check_cfg(cfg)
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

        norm = self._norm
        self.s1 = Namespace()
        self.s1.add_module("pathway0_stem", StemModule(cin[0], wpg, tk[0][0] + [7, 7], (1, 2, 2),
                                                       (tk[0][0][0] // 2, 3, 3), 1e-5, 0.1, norm))
        self.s1.add_module("pathway1_stem", StemModule(cin[1], wpg // beta_inv, tk[0][1] + [7, 7], (1, 2, 2),
                                                       (tk[0][1][0] // 2, 3, 3), 1e-5, 0.1, norm))
        self.s1_fuse = FuseModule(wpg // beta_inv, ratio, fk, alpha, norm=norm)
        widths = [wpg * 4, wpg * 8, wpg * 16, wpg * 32]
        depths = [d2, d3, d4, d5]
        prev = wpg
        for i, (wd, dp) in enumerate(zip(widths, depths)):
            st = StageModule(
                f"s{i + 2}", dim_in=[prev + prev // out_dim_ratio, prev // beta_inv], dim_out=[wd, wd // beta_inv],
                dim_inner=[dim_inner * (2 ** i), dim_inner * (2 ** i) // beta_inv], temp_kernel_sizes=tk[i + 1],
                stride=cfg.RESNET.SPATIAL_STRIDES[i], num_blocks=[dp] * 2,
                num_block_temp_kernel=cfg.RESNET.NUM_BLOCK_TEMP_KERNEL[i], stride_1x1=cfg.RESNET.STRIDE_1X1, ctx=ctx,
                nonlocal_inds=cfg.NONLOCAL.LOCATION[i], nonlocal_pool=cfg.NONLOCAL.POOL[i],
                nonlocal_group=cfg.NONLOCAL.GROUP[i], instantiation=cfg.NONLOCAL.INSTANTIATION, norm=norm)
            self.add_module(f"s{i + 2}", st)
            if i < 3:
                self.add_module(f"s{i + 2}_fuse", FuseModule(wd // beta_inv, ratio, fk, alpha, norm=norm))
            if i == 0:
                for p in range(2):
                    self.add_module(f"pathway{p}_pool", nn.Identity())
            prev = wd
        crop32 = cfg.DATA.TRAIN_CROP_SIZE // 32
        pools = None if cfg.MULTIGRID.SHORT_CYCLE or cfg.MODEL.MODEL_NAME == "ContrastiveModel" else [[cfg.DATA.NUM_FRAMES // alpha, crop32, crop32],
                                                         [cfg.DATA.NUM_FRAMES, crop32, crop32]]
        self.head = BasicHeadModule([wpg * 32, wpg * 32 // beta_inv], cfg.MODEL.NUM_CLASSES, cfg.MODEL.DROPOUT_RATE,
                                    cfg.MODEL.HEAD_ACT, pool_size=pools, contrastive=cfg.get("CONTRASTIVE"),
                                    detach_final_fc=cfg.MODEL.DETACH_FINAL_FC)
        init_resnet_weights(self, cfg.MODEL.FC_INIT_STD, cfg.RESNET.ZERO_INIT_FINAL_BN,
                            cfg.RESNET.ZERO_INIT_FINAL_CONV)
        self._ratio = ratio
        self._stem_saved = {}
        object.__setattr__(self, "_units", None)

    def _engine_units(self):
        if self._units is None:
            ctx = self.ctx
            crop = int(self.cfg.DATA.TRAIN_CROP_SIZE)
            u = {}
            for p, stem in enumerate((self.s1.pathway0_stem, self.s1.pathway1_stem)):
                cls = StemConvBN if StemConvBN.supported(stem.conv, crop) else ConvBN
                u[f"stem{p}"] = cls(f"s1.p{p}", stem.conv, stem.bn, ctx)
            for i in range(1, 5):
                f = getattr(self, f"s{i}_fuse")
                u[f"fuse{i}"] = ConvBN(f"s{i}_fuse", f.conv_f2s, f.bn, ctx)
            object.__setattr__(self, "_units", u)
        return self._units

    # ------------------------------------------------------------------ forward program
    def _forward_program(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
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
                    stage.run_block_forward(p, bi, x, out, (f"s{i}", p, bi))
                    x = full if full is not None else out
                outs.append(x)
            slow, fast = outs
            if i < 5:
                cs = stage.blocks(0)[-1]._dim_out
                self._fuse_forward(i, fast, slow.slice(cs, slow.c - cs))
            trace.append((slow, fast, cs))
        self._trace = trace
        return self._head_forward([slow, fast])

    def _fuse_forward(self, i: int, fast: Act, out: Act) -> None:
        unit = self._engine_units()[f"fuse{i}"]
        y = unit.fprop(fast.planes)
        ops.bn_apply(ops.f32view(y), unit.scale, unit.shift, out.planes, relu=True, **unit.split_kw)
        self.__dict__.setdefault("_fuse_saved", {})[i] = (fast, out)

    # ------------------------------------------------------------------ backward program
    def _backward_program(self, dlogits: torch.Tensor) -> None:
        u = self._engine_units()
        if not self._head_backward(dlogits):
            return
        for i in range(5, 1, -1):
            stage: StageModule = getattr(self, f"s{i}")
            if i < 5:
                fast, out = self._fuse_saved[i]
                u[f"fuse{i}"].bwd(out.grad_view(), out.planes, fast)
            for p in (0, 1):
                for bi in reversed(range(stage.num_blocks[p])):
                    stage.run_block_backward(p, bi)
        fast, out = self._fuse_saved[1]
        u["fuse1"].bwd(out.grad_view(), out.planes, fast)
        self._stem_backward(0, u["stem0"])
        self._stem_backward(1, u["stem1"])
