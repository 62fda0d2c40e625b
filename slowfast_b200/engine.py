"""Execution core shared by the engine's model builders.

A model is a static forward program over persistent device buffers plus its mirrored backward program; autograd
sees it as ONE custom ``torch.autograd.Function`` (``ModelFunction``) whose inputs are the clip tensors and every
parameter, so ``loss.backward()`` in the reference's unmodified ``train_epoch`` (tools/train_net.py:152) drives the
engine's own backward kernels and parameter gradients land in ``param.grad`` (and in DDP's reducer hooks) as usual.

Building blocks:
  * ``Storage``/``Act``  - channels-last split-bf16 activation storage (+ lazily allocated fp32 gradient) and a
                           channel-slice view of it ("concat in place").
  * ``ConvBN``           - conv (wgmma implicit GEMM) + train/eval BatchNorm statistics; backward = BN backward,
                           wgrad, dgrad (strided dgrad via ``conv_plan``).
  * ``Ctx``              - per-model buffer cache, scratch, flat gradient buffer, launch bookkeeping.
  * ``EngineModel``      - the base class of every engine network: what ``ModelFunction`` drives.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import ops
from .config import nsplit_of
from .conv_plan import dgrad_out_view, dgrad_plan
from .ops import F32, F32View, Planes
from .subbn import is_sub_bn


class Storage:
    """Channels-last activation storage [n, t, h, w, pitch] as split-bf16 planes, plus its fp32 gradient."""

    def __init__(self, n, t, h, w, pitch, nsplit, device, planes: bool = True):
        self.shape = (n, t, h, w, pitch)
        # planes=False: gradient-only storage (the activation itself is recomputed on the fly by its consumer)
        self.hi = torch.empty(self.shape if planes else (0, 0, 0, 0, pitch), dtype=torch.bfloat16, device=device)
        self.lo = torch.empty(self.shape, dtype=torch.bfloat16, device=device) if (nsplit == 3 and planes) else None
        self.grad: Optional[torch.Tensor] = None
        self.grad_written = False

    def ensure_grad(self) -> torch.Tensor:
        if self.grad is None:
            self.grad = torch.empty(self.shape, dtype=F32, device=self.hi.device)
        return self.grad


class Act:
    """Channel-slice view [c0, c0+c) of a Storage."""

    def __init__(self, storage: Storage, c0: int = 0, c: Optional[int] = None):
        self.s = storage
        self.c0 = c0
        self.c = storage.shape[4] - c0 if c is None else c

    @property
    def planes(self) -> Planes:
        n, t, h, w, _ = self.s.shape
        return Planes(self.s.hi, self.s.lo, n, t, h, w, self.c, self.c0)

    @property
    def dims(self):
        return self.s.shape[:4]

    def grad_view(self) -> F32View:
        g = self.s.ensure_grad()
        n, t, h, w, pitch = self.s.shape
        return F32View(g, n * t * h * w, self.c, pitch, self.c0)

    def slice(self, c0: int, c: int) -> "Act":
        return Act(self.s, self.c0 + c0, c)


MAX_ARENAS = 6


class Arena:
    """Buffers of one input signature (mode, grad mode, input shapes): see ``Ctx.use_arena``."""

    def __init__(self, key):
        self.key = key
        self.bufs: Dict[Tuple, torch.Tensor] = {}
        self.storages: Dict[Tuple, "Storage"] = {}
        self.scratch: Dict[str, torch.Tensor] = {}
        self.generation = 0      # bumped by every forward that writes this arena's activations
        self.last_use = 0
        self.on_evict: List = []


class Ctx:
    """Per-model execution context: precision mode, cached buffers, scratch and the flat gradient buffer."""

    def __init__(self, nsplit: int):
        assert nsplit in (1, 3)
        self.nsplit = nsplit
        self.device: Optional[torch.device] = None
        # One arena (named buffers, activation storages, scratch) per input signature: CUDA graphs bake raw device
        # pointers, so a forward at another shape (partial last batch of the val / test loaders, another crop) must
        # never reallocate the buffers a captured program replays into.
        self._arenas: Dict[Tuple, "Arena"] = {}
        self.arena: Arena = Arena(None)
        self._arenas[None] = self.arena
        self._bufs: Dict[Tuple, torch.Tensor] = self.arena.bufs
        self._storages: Dict[Tuple, Storage] = self.arena.storages
        self._scratch: Dict[str, torch.Tensor] = self.arena.scratch
        self.flat_grad: Optional[torch.Tensor] = None
        self.grad_slots: Dict[int, torch.Tensor] = {}  # id(param) -> view into flat_grad
        self.training = True

    # arenas -------------------------------------------------------------------------------------------
    def use_arena(self, key) -> "Arena":
        """Switch every cache (buf / storage / scratch) to the arena of this input signature, creating it on first
        use.  At most ``MAX_ARENAS`` signatures stay resident; the least recently used one is dropped together with the
        programs captured on it (``on_evict`` callbacks)."""
        a = self._arenas.get(key)
        if a is None:
            a = Arena(key)
            self._arenas[key] = a
            live = [k for k in self._arenas if k is not None and k != key]
            if len(live) >= MAX_ARENAS:
                victim = min(live, key=lambda k: self._arenas[k].last_use)
                old = self._arenas.pop(victim)
                for cb in old.on_evict:
                    cb()
        self._arena_clock = getattr(self, "_arena_clock", 0) + 1
        a.last_use = self._arena_clock
        self.arena = a
        self._bufs, self._storages, self._scratch = a.bufs, a.storages, a.scratch
        return a

    # persistent named buffers -------------------------------------------------------------------
    def buf(self, key: Tuple, shape: Sequence[int], dtype=F32, zero: bool = False) -> torch.Tensor:
        """Persistent buffer; ``zero``: zero-filled when (re)allocated (pad entries nobody writes stay 0)."""
        t = self._bufs.get(key)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = (torch.zeros if zero else torch.empty)(tuple(shape), dtype=dtype, device=self.device)
            self._bufs[key] = t
        return t

    def storage(self, key: Tuple, n, t, h, w, pitch, planes: bool = True) -> Storage:
        s = self._storages.get(key)
        if s is None or s.shape != (n, t, h, w, pitch):
            s = Storage(n, t, h, w, pitch, self.nsplit, self.device, planes)
            self._storages[key] = s
        return s

    # scratch that is reused by consecutive layers (single stream => safe) ---------------------------
    def scratch(self, tag: str, nelem: int, dtype) -> torch.Tensor:
        t = self._scratch.get(tag)
        if t is None or t.numel() < nelem or t.dtype != dtype:
            t = torch.empty(int(nelem), dtype=dtype, device=self.device)
            self._scratch[tag] = t
        return t[:nelem]

    def scratch_planes(self, tag: str, n, t, h, w, c) -> Planes:
        nelem = n * t * h * w * c
        hi = self.scratch(tag + ".hi", nelem, torch.bfloat16).view(n, t, h, w, c)
        lo = self.scratch(tag + ".lo", nelem, torch.bfloat16).view(n, t, h, w, c) if self.nsplit == 3 else None
        return Planes(hi, lo, n, t, h, w, c, 0)

    def begin_backward(self, params: Sequence[nn.Parameter]) -> None:
        """One flat fp32 gradient buffer per backward pass; every parameter's gradient is a view into it (the
        single all-reduce bucket of the data-parallel step).  Slots start on 256-byte boundaries (``flat_offsets``):
        the wgrad kernels issue 16-byte vector reductions straight into them."""
        offsets, total = flat_offsets(params)
        self.flat_grad = torch.zeros(total, dtype=F32, device=self.device) if total != sum(p.numel() for p in params) \
            else torch.empty(total, dtype=F32, device=self.device)
        self.grad_slots = {}
        for p, off in zip(params, offsets):
            self.grad_slots[id(p)] = self.flat_grad[off:off + p.numel()].view(p.shape)
        for s in self._storages.values():
            s.grad_written = False

    def grad_of(self, p: nn.Parameter) -> torch.Tensor:
        return self.grad_slots[id(p)]

    def grads(self, params: Sequence[nn.Parameter]) -> List[Optional[torch.Tensor]]:
        """Every parameter's gradient slot; None for a parameter this backward writes none for (not in the list
        ``begin_backward`` took)."""
        return [self.grad_slots.get(id(p)) for p in params]


FLAT_ALIGN = 64  # fp32 elements: every gradient slot of the flat bucket starts on a 256-byte boundary


def flat_offsets(params: Sequence[nn.Parameter], align: int = FLAT_ALIGN) -> Tuple[List[int], int]:
    """Element offset of every parameter's slot in the flat gradient bucket, and the bucket length."""
    offsets, off = [], 0
    for p in params:
        offsets.append(off)
        off += (p.numel() + align - 1) // align * align
    return offsets, off


def allreduce_flat_gradients(flat: torch.Tensor, params: Sequence[nn.Parameter], group=None,
                             repoint: bool = True) -> None:
    """The data-parallel exchange step (SURVEY.md section 8e): ONE all-reduce (average) over the flat gradient bucket,
    then ``param.grad`` is re-pointed at the bucket slices wherever autograd made a private copy.  Works on any
    ``torch.distributed`` backend (NCCL on the GPUs; gloo in the CPU tests)."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    if dist.get_backend(group) == "nccl":
        dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=group)
    else:  # gloo has no AVG
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.div_(world)
    if not repoint:   # (flat_grad_only models: the optimizer reads the bucket itself)
        return
    offsets, total = flat_offsets(params)
    assert total == flat.numel(), "flat bucket does not match the parameter list"
    for p, off in zip(params, offsets):
        n = p.numel()
        if p.grad is None or p.grad.data_ptr() != flat.data_ptr() + flat.element_size() * off:
            p.grad = flat[off:off + n].view_as(p)


def check_head_act(act_func: str) -> None:
    """MODEL.HEAD_ACT of a classification head: the eval-mode softmax / sigmoid, or none; anything else is rejected."""
    if act_func not in ops.HEAD_ACTS:
        raise NotImplementedError(f"head activation {act_func!r} is not on the engine path (MODEL.HEAD_ACT takes "
                                  f"softmax, sigmoid or none)")


def _t3(v) -> Tuple[int, int, int]:
    return tuple(int(x) for x in v)


class ConvBN:
    """nn.Conv3d followed by nn.BatchNorm3d (or by nothing: ``bn=None``), executed by the library's kernels.

    The torch modules are parameter containers only (their ``forward`` is never called); they keep the reference's
    ``state_dict`` names and ``_NormBase`` identity (optimizer.py:41-56, checkpoint.py, precise-BN).

    A conv bias (the Non-local block's conv_out) never enters the conv output ``y``: train-mode batch statistics cancel
    it, so it only moves the BN's running mean, the eval-mode shift and its own gradient (the column sum of the BN-input
    gradient).  Without a BN the caller adds it (``ops.bias_split``) and computes its gradient.

    ``bn`` may be a sub-batch BN container (subbn.py): gamma / beta are the container's; a training pass takes its
    statistics per split (``bn_split_stats``) into ``split_bn`` and emits [S][C] coefficient tables, which every
    apply / backward kernel indexes by the split of the row's clip (``split_kw``); eval is the plain path on ``bn``.

    The BN runs on batch statistics (and updates its running buffers) iff the model AND its own module are in training
    mode (``bn_mode``): ``misc.frozen_bn_stats`` (MODEL.FROZEN_BN) puts BN modules in eval inside a training model, and
    such a unit takes the running statistics forward and backward while its conv still trains."""

    def __init__(self, name: str, conv: nn.Conv3d, bn: Optional[nn.Module], ctx: Ctx):
        assert conv.groups == 1 and _t3(conv.dilation) == (1, 1, 1), \
            f"{name}: only dense, undilated Conv3d is on this path"
        self.name, self.conv, self.bn, self.ctx = name, conv, bn, ctx
        self.bias = conv.bias
        self.sub = bn is not None and is_sub_bn(bn)
        assert bn is None or self._stats_bn(True).momentum is not None, \
            f"{name}: BatchNorm momentum=None (cumulative moving average) is not on the engine path"
        assert not self.sub or (bn.affine and conv.out_channels % 8 == 0), \
            f"{name}: sub-batch BN needs an affine container and a multiple of 8 channels"
        self.splits, self.rows_per_clip = 1, 0
        self.bn_train = False
        self.k, self.stride, self.pad = _t3(conv.kernel_size), _t3(conv.stride), _t3(conv.padding)
        self.cin, self.cout = conv.in_channels, conv.out_channels
        self.cin_pad = ops.pad8(self.cin)
        # output channels are padded to a multiple of 8 as well (X3D's 54 / 108 wide bottlenecks): the conv output,
        # the BN coefficient vectors and every downstream activation carry exact zeros in the pad channels
        self.cout_pad = ops.pad8(self.cout)
        self.taps = self.k[0] * self.k[1] * self.k[2]
        # forward state
        self.x: Optional[Planes] = None
        self.geom = None
        self.y: Optional[torch.Tensor] = None

    # ---------------------------------------------------------------------------------- forward
    def out_dims(self, t, h, w):
        return tuple(ops.conv_out_size(i, k, s, p) for i, k, s, p in zip((t, h, w), self.k, self.stride, self.pad))

    def _stats_bn(self, training: bool) -> nn.Module:
        """The BatchNorm whose running statistics this pass uses: split_bn (training) / bn (eval) of a sub-batch BN."""
        if not self.sub:
            return self.bn
        return self.bn.split_bn if training else self.bn.bn

    def _set_bn_mode(self) -> None:
        """The BN mode of this forward (and of the backward that follows it): see ``bn_mode``."""
        self.bn_train = self.bn is not None and bn_mode(self.ctx, self.bn)
        if self.sub and self.ctx.training and not (self.bn.training and self.bn.split_bn.training and
                                                   self.bn.bn.training):
            raise NotImplementedError(f"{self.name}: MODEL.FROZEN_BN (a sub-batch BN, or one of its inner BNs, in eval "
                                      f"mode inside a training model) is not on the engine path")

    @property
    def split_kw(self) -> dict:
        """Split geometry of the last forward, for the kernels that apply this unit's coefficients."""
        return {"splits": self.splits, "rows_per_clip": self.rows_per_clip}

    def _bn_forward(self, y: torch.Tensor, stats: Optional[torch.Tensor], m_tiles: int, cp: int, zero: bool) -> None:
        """Finalize the BN of conv output ``y`` [n, t, h, w, cp]: scale / shift / mean / invstd ([splits][cp] tables
        under sub-batch BN training; there the conv ran without epilogue statistics and they are taken here)."""
        ctx, bn, c, s = self.ctx, self.bn, self.cout, self.splits
        rows = y.numel() // y.shape[-1]
        if s > 1:
            m_tiles = ops.bn_split_stats_tiles(rows, self.rows_per_clip, s, c)
            stats = ctx.buf((self.name, "stats.split"), (2, s * c, m_tiles))
            ops.bn_split_stats(ops.f32view(y), s, self.rows_per_clip, stats)
        self.scale = ctx.buf((self.name, "scale"), (s * cp,), zero=zero)
        self.shift = ctx.buf((self.name, "shift"), (s * cp,), zero=zero)
        self.mean = ctx.buf((self.name, "mean"), (s * cp,), zero=zero)
        self.invstd = ctx.buf((self.name, "invstd"), (s * cp,), zero=zero)
        sbn = self._stats_bn(self.bn_train)
        momentum = sbn.momentum if sbn.momentum is not None else 0.1
        ops.bn_finalize(stats, m_tiles, s * c, rows // s, bn.weight, bn.bias, sbn.running_mean, sbn.running_var,
                        momentum, sbn.eps, self.bn_train, self.scale, self.shift, self.mean, self.invstd, affine_c=c)
        if self.bias is not None:
            ops.bn_conv_bias(self.bias, c, momentum, self.bn_train, sbn.running_mean, self.scale, self.shift, self.mean,
                             splits=s)

    def fprop(self, x: Planes) -> torch.Tensor:
        """y = conv(x) (fp32, dense channels-last) + BN statistics -> self.scale/self.shift."""
        ctx = self.ctx
        assert x.c == self.cin_pad, (self.name, x.c, self.cin_pad)
        geom = ops.fprop_geom(x, self.k, self.stride, self.pad)
        ot, oh, ow = geom.out
        f = ctx.buf((self.name, "f.hi"), (self.cout, self.taps * self.cin_pad), torch.bfloat16)
        flo = ctx.buf((self.name, "f.lo"), f.shape, torch.bfloat16) if ctx.nsplit == 3 else None
        fm = ops.FilterMat(f, flo, self.cout, self.taps, self.cin_pad)
        ops.filter_pack(self.conv.weight, fm)
        c, cp = self.cout, self.cout_pad
        y = ctx.buf((self.name, "y"), (x.n, ot, oh, ow, cp))
        strides = (ot * oh * ow * cp, oh * ow * cp, ow * cp, cp)
        m_tiles = ops.conv_stats_tiles(x, fm, geom, y, strides, nsplit=ctx.nsplit)
        self._set_bn_mode()
        self.splits = self.bn.num_splits if (self.sub and self.bn_train) else 1
        self.rows_per_clip = ot * oh * ow
        # (sub-batch BN: the epilogue's 128-row tiles cross clips, so the statistics are a separate pass)
        stats = ctx.buf((self.name, "stats"), (2, c, m_tiles)) if (self.bn_train and self.splits == 1) else None
        # (the epilogue stores whole float4 groups: columns [c, cp) receive the zero accumulators of filter rows
        # the TMA box reads out of bounds)
        ops.conv_igemm(x, fm, geom, y, strides, stats=stats, nsplit=ctx.nsplit)
        self.x, self.geom, self.y = x, geom, y
        if self.bn is None:
            return y
        self._bn_forward(y, stats, m_tiles, cp, zero=True)
        return y

    # ---------------------------------------------------------------------------------- backward
    def bwd(self, dout: F32View, mask: Optional[Planes], x_act: Optional[Act], dres: Optional[F32View] = None,
            dres_accumulate: bool = False, mask_from_y: bool = False) -> None:
        """dout: gradient w.r.t. act(bn(conv(x))) (before the ReLU mask is applied); x_act: where the data
        gradient goes (None = input needs no gradient).  mask_from_y: the ReLU output was never materialised;
        recompute its mask from y and the forward affine."""
        ctx = self.ctx
        n, ot, oh, ow, c = self.y.shape
        dy = ctx.scratch_planes("dy", n, ot, oh, ow, c)
        partials, coef = self._bwd_scratch(n * ot * oh * ow, c)
        bn = self.bn
        ops.bn_bwd(dout, mask, ops.f32view(self.y), self.mean, self.invstd, bn.weight, ctx.grad_of(bn.weight),
                   ctx.grad_of(bn.bias), dy, partials, coef, training=self.bn_train, dres=dres,
                   dres_accumulate=dres_accumulate, c_valid=self.cout,
                   mask_affine=(self.scale, self.shift) if mask_from_y else None, **self.split_kw)
        if self.bias is not None:
            rows = n * ot * oh * ow
            dyf = ctx.scratch("bias.dy", rows * c, F32).view(rows, c)
            ops.planes_to_f32(dy, ops.f32view(dyf))
            part = ctx.scratch("colsum.part", ops.colsum_blocks(rows) * self.cout, F32)
            ops.colsum(dyf, rows, self.cout, ctx.grad_of(self.bias), part, pitch=c)
        self.wgrad(dy)
        if x_act is not None:
            self.dgrad(dy, x_act)

    def _bwd_scratch(self, rows, c):
        nb = ops.bn_bwd_blocks(rows, c, self.splits, self.rows_per_clip)
        return (self.ctx.scratch("bnb.partials", nb * 2 * c, F32).view(nb, 2, c),
                self.ctx.scratch("bnb.coef", 3 * self.splits * c, F32).view(3, self.splits * c))

    def wgrad(self, dy: Planes) -> None:
        ctx = self.ctx
        gw = ctx.grad_of(self.conv.weight)
        if self.taps == 1 and self.cin_pad == self.cin and self.cout_pad == self.cout:
            # the GEMM result layout [cout][cin] IS the parameter layout: accumulate straight into the grad slot
            ops.zero_f32(ops.f32view(gw.view(self.cout, self.cin)))
            ops.conv_wgrad(self.x, dy, self.geom, gw, nsplit=ctx.nsplit)
        else:
            dwm = ctx.scratch("dwm", self.cout_pad * self.taps * self.cin_pad, F32).view(self.cout_pad, -1)
            ops.zero_f32(ops.f32view(dwm))
            ops.conv_wgrad(self.x, dy, self.geom, dwm, nsplit=ctx.nsplit)
            ops.filter_unpack_grad(dwm, gw, self.cin_pad, accumulate=False)

    def dgrad(self, dy: Planes, x_act: Act) -> None:
        """Data gradient into x_act's gradient storage.  The first contribution is stored directly; later ones are
        added in the GEMM epilogue with vector float reductions (``accumulate=2``): every element receives exactly one
        add per launch, and positions no tap reaches keep their value."""
        ctx = self.ctx
        _, t, h, w, pitch = x_act.s.shape
        plan = dgrad_plan((t, h, w), self.k, self.stride, self.pad)
        acc = x_act.s.grad_written
        g = x_act.s.ensure_grad()
        if plan.needs_zero_fill and not acc:
            ops.zero_f32(x_act.grad_view())
        for sub in plan.subs:
            ntap = len(sub.tapmap)
            cp = ops.pad8(self.cout)
            f = ctx.scratch("dgf.hi", self.cin * ntap * cp, torch.bfloat16).view(self.cin, ntap * cp)
            flo = ctx.scratch("dgf.lo", self.cin * ntap * cp, torch.bfloat16).view(self.cin, ntap * cp) \
                if ctx.nsplit == 3 else None
            fm = ops.FilterMat(f, flo, self.cin, ntap, cp)
            ops.filter_pack(self.conv.weight, fm, tapmap=sub.tapmap, transpose=True)
            off, strides = dgrad_out_view((t, h, w), self.stride, sub, pitch, x_act.c0)
            ops.conv_igemm(dy, fm, ops.ConvGeom(sub.k, (1, 1, 1), sub.low, sub.out), g, strides, out_offset=off,
                           accumulate=2 if acc else 0, nsplit=ctx.nsplit)
        x_act.s.grad_written = True


class StemConvBN(ConvBN):
    """Stem conv (C_in <= 4, W stride 2) + BN through the W-shift kernels (csrc/conv_stem.cu): the clip is packed
    with W folded by the stride, so fprop / wgrad read each input row once per (kt, kh) instead of once per tap."""

    def __init__(self, name, conv, bn, ctx):
        super().__init__(name, conv, bn, ctx)
        self.g = ops.StemGeom(self.cin, self.cout, self.k, self.stride, self.pad)
        self.t8 = False

    @staticmethod
    def supported(conv: nn.Conv3d, w: int) -> bool:
        return (conv.out_channels <= 64 and conv.out_channels % 8 == 0 and
                ops.stem_supported(conv.in_channels, _t3(conv.kernel_size), _t3(conv.stride), _t3(conv.padding), w))

    def pack_input(self, x: torch.Tensor, key) -> "Act":
        n, c, t, h, w = x.shape
        x_f32 = x.contiguous().float()
        # 8 output channels: one GEMM row = 8 output pixels (Toeplitz operands, csrc/conv_stem8.cu) when the extent allows
        self.t8 = bool(self.cout == 8 and
                       ops.stem8_supported(self.cin, self.cout, self.k, self.stride, self.pad, t, h, w))
        if self.t8:
            xin = Act(self.ctx.storage((key, "t8"), *ops.stem8_plane_dims(n, t, h, w)))
            ops.stem8_input_fold(x_f32, xin.planes)
            return xin
        xin = Act(self.ctx.storage(key, n, t, h, w // 2, 8))
        ops.stem_input_fold(x_f32, xin.planes)
        return xin

    def fprop(self, x: Planes) -> torch.Tensor:
        ctx, g = self.ctx, self.g
        c = self.cout
        self._set_bn_mode()
        self.splits = self.bn.num_splits if (self.sub and self.bn_train) else 1
        want_stats = self.bn_train and self.splits == 1  # (sub-batch BN: statistics in a separate pass)
        if self.t8:
            n, t, h, w = x.n, x.t // 2, x.h * 2, (x.w // 8 - 1) * 16
            ot, oh, ow = g.out_dims(t, h, w)
            f = ctx.buf((self.name, "z.hi"), (self.k[0] * ops.STEM8_ZG * 64,), torch.bfloat16)
            flo = ctx.buf((self.name, "z.lo"), f.shape, torch.bfloat16) if ctx.nsplit == 3 else None
            ops.stem8_filter_fold(self.conv.weight, f, flo)
            y = ctx.buf((self.name, "y"), (n, ot, oh, ow, c))
            m_tiles = ops.stem8_m_tiles(x, g)
            stats = ctx.buf((self.name, "stats8"), (2, c, m_tiles)) if want_stats else None
            ops.stem8_fprop(x, f, flo, g, y, stats, nsplit=ctx.nsplit)
        else:
            n = x.n
            ot, oh, ow = g.out_dims(x.t, x.h, 2 * x.w)
            f = ctx.buf((self.name, "f.hi"), (self.cout, g.kfold), torch.bfloat16)
            flo = ctx.buf((self.name, "f.lo"), f.shape, torch.bfloat16) if ctx.nsplit == 3 else None
            fm = ops.FilterMat(f, flo, self.cout, g.kfold // 8, 8)
            ops.stem_filter_fold(self.conv.weight, g, fm)
            y = ctx.buf((self.name, "y"), (n, ot, oh, ow, c))
            m_tiles = ops.stem_m_tiles(x, g)
            stats = ctx.buf((self.name, "stats"), (2, c, m_tiles)) if want_stats else None
            ops.stem_fprop(x, fm, g, y, stats, nsplit=ctx.nsplit)
        self.rows_per_clip = ot * oh * ow
        self._bn_forward(y, stats, m_tiles, c, zero=False)
        self.x, self.y = x, y
        return y

    def wgrad(self, dy: Planes) -> None:
        ctx, g = self.ctx, self.g
        dwm = ctx.scratch("dwm", self.cout * g.kfold, F32).view(self.cout, g.kfold)
        ops.zero_f32(ops.f32view(dwm))
        if self.t8:
            ops.stem8_wgrad(self.x, dy, g, dwm, nsplit=ctx.nsplit)
        else:
            ops.stem_wgrad(self.x, dy, g, dwm, nsplit=ctx.nsplit)
        ops.stem_filter_unfold_grad(dwm, ctx.grad_of(self.conv.weight), g)

    def dgrad(self, dy, x_act):  # pragma: no cover - the clip needs no gradient
        raise RuntimeError("stem convolutions have no data gradient")


class GraphedProgram:
    """Forward and backward programs of one (mode, input-signature) captured as two CUDA graphs.

    Every buffer the programs touch is persistent (``Ctx`` caches, graph memory pool), every kernel argument
    (pointers, TMA tensor maps, geometry) is fixed for a given signature, and per-step randomness lives in device
    memory, so a replay is bit-for-bit the eager program minus ~1.6k launch calls and their host overhead."""

    def __init__(self, model, inputs: List[torch.Tensor], with_backward: bool = False):
        self.model = model
        self.params = list(model.parameters())
        self.pool = torch.cuda.graph_pool_handle()
        self.static_in = [torch.empty_like(x) for x in inputs]
        for s, x in zip(self.static_in, inputs):
            s.copy_(x)
        self.fwd_graph = torch.cuda.CUDAGraph()
        n0 = ops.launches()
        with torch.cuda.graph(self.fwd_graph, pool=self.pool):
            self.static_out = model._engine_forward(self.static_in)
        self.fwd_launches = ops.launches() - n0
        self.bwd_graph = None
        self.bwd_launches = 0
        self.static_dout = torch.empty_like(self.static_out)
        self.static_grads = None
        if with_backward:
            # the backward program is captured NOW, while the python-side saved state (unit.x / unit.y / _saved ...)
            # is the one this forward capture produced; a lazy capture could pick up another forward's state
            self._capture_backward()

    def _capture_backward(self) -> None:
        self.bwd_graph = torch.cuda.CUDAGraph()
        n0 = ops.launches()
        with torch.cuda.graph(self.bwd_graph, pool=self.pool):
            self.static_grads = self.model._engine_backward(self.static_dout)
        self.bwd_launches = ops.launches() - n0
        self.flat_grad = self.model.ctx.flat_grad

    def run_forward(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        for s, x in zip(self.static_in, inputs):
            if s.data_ptr() != x.data_ptr():
                s.copy_(x)
        self.fwd_graph.replay()
        ops.add_launches(self.fwd_launches)
        return self.static_out.clone()

    def run_backward(self, dout: torch.Tensor):
        if self.bwd_graph is None:
            raise RuntimeError("this program was captured without a backward (forward ran under no_grad)")
        if self.static_grads is not None:
            # gradient accumulation (zero_grad(set_to_none=False), or .grad re-pointed at the bucket by
            # allreduce_flat_gradients): a live .grad must never alias the static slot the replay overwrites
            for p, g in zip(self.params, self.static_grads):
                if g is not None and p.grad is not None and p.grad.data_ptr() == g.data_ptr():
                    p.grad = p.grad.clone()
        self.static_dout.copy_(dout)
        self.bwd_graph.replay()
        self.model.ctx.flat_grad = self.flat_grad  # the bucket allreduce_gradients() exchanges
        ops.add_launches(self.bwd_launches)
        return self.static_grads


def pointer_signature(model: "EngineModel", params) -> int:
    """Hash of the device pointers a captured program bakes in: every parameter and every BatchNorm buffer."""
    ptrs = [p.data_ptr() for p in params]
    for b in model._all_bns():
        if b.running_mean is not None:
            ptrs.append(b.running_mean.data_ptr())
            ptrs.append(b.running_var.data_ptr())
            ptrs.append(b.num_batches_tracked.data_ptr())
    return hash(tuple(ptrs))


def bn_momentum_signature(model: "EngineModel") -> Tuple:
    bns = model._all_bns()
    if not bns or not model.training:
        return ()
    first = bns[0].momentum
    return (first,) if all(b.momentum == first for b in bns) else tuple(b.momentum for b in bns)


def bn_mode(ctx: Ctx, bn: nn.Module) -> bool:
    """True: this BN normalises with batch statistics and updates its running buffers (model and module both in
    training mode); False: it applies its running statistics, in eval and under MODEL.FROZEN_BN alike."""
    return ctx.training and bn.training


def bn_mode_signature(model: "EngineModel") -> Tuple:
    """Indices of the BatchNorm modules in eval mode inside a training model (MODEL.FROZEN_BN freezes them all,
    a hand-frozen subset some): a captured program bakes each BN's mode into its kernel arguments."""
    if not model.training:
        return ()
    return tuple(i for i, b in enumerate(model._all_bns()) if not b.training)


def program_key(model: "EngineModel", needs_grad: bool, inputs: Sequence[torch.Tensor]) -> Tuple:
    """Arena / CUDA-graph key of one forward: mode, grad mode, input signature, BN momenta and BN modes."""
    # BatchNorm momentum is a by-value kernel argument (baked into a captured program): precise-BN (fvcore
    # update_bn_stats, tools/train_net.py:425-446) temporarily sets it to 1.0, so it is part of the signature
    return (model.training, needs_grad, tuple((tuple(x.shape), x.dtype) for x in inputs), bn_momentum_signature(model),
            bn_mode_signature(model))


class ModelFunction(torch.autograd.Function):
    """The whole engine model as one autograd node: forward(program) / backward(program)."""

    @staticmethod
    def forward(fctx, model, n_inputs, *tensors):
        inputs = [t.contiguous() for t in tensors[:n_inputs]]
        fctx.model = model
        fctx.n_inputs = n_inputs
        fctx.prog = None
        # (grad mode is always off inside Function.forward; needs_input_grad says whether a backward can follow)
        needs_grad = any(fctx.needs_input_grad)
        key = program_key(model, needs_grad, inputs)
        arena = model.ctx.use_arena(key)
        arena.generation += 1
        model._fwd_generation += 1
        fctx.key, fctx.arena, fctx.arena_gen, fctx.model_gen = key, arena, arena.generation, model._fwd_generation
        if model.cuda_graphs and inputs[0].is_cuda:
            prog = model._graphs.get(key)
            sig = pointer_signature(model, tensors[n_inputs:])
            if prog is not None and prog.ptr_sig != sig:
                # a parameter or BatchNorm buffer was REPLACED (fvcore's precise-BN assigns new running_mean / running_var
                # tensors, module.to() re-allocates): the captured programs hold stale device pointers - capture again
                model._graphs.pop(key, None)
                prog = None
            if prog is None:
                seen = model._graph_seen.get(key, 0)
                model._graph_seen[key] = seen + 1
                if seen >= model.graph_warmup:  # buffers / function attributes exist: capture now
                    prog = GraphedProgram(model, inputs, with_backward=needs_grad)
                    prog.ptr_sig = sig
                    model._graphs[key] = prog
                    arena.on_evict.append(lambda k=key: (model._graphs.pop(k, None), model._graph_seen.pop(k, None)))
            if prog is not None:
                fctx.prog = prog
                return prog.run_forward(inputs)
        return model._engine_forward(inputs)

    @staticmethod
    def backward(fctx, dout):
        model = fctx.model
        dout = dout.contiguous()
        if fctx.arena.generation != fctx.arena_gen:
            raise RuntimeError(
                "slowfast_b200: another forward with the same input signature ran before this backward; the engine "
                "keeps ONE set of saved activations per signature (run backward before the next forward)")
        if fctx.prog is not None:
            grads = fctx.prog.run_backward(dout)
        else:
            if model._fwd_generation != fctx.model_gen:
                raise RuntimeError(
                    "slowfast_b200: another forward ran between this (eager) forward and its backward; the saved "
                    "activations are per model - run backward first, or enable cfg.B200.CUDA_GRAPH")
            model.ctx.use_arena(fctx.key)
            grads = model._engine_backward(dout)
        if model.flat_grad_only:
            # the caller consumes ctx.flat_grad directly (slowfast_b200.optim.FlatOptimizer): no param.grad copies
            return (None, None) + (None,) * (fctx.n_inputs + len(grads))
        # (None: a parameter in front of MODEL.DETACH_FINAL_FC's detach, whose .grad stays None as in the reference)
        return (None, None) + (None,) * fctx.n_inputs + tuple(grads)


class EngineModel(nn.Module):
    """What every engine network provides to ``ModelFunction`` and ``GraphedProgram``.

    A subclass calls ``super().__init__(cfg)`` before it registers any module, and supplies
      * ``forward``: its own input handling, then ``self._run(inputs)`` with the list of input tensors;
      * ``_forward_program(inputs)``: the forward kernels, returning the output tensor autograd receives;
      * ``_backward_program(dout)``: the backward kernels, writing the gradient of every ``grad_params()`` entry into
        its slot ``ctx.grad_of(p)``; under MODEL.DETACH_FINAL_FC it stops at the detach;
      * a module ``head`` with ``detach_final_fc`` and, when that is set, ``params_after_detach()`` (the pre-training
        models, which have no classification head, have no ``head``).

    The base holds the rest:
      * ``ctx``: the execution context (``Ctx``) at cfg.B200.NSPLIT;
      * ``cuda_graphs``: capture each input signature's programs as CUDA graphs after ``graph_warmup`` eager calls
        (cfg.B200.CUDA_GRAPH; a config without a B200 section, such as the reference's own, keeps the default on);
      * ``flat_grad_only``: autograd receives no parameter gradients, the caller reads ``ctx.flat_grad`` itself
        (``optim.FlatOptimizer``);
      * ``_seed``: cfg.RNG_SEED, the seed of the device-side dropout / stochastic-depth draws;
      * the BatchNorm registry behind the program key and the ``num_batches_tracked`` updates;
      * the flat gradient bucket (``grad_params``) and its data-parallel exchange (``allreduce_gradients``).
    The base registers no parameter, buffer or submodule and draws no random numbers, so a subclass's ``state_dict``
    and initial values stay the reference's."""

    cuda_graphs = True
    graph_warmup = 2
    flat_grad_only = False

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.ctx = Ctx(nsplit_of(cfg))
        b200 = getattr(cfg, "B200", None)
        if b200 is not None and "CUDA_GRAPH" in b200:
            self.cuda_graphs = bool(b200["CUDA_GRAPH"])
        self._graphs: Dict[Tuple, GraphedProgram] = {}
        self._graph_seen: Dict[Tuple, int] = {}
        self._fwd_generation = 0
        self._seed = int(getattr(cfg, "RNG_SEED", 0))
        self._drop_counter: Optional[torch.Tensor] = None
        self._bns: Optional[Tuple[List[nn.Module], List[nn.Module]]] = None

    def _run(self, inputs: Sequence[torch.Tensor]) -> torch.Tensor:
        return ModelFunction.apply(self, len(inputs), *inputs, *self.parameters())

    def _engine_forward(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
        ctx.device = inputs[0].device
        ctx.training = self.training
        if ctx.device.type != "cuda":
            raise ops.L.NativeLibraryError("slowfast_b200 runs on CUDA devices only (no CPU fallback)")
        out = self._forward_program(inputs)
        if ctx.training:
            # torch's BatchNorm increments num_batches_tracked once per training forward of a BN in training mode (one
            # fused op for all BNs); a frozen BN (module in eval) keeps its count
            ts = [b.num_batches_tracked for b in self._train_bns() if b.num_batches_tracked is not None and b.training]
            if ts:
                torch._foreach_add_(ts, 1)
        return out

    def _engine_backward(self, dout: torch.Tensor) -> List[Optional[torch.Tensor]]:
        params = list(self.parameters())
        self.ctx.begin_backward(self.grad_params())
        self._backward_program(dout)
        return self.ctx.grads(params)

    def grad_params(self) -> List[nn.Parameter]:
        """The parameters the backward writes gradients for, in flat-bucket order: all of them, or the head's
        parameters behind MODEL.DETACH_FINAL_FC's detach."""
        head = getattr(self, "head", None)
        if head is not None and head.detach_final_fc:
            return head.params_after_detach()
        return list(self.parameters())

    def allreduce_gradients(self, group=None) -> None:
        """Data-parallel exchange step (SURVEY.md §8e): ONE NCCL all-reduce (average) over the flat gradient
        bucket the last backward filled; ``param.grad`` is re-pointed at the bucket slices where autograd made a
        private copy.  (Under the reference's build_model the DDP wrapper does its own bucketing instead.)"""
        assert self.ctx.flat_grad is not None, "call after backward()"
        allreduce_flat_gradients(self.ctx.flat_grad, self.grad_params(), group, repoint=not self.flat_grad_only)

    def _bn_registry(self) -> Tuple[List[nn.Module], List[nn.Module]]:
        if self._bns is None:
            mods = list(self.modules())
            eval_only = {id(m.bn) for m in mods if is_sub_bn(m)}
            bns = [m for m in mods if isinstance(m, nn.modules.batchnorm._BatchNorm)]
            self._bns = (bns, [b for b in bns if id(b) not in eval_only])
        return self._bns

    def _all_bns(self) -> List[nn.Module]:
        """Every BatchNorm module in module order, both BNs of a sub-batch BN included (fvcore's precise-BN sees them
        all too): their momenta, modes and buffer pointers are part of a captured program's key."""
        return self._bn_registry()[0]

    def _train_bns(self) -> List[nn.Module]:
        """The BNs a training forward runs: a sub-batch BN runs its split_bn only, never its eval ``bn``."""
        return self._bn_registry()[1]

    def _head_drop_counter(self) -> torch.Tensor:
        """The head dropout's device-side step counter: one per model, so that the captured programs of every input
        signature advance the same draw.  Created at zero on the device of the forward, not in ``__init__``: a plain
        tensor attribute does not follow ``module.to()``."""
        if self._drop_counter is None or self._drop_counter.device != self.ctx.device:
            self._drop_counter = torch.zeros(1, dtype=torch.int64, device=self.ctx.device)
        return self._drop_counter


class Namespace(nn.Module):
    """Inert container used to mirror the reference's module tree (state_dict key parity)."""

    def forward(self, *a, **k):  # pragma: no cover - containers are never called
        raise RuntimeError("engine containers hold parameters only; call the top-level model")
