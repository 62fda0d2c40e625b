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
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import ops
from .conv_plan import dgrad_out_view, dgrad_plan
from .ops import F32, F32View, Planes


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
        # batched filter packing (opt-in): one plan per phase, recorded on the first pass
        self.pack_plans: Dict[str, ops.PackPlan] = {}
        self._pack_phase: Optional[str] = None
        self._pack_recording = False

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

    # batched filter packing --------------------------------------------------------------------------
    def begin_phase(self, phase: str) -> None:
        """Called by the model at the start of its forward / backward program."""
        if not BATCHED_PACK:
            return
        self._pack_phase = phase
        phase = (phase, self.arena.key)
        self._pack_phase = phase
        plan = self.pack_plans.get(phase)
        if plan is not None and plan.ready and plan.signature() == plan._sig:
            plan.launch()              # every filter of this phase is packed now
            self._pack_recording = False
        else:
            self.pack_plans[phase] = ops.PackPlan()
            self._pack_recording = True

    def end_phase(self) -> None:
        if not BATCHED_PACK or self._pack_phase is None:
            return
        if self._pack_recording:
            plan = self.pack_plans[self._pack_phase]
            if plan.jobs:
                plan.finalize(self.device)
        self._pack_phase, self._pack_recording = None, False

    def pack(self, w: torch.Tensor, fm, tapmap=None, transpose: bool = False) -> None:
        """Filter packing of one layer: immediate (default), or part of the phase's batched launch."""
        if BATCHED_PACK and self._pack_phase is not None:
            if not self._pack_recording:
                if fm.ntaps <= 32:
                    return             # already packed by begin_phase's launch (static program: same jobs every pass)
            else:
                self.pack_plans[self._pack_phase].record(w, fm, tapmap, transpose)
        ops.filter_pack(w, fm, tapmap=tapmap, transpose=transpose)

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


# Second and later data-gradient contributions to one tensor: read-modify-write in the GEMM epilogue (coalesced since
# the epilogue stores whole 128-byte lines) instead of a scratch tensor + add pass.  Measured SLOWER (the dependent
# load-add-store chain is latency-bound with 4 epilogue warps: 50.2 vs 37.9 ms/step), so it is opt-in: SFB_RMW_DGRAD=1.
RMW_DGRAD = os.environ.get("SFB_RMW_DGRAD", "0") != "0"
# r2: the same accumulation with `red.global.add.v4.f32` (no load, no dependent chain): every element still receives exactly one
# add per launch, so the result equals the scratch + add pass bit for bit; SFB_ATOMIC_DGRAD=0 = scratch tensor + add pass.
ATOMIC_DGRAD = os.environ.get("SFB_ATOMIC_DGRAD", "1") != "0"
# fast-pathway stem weight gradient on the fp32 pipes (csrc/conv_stem.cu, stem_wgrad_direct); 0 = tensor-core W-shift path
DIRECT_STEM_WGRAD = os.environ.get("SFB_DIRECT_STEM_WGRAD", "1") != "0"
# Toeplitz wgmma kernels for the 8-channel (fast pathway) stem, csrc/conv_stem8.cu: "0" = W-shift fprop + SIMT wgrad of r1
STEM_T8 = os.environ.get("SFB_STEM_T8", "1") != "0"
STEM_T8_WGRAD = os.environ.get("SFB_STEM_T8_WGRAD", "1") != "0"
# one filter-packing launch per phase (ops.PackPlan) instead of one per layer.  Under CUDA-graph replay the ~250 tiny pack
# kernels are already hidden, so it stays opt-in; it matters for eager (graph-less) runs.
BATCHED_PACK = os.environ.get("SFB_BATCHED_PACK", "0") != "0"


def _t3(v) -> Tuple[int, int, int]:
    return tuple(int(x) for x in v)


class ConvBN:
    """nn.Conv3d (bias-free) followed by nn.BatchNorm3d, executed by the library's kernels.

    The torch modules are parameter containers only (their ``forward`` is never called); they keep the reference's
    ``state_dict`` names and ``_NormBase`` identity (optimizer.py:41-56, checkpoint.py, precise-BN)."""

    def __init__(self, name: str, conv: nn.Conv3d, bn: nn.BatchNorm3d, ctx: Ctx):
        assert conv.bias is None and conv.groups == 1 and _t3(conv.dilation) == (1, 1, 1), \
            f"{name}: only dense, bias-free, undilated Conv3d is on this path"
        self.name, self.conv, self.bn, self.ctx = name, conv, bn, ctx
        assert bn is None or bn.momentum is not None, \
            f"{name}: BatchNorm momentum=None (cumulative moving average) is not on the engine path"
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

    def fprop(self, x: Planes) -> torch.Tensor:
        """y = conv(x) (fp32, dense channels-last) + BN statistics -> self.scale/self.shift."""
        ctx = self.ctx
        assert x.c == self.cin_pad, (self.name, x.c, self.cin_pad)
        geom = ops.fprop_geom(x, self.k, self.stride, self.pad)
        ot, oh, ow = geom.out
        f = ctx.buf((self.name, "f.hi"), (self.cout, self.taps * self.cin_pad), torch.bfloat16)
        flo = ctx.buf((self.name, "f.lo"), f.shape, torch.bfloat16) if ctx.nsplit == 3 else None
        fm = ops.FilterMat(f, flo, self.cout, self.taps, self.cin_pad)
        ctx.pack(self.conv.weight, fm)
        c, cp = self.cout, self.cout_pad
        y = ctx.buf((self.name, "y"), (x.n, ot, oh, ow, cp))
        m_tiles = ops.conv_m_tiles(x.n, geom)
        stats = ctx.buf((self.name, "stats"), (2, c, m_tiles)) if (ctx.training and self.bn is not None) else None
        # (the epilogue stores whole float4 groups: columns [c, cp) receive the zero accumulators of filter rows
        # the TMA box reads out of bounds)
        ops.conv_igemm(x, fm, geom, y, (ot * oh * ow * cp, oh * ow * cp, ow * cp, cp), stats=stats, nsplit=ctx.nsplit)
        self.x, self.geom, self.y = x, geom, y
        if self.bn is None:
            return y
        self.scale = ctx.buf((self.name, "scale"), (cp,), zero=True)
        self.shift = ctx.buf((self.name, "shift"), (cp,), zero=True)
        self.mean = ctx.buf((self.name, "mean"), (cp,), zero=True)
        self.invstd = ctx.buf((self.name, "invstd"), (cp,), zero=True)
        bn = self.bn
        ops.bn_finalize(stats, m_tiles, c, x.n * ot * oh * ow, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                        bn.momentum if bn.momentum is not None else 0.1, bn.eps, ctx.training, self.scale,
                        self.shift, self.mean, self.invstd)
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
                   ctx.grad_of(bn.bias), dy, partials, coef, training=ctx.training, dres=dres,
                   dres_accumulate=dres_accumulate, c_valid=self.cout,
                   mask_affine=(self.scale, self.shift) if mask_from_y else None)
        self.wgrad(dy)
        if x_act is not None:
            self.dgrad(dy, x_act)

    def _bwd_scratch(self, rows, c):
        nb = ops.L.load().sfb_bn_bwd_blocks(rows, c)
        return (self.ctx.scratch("bnb.partials", nb * 2 * c, F32).view(nb, 2, c),
                self.ctx.scratch("bnb.coef", 3 * c, F32).view(3, c))

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
        """Data gradient into x_act's gradient storage.  The first contribution is stored directly; later ones go
        through a scratch tensor of the same geometry and are merged by one coalesced add pass (a read-modify-write
        GEMM epilogue would touch 32 different cache lines per instruction)."""
        ctx = self.ctx
        n, t, h, w, pitch = x_act.s.shape
        plan = dgrad_plan((t, h, w), self.k, self.stride, self.pad)
        acc = x_act.s.grad_written
        rmw = acc and (RMW_DGRAD or ATOMIC_DGRAD)  # (positions no tap reaches simply keep their value)
        acc_mode = (2 if ATOMIC_DGRAD and not RMW_DGRAD else 1) if rmw else 0
        if acc and not rmw:
            g = ctx.scratch("dgrad.tmp", n * t * h * w * pitch, F32).view(n, t, h, w, pitch)
            view = F32View(g, n * t * h * w, x_act.c, pitch, x_act.c0)
        else:
            g = x_act.s.ensure_grad()
            view = x_act.grad_view()
        if plan.needs_zero_fill and not rmw:
            ops.zero_f32(view)
        for i, sub in enumerate(plan.subs):
            ntap = len(sub.tapmap)
            cp = ops.pad8(self.cout)
            if BATCHED_PACK:  # the batched launch packs ahead of time: every (layer, sub-problem) owns its buffers
                f = ctx.buf((self.name, "dgf.hi", i), (self.cin, ntap * cp), torch.bfloat16)
                flo = ctx.buf((self.name, "dgf.lo", i), (self.cin, ntap * cp), torch.bfloat16) \
                    if ctx.nsplit == 3 else None
            else:
                f = ctx.scratch("dgf.hi", self.cin * ntap * cp, torch.bfloat16).view(self.cin, ntap * cp)
                flo = ctx.scratch("dgf.lo", self.cin * ntap * cp, torch.bfloat16).view(self.cin, ntap * cp) \
                    if ctx.nsplit == 3 else None
            fm = ops.FilterMat(f, flo, self.cin, ntap, cp)
            ctx.pack(self.conv.weight, fm, tapmap=sub.tapmap, transpose=True)
            off, strides = dgrad_out_view((t, h, w), self.stride, sub, pitch, x_act.c0)
            ops.conv_igemm(dy, fm, ops.ConvGeom(sub.k, (1, 1, 1), sub.low, sub.out), g, strides, out_offset=off,
                           accumulate=acc_mode, nsplit=ctx.nsplit)
        if acc and not rmw:
            ops.add_f32(x_act.grad_view(), view)
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
        self.x_f32 = x.contiguous().float()  # kept for the direct weight-gradient kernel (narrow stems)
        # 8 output channels: one GEMM row = 8 output pixels (Toeplitz operands, csrc/conv_stem8.cu) when the extent allows
        self.t8 = bool(STEM_T8 and self.cout == 8 and
                       ops.stem8_supported(self.cin, self.cout, self.k, self.stride, self.pad, t, h, w))
        if self.t8:
            xin = Act(self.ctx.storage((key, "t8"), *ops.stem8_plane_dims(n, t, h, w)))
            ops.stem8_input_fold(self.x_f32, xin.planes)
            return xin
        xin = Act(self.ctx.storage(key, n, t, h, w // 2, 8))
        ops.stem_input_fold(self.x_f32, xin.planes)
        return xin

    def fprop(self, x: Planes) -> torch.Tensor:
        ctx, g = self.ctx, self.g
        c = self.cout
        if self.t8:
            n, t, h, w = x.n, x.t // 2, x.h * 2, (x.w // 8 - 1) * 16
            ot, oh, ow = g.out_dims(t, h, w)
            f = ctx.buf((self.name, "z.hi"), (self.k[0] * ops.STEM8_ZG * 64,), torch.bfloat16)
            flo = ctx.buf((self.name, "z.lo"), f.shape, torch.bfloat16) if ctx.nsplit == 3 else None
            ops.stem8_filter_fold(self.conv.weight, f, flo)
            y = ctx.buf((self.name, "y"), (n, ot, oh, ow, c))
            m_tiles = ops.stem8_m_tiles(x, g)
            stats = ctx.buf((self.name, "stats8"), (2, c, m_tiles)) if ctx.training else None
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
            stats = ctx.buf((self.name, "stats"), (2, c, m_tiles)) if ctx.training else None
            ops.stem_fprop(x, fm, g, y, stats, nsplit=ctx.nsplit)
        self.scale = ctx.buf((self.name, "scale"), (c,))
        self.shift = ctx.buf((self.name, "shift"), (c,))
        self.mean = ctx.buf((self.name, "mean"), (c,))
        self.invstd = ctx.buf((self.name, "invstd"), (c,))
        bn = self.bn
        ops.bn_finalize(stats, m_tiles, c, n * ot * oh * ow, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                        bn.momentum if bn.momentum is not None else 0.1, bn.eps, ctx.training, self.scale,
                        self.shift, self.mean, self.invstd)
        self.x, self.y = x, y
        return y

    def wgrad(self, dy: Planes) -> None:
        ctx, g = self.ctx, self.g
        if self.t8 and STEM_T8_WGRAD and dy.pitch == 8:
            dwm = ctx.scratch("dwm", self.cout * g.kfold, F32).view(self.cout, g.kfold)
            ops.zero_f32(ops.f32view(dwm))
            ops.stem8_wgrad(self.x, dy, g, dwm, nsplit=ctx.nsplit)
            ops.stem_filter_unfold_grad(dwm, ctx.grad_of(self.conv.weight), g)
            return
        if (DIRECT_STEM_WGRAD and self.cout == 8 and self.cin == 3 and self.stride == (1, 2, 2) and self.pad[2] <= 4
                and self.cin * self.taps <= 768 and dy.pitch == 8):
            # 8 output channels fill 8 of the 128 UMMA rows: the fp32 SIMT kernel is ~3x faster and exact
            ops.stem_wgrad_direct(self.x_f32, dy, self.k, self.stride, self.pad, ctx.grad_of(self.conv.weight))
            return
        assert not self.t8, "the W-shift weight gradient needs the W-shift clip layout (SFB_STEM_T8_WGRAD=0 needs the direct kernel)"
        dwm = ctx.scratch("dwm", self.cout * g.kfold, F32).view(self.cout, g.kfold)
        ops.zero_f32(ops.f32view(dwm))
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
                if p.grad is not None and p.grad.data_ptr() == g.data_ptr():
                    p.grad = p.grad.clone()
        self.static_dout.copy_(dout)
        self.bwd_graph.replay()
        self.model.ctx.flat_grad = self.flat_grad  # the bucket allreduce_gradients() exchanges
        ops.add_launches(self.bwd_launches)
        return self.static_grads


def pointer_signature(model, params) -> int:
    """Hash of the device pointers a captured program bakes in: every parameter and every BatchNorm buffer."""
    bn_momentum_signature(model)  # (fills the BN module cache)
    ptrs = [p.data_ptr() for p in params]
    for b in model.__dict__["_bn_list"]:
        if b.running_mean is not None:
            ptrs.append(b.running_mean.data_ptr())
            ptrs.append(b.running_var.data_ptr())
            ptrs.append(b.num_batches_tracked.data_ptr())
    return hash(tuple(ptrs))


def bn_momentum_signature(model) -> Tuple:
    bns = model.__dict__.get("_bn_list")
    if bns is None:
        bns = [m for m in model.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]
        object.__setattr__(model, "_bn_list", bns)
    if not bns or not model.training:
        return ()
    first = bns[0].momentum
    return (first,) if all(b.momentum == first for b in bns) else tuple(b.momentum for b in bns)


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
        # BatchNorm momentum is a by-value kernel argument (baked into a captured program): precise-BN (fvcore
        # update_bn_stats, tools/train_net.py:425-446) temporarily sets it to 1.0, so it is part of the signature
        key = (model.training, needs_grad, tuple((tuple(x.shape), x.dtype) for x in inputs), bn_momentum_signature(model))
        arena = model.ctx.use_arena(key)
        arena.generation += 1
        gen = getattr(model, "_fwd_generation", 0) + 1
        object.__setattr__(model, "_fwd_generation", gen)
        fctx.key, fctx.arena, fctx.arena_gen, fctx.model_gen = key, arena, arena.generation, gen
        if getattr(model, "cuda_graphs", False) and inputs[0].is_cuda:
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
            if getattr(model, "_fwd_generation", 0) != fctx.model_gen:
                raise RuntimeError(
                    "slowfast_b200: another forward ran between this (eager) forward and its backward; the saved "
                    "activations are per model - run backward first, or enable cfg.B200.CUDA_GRAPH")
            model.ctx.use_arena(fctx.key)
            grads = model._engine_backward(dout)
        if getattr(model, "flat_grad_only", False):
            # the caller consumes ctx.flat_grad directly (slowfast_b200.optim.FlatOptimizer): no param.grad copies
            return (None, None) + (None,) * (fctx.n_inputs + len(grads))
        return (None, None) + (None,) * fctx.n_inputs + tuple(grads)


class Namespace(nn.Module):
    """Inert container used to mirror the reference's module tree (state_dict key parity)."""

    def forward(self, *a, **k):  # pragma: no cover - containers are never called
        raise RuntimeError("engine containers hold parameters only; call the top-level model")


def bump_num_batches_tracked(bns: List[nn.BatchNorm3d]) -> None:
    """torch's BatchNorm increments num_batches_tracked once per training forward (one fused op for all BNs)."""
    ts = [b.num_batches_tracked for b in bns if b.num_batches_tracked is not None]
    if ts:
        torch._foreach_add_(ts, 1)
