"""Engine-native optimizer step on the flat gradient bucket (SURVEY.md section 8f-1).

The engine's backward writes every parameter gradient into ONE contiguous fp32 bucket (``model.ctx.flat_grad``, the single
all-reduce message).  ``FlatOptimizer`` consumes that bucket directly: gradient norm (+ optional clipping, + AMP unscale)
and the SGD-nesterov / AdamW update of every parameter are three kernel launches in total (csrc/optim.cu), instead of the
reference's per-tensor ATen kernels (slowfast/models/optimizer.py:105-136 builds torch.optim.SGD / AdamW; tools/train_net.py
:154-172 computes the norm with one torch.norm per parameter).  Parameter grouping restates ``construct_optimizer``
(optimizer.py:26-91): BatchNorm parameters (BN.WEIGHT_DECAY), 1-D / bias / ``no_weight_decay()`` parameters (0) and the
rest (SOLVER.WEIGHT_DECAY).

This is an engine-side API for loops that own their optimizer (bench.py); the reference's unmodified ``train_epoch`` keeps
using the torch optimizer its own ``construct_optimizer`` built, on the ``param.grad`` tensors autograd hands it.
With ``model.flat_grad_only = True`` the autograd node stops materialising ``param.grad`` (one copy kernel per parameter).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

from . import lib as L
from .engine import flat_offsets

CHUNK = 8192  # elements per thread block


def param_groups_from_cfg(model: nn.Module, cfg) -> List[Dict]:
    """The three groups of slowfast/models/optimizer.py:26-80 (LAYER_DECAY == 1): BN, zero-weight-decay, the rest."""
    solver = cfg.SOLVER
    skip = model.no_weight_decay() if hasattr(model, "no_weight_decay") else {}
    bn, rest, zero = [], [], []
    for name_m, m in model.named_modules():
        is_bn = isinstance(m, nn.modules.batchnorm._NormBase)
        for name_p, p in m.named_parameters(recurse=False):
            name = f"{name_m}.{name_p}".strip(".")
            if not p.requires_grad:
                continue
            if is_bn:
                bn.append(p)
            elif any(k in name for k in skip):
                zero.append(p)
            elif getattr(solver, "ZERO_WD_1D_PARAM", False) and (p.dim() == 1 or name.endswith(".bias")):
                zero.append(p)
            else:
                rest.append(p)
    groups = [dict(params=bn, weight_decay=float(cfg.BN.WEIGHT_DECAY)),
              dict(params=rest, weight_decay=float(solver.WEIGHT_DECAY)),
              dict(params=zero, weight_decay=0.0)]
    return [g for g in groups if g["params"]]


class FlatOptimizer:
    """SGD (momentum / nesterov / dampening) or AdamW over the engine's flat gradient bucket.

    ``groups``: list of ``{"params": [...], "weight_decay": w, "lr": optional, "layer_decay": optional}``; parameters not
    listed are not updated.  ``clip_grad_l2norm`` > 0 scales every gradient by min(1, max_norm / (||g|| + 1e-6))
    (torch.nn.utils.clip_grad_norm_).  ``step(grad_scale=s)`` divides the gradients by ``s`` first (AMP loss scale)."""

    def __init__(self, model: nn.Module, kind: str, groups: Optional[Sequence[Dict]] = None, lr: float = 0.1,
                 momentum: float = 0.9, dampening: float = 0.0, nesterov: bool = True, weight_decay: float = 0.0,
                 betas=(0.9, 0.999), eps: float = 1e-8, clip_grad_l2norm: float = 0.0):
        assert kind in ("sgd", "adamw")
        self.model, self.kind = model, kind
        self.momentum, self.dampening, self.nesterov = float(momentum), float(dampening), bool(nesterov)
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        self.clip = float(clip_grad_l2norm)
        # the bucket holds the parameters the backward writes (all of them, or the head under MODEL.DETACH_FINAL_FC);
        # the others keep their values, momentum and weight decay included, as torch SGD leaves a None .grad
        params = model.grad_params() if hasattr(model, "grad_params") else list(model.parameters())
        written = {id(p) for p in params}
        if groups is None:
            groups = [dict(params=[p for p in params if p.requires_grad], weight_decay=weight_decay)]
        self.param_groups = []
        for g in groups:
            self.param_groups.append(dict(params=[p for p in g["params"] if id(p) in written], lr=float(g.get("lr", lr)),
                                          weight_decay=float(g.get("weight_decay", weight_decay)),
                                          layer_decay=float(g.get("layer_decay", 1.0))))
        self._params = params
        self._offsets, self._total = flat_offsets(params)
        self._steps = 0
        self._dev = None

    # ------------------------------------------------------------------------------------------ setup (first step)
    def _setup(self, device) -> None:
        lib = L.load()
        assert lib.sfb_opt_chunk_size() == C.sizeof(L.OptChunk)
        off_of = {id(p): o for p, o in zip(self._params, self._offsets)}
        chunks = []
        for gi, g in enumerate(self.param_groups):
            for p in g["params"]:
                assert p.is_contiguous() and p.dtype == torch.float32 and p.device == device
                n, base, ptr = p.numel(), off_of[id(p)], p.data_ptr()
                for c0 in range(0, n, CHUNK):
                    chunks.append((ptr + 4 * c0, base + c0, min(CHUNK, n - c0), gi))
        arr = (L.OptChunk * len(chunks))()
        for k, (ptr, off, cnt, gi) in enumerate(chunks):
            arr[k].param, arr[k].offset, arr[k].count, arr[k].group = ptr, off, cnt, gi
        self._table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(device)
        self._n_chunks = len(chunks)
        self._ptrs = [p.data_ptr() for g in self.param_groups for p in g["params"]]
        self._state1 = torch.zeros(self._total, dtype=torch.float32, device=device)
        self._state2 = torch.zeros(self._total, dtype=torch.float32, device=device) if self.kind == "adamw" else None
        self._partials = torch.empty(lib.sfb_flat_sumsq_blocks(), dtype=torch.float64, device=device)
        self._norm = torch.ones(3, dtype=torch.float32, device=device)
        self._glr = torch.empty(len(self.param_groups), dtype=torch.float32, device=device)
        self._gwd = torch.empty(len(self.param_groups), dtype=torch.float32, device=device)
        self._hyper_host = None
        self._dev = device

    def _push_hyper(self) -> None:
        lr = [g["lr"] * g["layer_decay"] for g in self.param_groups]
        wd = [g["weight_decay"] for g in self.param_groups]
        if self._hyper_host != (lr, wd):   # the LR schedule changes it (once per iteration at most): 2 tiny H2D copies
            self._glr.copy_(torch.tensor(lr, dtype=torch.float32), non_blocking=True)
            self._gwd.copy_(torch.tensor(wd, dtype=torch.float32), non_blocking=True)
            self._hyper_host = (lr, wd)

    # ------------------------------------------------------------------------------------------ public API
    def set_lr(self, new_lr: float) -> None:
        """slowfast/models/optimizer.py set_lr: every group's lr (scaled by its layer_decay at use)."""
        for g in self.param_groups:
            g["lr"] = float(new_lr)

    def zero_grad(self, set_to_none: bool = True) -> None:
        """The bucket is rewritten by every backward; only stale ``param.grad`` views are dropped."""
        if not getattr(self.model, "flat_grad_only", False):
            for p in self._params:
                p.grad = None

    @property
    def grad_norm(self) -> torch.Tensor:
        """Device scalar: L2 norm of the (unscaled) gradient the last ``step`` saw (get_grad_norm_, optimizer.py:362)."""
        return self._norm[0]

    def state_tensors(self):
        return dict(state1=self._state1, state2=self._state2, steps=self._steps)

    @torch.no_grad()
    def step(self, grad_scale: float = 1.0) -> None:
        flat = self.model.ctx.flat_grad
        if flat is None:
            raise RuntimeError("FlatOptimizer.step(): no gradient bucket - call after backward()")
        if self._dev is None:
            self._setup(flat.device)
        assert flat.numel() == self._total and flat.device == self._dev
        lib = L.load()
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self._push_hyper()
        L.check(lib.sfb_flat_sumsq(flat.data_ptr(), self._total, self._partials.data_ptr(), self.clip, 1.0 / grad_scale,
                                   self._norm.data_ptr(), st), "sfb_flat_sumsq")
        self._steps += 1
        if self.kind == "sgd":
            L.check(lib.sfb_flat_sgd(self._table.data_ptr(), self._n_chunks, flat.data_ptr(), self._state1.data_ptr(),
                                     self._glr.data_ptr(), self._gwd.data_ptr(), self._norm.data_ptr(), self.momentum,
                                     self.dampening, 1 if self.nesterov else 0, 1 if self._steps == 1 else 0, st),
                    "sfb_flat_sgd")
        else:
            L.check(lib.sfb_flat_adamw(self._table.data_ptr(), self._n_chunks, flat.data_ptr(), self._state1.data_ptr(),
                                       self._state2.data_ptr(), self._glr.data_ptr(), self._gwd.data_ptr(),
                                       self._norm.data_ptr(), self.betas[0], self.betas[1], self.eps, self._steps, st),
                    "sfb_flat_adamw")
        from . import ops
        ops.add_launches(3)
