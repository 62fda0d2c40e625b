"""MoCo pre-training (slowfast/models/contrastive.py ContrastiveModel, CONTRASTIVE.TYPE moco) on the engine.

``B200ContrastiveModel`` IS the reference's ``ContrastiveModel`` - queue, InfoNCE logits, batch shuffle, kNN memory and
momentum annealing are its code - with two changes:

  * ``backbone`` and ``backbone_hist`` are engine ResNet-family models: the reference builds them from the module dict
    ``contrastive._MODEL_TYPES`` (not from MODEL_REGISTRY), so that dict points at the engine classes while
    ``__init__`` runs, and is restored afterwards;
  * ``_update_history`` updates the key encoder IN PLACE with one ``sfb_momentum_update`` launch.  The reference
    assigns ``p.data = q * (1 - m) + p * m``, a new tensor per parameter per step, which would change every pointer a
    captured CUDA graph of the key encoder holds and force a re-capture on every step.  The result is bitwise the
    reference's (no FMA contraction, coefficients rounded to fp32 like ATen's scalars).

This is the only module of the package that imports the reference; it is loaded lazily through
``integration.ENGINE_CLASSES``.
"""
from __future__ import annotations

import contextlib

import slowfast.models.contrastive as _ref
import torch

from .. import ops
from .resnet import B200SlowFast
from .resnet_single import B200ResNet

# MODEL.ARCH -> engine backbone (the ResNet-family rows of contrastive._MODEL_TYPES)
ENGINE_BACKBONES = {"slowfast": B200SlowFast, "slow": B200ResNet, "c2d": B200ResNet, "i3d": B200ResNet,
                    "slow_c2d": B200ResNet}


@contextlib.contextmanager
def _engine_model_types():
    saved = dict(_ref._MODEL_TYPES)
    _ref._MODEL_TYPES.update(ENGINE_BACKBONES)
    try:
        yield
    finally:
        _ref._MODEL_TYPES.clear()
        _ref._MODEL_TYPES.update(saved)


class B200ContrastiveModel(_ref.ContrastiveModel):
    """``ContrastiveModel`` with engine backbones and an in-place key-encoder update (TYPE moco only)."""

    def __init__(self, cfg):
        kind = cfg.CONTRASTIVE.TYPE
        if kind != "moco":
            why = {"byol": "a predictor head and several gradient-carrying forwards per backward",
                   "simclr": "several gradient-carrying forwards per backward",
                   "swav": "several gradient-carrying forwards per backward and prototypes",
                   "mem": "the memory-bank model is not built", "self": "the memory-bank model is not built"}
            raise NotImplementedError(f"CONTRASTIVE.TYPE {kind!r} is not on the engine path "
                                      f"({why.get(kind, 'unknown type')}); only 'moco' is served")
        if not cfg.CONTRASTIVE.SEQUENTIAL:
            raise NotImplementedError("CONTRASTIVE.SEQUENTIAL False is not on the engine path: contrastive_forward would "
                                      "run every query clip's forward before one backward, and an engine model keeps "
                                      "one pending forward")
        if cfg.MODEL.ARCH not in ENGINE_BACKBONES:
            raise NotImplementedError(f"MODEL.ARCH {cfg.MODEL.ARCH!r}: ContrastiveModel on the engine serves the "
                                      f"ResNet-family backbones {sorted(ENGINE_BACKBONES)} only")
        with _engine_model_types():
            super().__init__(cfg)
        self._momentum_table = None
        self._momentum_ptrs = None

    def _pairs(self):
        q = dict(self.backbone.named_parameters())
        return [(q[name], k) for name, k in self.backbone_hist.named_parameters()]

    @torch.no_grad()
    def _update_history(self):
        pairs = self._pairs()
        if int(self.iter) == 0:
            for q, k in pairs:
                k.data.copy_(q.data)
        ptrs = tuple((q.data_ptr(), k.data_ptr()) for q, k in pairs)
        if ptrs != self._momentum_ptrs:  # first step, or the parameters moved (module.to())
            self._momentum_table = ops.momentum_table(pairs)
            self._momentum_ptrs = ptrs
        ops.momentum_update(self._momentum_table, self.mmt)
