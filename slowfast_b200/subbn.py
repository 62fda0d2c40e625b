"""Sub-batch BatchNorm (``BN.NORM_TYPE sub_batchnorm``): the parameter container and the norm factory.

Multigrid training's long cycle (slowfast/utils/multigrid.py:58-107) grows the per-GPU batch while it shrinks the clips,
and keeps the BatchNorm statistics at ``MULTIGRID.BN_BASE_SIZE`` clips by normalising S = batch / BN_BASE_SIZE
sub-batches separately.  The reference's module (batchnorm_helper.py:40-112) holds:

  * ``weight`` / ``bias``  - ONE affine, shared by every split (its own Parameters: not a ``_NormBase``, so the
                             optimizer puts them in the weight-decay group and ``init_weights`` never touches them);
  * ``bn``                 - BatchNorm3d(C, affine=False): the statistics eval uses;
  * ``split_bn``           - BatchNorm3d(S*C, affine=False): training normalises ``x.view(n // S, C*S, t, h, w)``, so
                             clip k is in split k % S and its channel c is split_bn channel s*C + c.

``aggregate_stats()`` turns the split statistics into ``bn``'s before eval.  The engine executes all of it with its
own kernels (engine.ConvBN); these modules only hold parameters and buffers under the reference's state_dict names.
``integration.register()`` makes the engine build the reference's own class instead, so that the reference's
``misc.aggregate_sub_bn_stats`` (an isinstance check) finds the engine's containers.
"""
from __future__ import annotations

from functools import partial
from typing import Callable, Tuple

import torch
import torch.nn as nn


class SubBatchNorm3d(nn.Module):
    """Parameter container with the reference SubBatchNorm3d's constructor, state_dict keys and order."""

    def __init__(self, num_splits: int, num_features: int, eps: float = 1e-5, momentum: float = 0.1,
                 affine: bool = True, **bn_kwargs):
        super().__init__()
        self.num_splits = int(num_splits)
        self.affine = bool(affine)
        if self.affine:
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
        self.bn = nn.BatchNorm3d(num_features, eps=eps, momentum=momentum, affine=False, **bn_kwargs)
        self.split_bn = nn.BatchNorm3d(num_features * self.num_splits, eps=eps, momentum=momentum, affine=False,
                                       **bn_kwargs)

    def aggregate_stats(self) -> None:
        """``bn``'s running statistics from the splits' (call before eval).  The tensors are REPLACED (``.data``), as
        in the reference, so a captured eval program sees new pointers and is captured again."""
        if self.split_bn.track_running_stats:
            self.bn.running_mean.data, self.bn.running_var.data = aggregate_split_stats(
                self.split_bn.running_mean, self.split_bn.running_var, self.num_splits)

    def forward(self, *a, **k):  # pragma: no cover - containers are never called
        raise RuntimeError("engine containers hold parameters only; call the top-level model")


def aggregate_split_stats(means: torch.Tensor, variances: torch.Tensor, splits: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Statistics of the union of S equally sized splits from the splits' [S*C] statistics: the mean of the means, and
    the mean of the variances plus the (population) variance of the means - the reference's arithmetic, op for op."""
    m = means.view(splits, -1)
    mean = m.sum(0) / splits
    var = variances.view(splits, -1).sum(0) / splits + ((m - mean) ** 2).sum(0) / splits
    return mean.detach(), var.detach()


# The container class the norm factory builds; integration.register() swaps in the reference's own class.
SUB_BN_CLASS = SubBatchNorm3d


def is_sub_bn(m: nn.Module) -> bool:
    return hasattr(m, "split_bn") and hasattr(m, "num_splits")


def norm_factory(cfg) -> Callable[..., nn.Module]:
    """The BN module of every ResNet-family BN site, chosen from ``cfg.BN`` as the reference's ``get_norm`` does
    (batchnorm_helper.py:16); called as ``norm(num_features=..., eps=..., momentum=...)``."""
    kind = cfg.BN.NORM_TYPE
    if kind == "batchnorm":
        return nn.BatchNorm3d
    if kind == "sub_batchnorm":
        splits = int(cfg.BN.NUM_SPLITS)
        if splits < 1:
            raise ValueError(f"BN.NUM_SPLITS must be >= 1 for sub_batchnorm, got {splits}")
        return partial(SUB_BN_CLASS, num_splits=splits)
    if kind == "sync_batchnorm":
        raise NotImplementedError(
            "BN.NORM_TYPE sync_batchnorm (BatchNorm statistics shared across GPUs, which multigrid selects when the "
            "per-GPU batch is below MULTIGRID.BN_BASE_SIZE) is not supported by the engine; use batchnorm or "
            "sub_batchnorm")
    raise NotImplementedError(f"BN.NORM_TYPE {kind!r} is not supported by the engine (batchnorm, sub_batchnorm)")


def num_splits_of(cfg) -> int:
    """Splits of the training batch: BN.NUM_SPLITS under sub_batchnorm, else 1."""
    return int(cfg.BN.NUM_SPLITS) if cfg.BN.NORM_TYPE == "sub_batchnorm" else 1


def aggregate_sub_bn_stats(model: nn.Module) -> int:
    """Call ``aggregate_stats()`` on every sub-batch BN of ``model`` (for training loops other than the reference's,
    which calls misc.aggregate_sub_bn_stats after precise-BN).  Returns how many were aggregated."""
    count = 0
    for m in model.modules():
        if is_sub_bn(m):
            m.aggregate_stats()
            count += 1
    return count
