"""Drop-in wiring behind ``slowfast.models.build_model`` (slowfast/models/build.py:22).

``build_model(cfg)`` looks ``cfg.MODEL.MODEL_NAME`` up in ``MODEL_REGISTRY`` (fvcore Registry, build.py:13) and calls
the class with ``cfg``; it then moves the module to the GPU and wraps it in DistributedDataParallel when
``NUM_GPUS > 1`` (build.py:55-80).  The engine plugs in at exactly that lookup, without editing the reference:

  * ``register()`` adds the engine classes under NEW names (``B200SlowFast`` ...): select them with the CLI override
    ``MODEL.MODEL_NAME B200SlowFast`` (the registry refuses duplicate names, so new names are the conservative route);
  * ``register(replace=True)`` additionally swaps the stock names (``SlowFast`` ...) to the engine classes, so that
    an unmodified yaml + ``tools/run_net.py`` trains on the engine.

Both require the reference package to be importable (``import slowfast``); nothing else in this package does.
See INTEGRATION.md for the launcher recipe and the module/state_dict contract.
"""
from __future__ import annotations

from typing import Dict

ENGINE_CLASSES: Dict[str, str] = {
    # reference name -> (module, class)
    "SlowFast": "slowfast_b200.nets.resnet:B200SlowFast",
    "ResNet": "slowfast_b200.nets.resnet_single:B200ResNet",
    "MViT": "slowfast_b200.nets.mvit:B200MViT",
    "X3D": "slowfast_b200.nets.x3d:B200X3D",
    "MaskMViT": "slowfast_b200.nets.maskfeat:B200MaskMViT",
    "ContrastiveModel": "slowfast_b200.nets.contrastive:B200ContrastiveModel",
}


def _resolve(spec: str):
    import importlib
    mod, cls = spec.split(":")
    return getattr(importlib.import_module(mod), cls)


def register(replace: bool = False):
    """Register the engine models in the reference's MODEL_REGISTRY. Returns the list of names now served by the
    engine."""
    from slowfast.models.build import MODEL_REGISTRY  # the reference's registry object
    from slowfast.models.batchnorm_helper import SubBatchNorm3d
    from . import subbn

    # BN.NORM_TYPE sub_batchnorm: build the reference's own container class (only its parameters and buffers are used,
    # never its forward), so that the unmodified misc.aggregate_sub_bn_stats - an isinstance check - finds it
    subbn.SUB_BN_CLASS = SubBatchNorm3d
    served = []
    for ref_name, spec in ENGINE_CLASSES.items():
        cls = _resolve(spec)
        if cls.__name__ not in MODEL_REGISTRY._obj_map:
            MODEL_REGISTRY._obj_map[cls.__name__] = cls
        served.append(cls.__name__)
        if replace:
            MODEL_REGISTRY._obj_map[ref_name] = cls
            served.append(ref_name)
    return served
