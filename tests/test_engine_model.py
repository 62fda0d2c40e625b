"""CPU: the engine model contract is declared once, by ``engine.EngineModel``.

  * every engine network is an ``EngineModel``;
  * ``slowfast_b200/nets/*.py`` keep no copy of the contract (config switches, context, autograd entry, gradient
    bucket, BatchNorm registry), and ``engine.py`` reads it without ``getattr`` defaults or ``__dict__`` side channels;
  * the base applies cfg.B200.CUDA_GRAPH, and a reference config (no B200 section) keeps CUDA graphs on;
  * models without a detachable head write every parameter's gradient.
"""
import ast
import os

import pytest
import torch

ROOT = os.path.join(os.path.dirname(__file__), os.pardir, "slowfast_b200")
NETS = os.path.join(ROOT, "nets")
SMALL = dict(NUM_FRAMES=4, TRAIN_CROP_SIZE=64, TEST_CROP_SIZE=64)

# family: (light preset, overrides, reference yaml, reference overrides)
FAMILIES = {
    "slowfast": ("SLOWFAST_8x8_R50", dict(DATA=dict(SMALL, NUM_FRAMES=16)), "Kinetics/SLOWFAST_8x8_R50.yaml", []),
    "resnet": ("C2D_8x8_R50", dict(DATA=dict(SMALL, NUM_FRAMES=8)), "Kinetics/SLOW_8x8_R50.yaml", []),
    "x3d": ("X3D_M", dict(DATA=SMALL), "Kinetics/X3D_M.yaml", []),
    "mvit": ("MVITv2_S_16x4", dict(DATA=dict(SMALL, NUM_FRAMES=8)), "Kinetics/MVITv2_S_16x4.yaml", []),
    "mae": ("VIT_B_16x4_MAE_PT", dict(DATA=SMALL, MVIT={"DEPTH": 2}, MASK={"PRETRAIN_DEPTH": [1]}),
            "masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml", []),
    "maskfeat": ("MVITv2_S_16x4_MaskFeat_PT", dict(DATA=dict(SMALL, NUM_FRAMES=8)),
                 "masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml", ["DATA.NUM_FRAMES", 8]),
}
REF_SMALL = ["DATA.NUM_FRAMES", 4, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    refshim.install()
    return refshim


def _class_of(cfg):
    from slowfast_b200.integration import ENGINE_CLASSES, _resolve
    return _resolve(ENGINE_CLASSES[cfg.MODEL.MODEL_NAME])


def _light(family, **extra):
    from slowfast_b200.config import get_cfg
    preset, over, _, _ = FAMILIES[family]
    cfg = get_cfg(preset, **over)
    cfg.merge(extra)
    torch.manual_seed(0)
    return _class_of(cfg)(cfg)


def test_every_engine_class_is_an_engine_model():
    from slowfast_b200.engine import EngineModel
    from slowfast_b200.integration import ENGINE_CLASSES, _resolve
    from slowfast_b200.nets.mae import B200MAE
    classes = [_resolve(spec) for name, spec in ENGINE_CLASSES.items() if name != "ContrastiveModel"]
    for cls in classes + [B200MAE]:
        assert issubclass(cls, EngineModel), cls.__name__


def test_moco_backbones_are_engine_models():
    refshim = _refshim()
    from slowfast_b200.engine import EngineModel
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    cfg = refshim.load_cfg("contrastive_ssl/MoCo_SlowR50_8x8.yaml", ["CONTRASTIVE.QUEUE_LEN", 256,
                                                                     "CONTRASTIVE.LENGTH", 64])
    m = B200ContrastiveModel(cfg)
    assert isinstance(m.backbone, EngineModel) and isinstance(m.backbone_hist, EngineModel)


# the contract pieces the base class owns: nets/ must not restate them
CONTRACT_METHODS = {"grad_params", "allreduce_gradients", "_engine_forward", "_engine_backward", "_all_bns",
                    "_train_bns"}
CONTRACT_CFG_KEYS = {"CUDA_GRAPH", "RNG_SEED"}


def _contract_copies(tree):
    found = []
    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef)) and node.name in CONTRACT_METHODS:
            found.append((node.lineno, f"def {node.name}"))
        elif isinstance(node, ast.Attribute) and node.attr in CONTRACT_CFG_KEYS:
            found.append((node.lineno, f".{node.attr}"))
        elif isinstance(node, ast.Constant) and node.value in CONTRACT_CFG_KEYS:
            found.append((node.lineno, repr(node.value)))
        elif isinstance(node, ast.Call):
            f = node.func
            if isinstance(f, ast.Name) and f.id == "Ctx":
                found.append((node.lineno, "Ctx("))
            elif isinstance(f, ast.Attribute) and f.attr == "begin_backward":
                found.append((node.lineno, "begin_backward"))
            elif (isinstance(f, ast.Attribute) and f.attr == "apply" and isinstance(f.value, ast.Name)
                  and f.value.id == "ModelFunction"):
                found.append((node.lineno, "ModelFunction.apply"))
    return found


def test_nets_keep_no_copy_of_the_contract():
    files = sorted(f for f in os.listdir(NETS) if f.endswith(".py"))
    assert "mvit.py" in files and "resnet.py" in files
    bad = []
    for fn in files:
        bad += [(fn,) + hit for hit in _contract_copies(ast.parse(open(os.path.join(NETS, fn)).read(), fn))]
    assert not bad, bad


CONTRACT_ATTRS = {"cuda_graphs", "graph_warmup", "flat_grad_only", "_fwd_generation", "_graphs", "_graph_seen",
                  "_bn_list", "_bns"}


def test_engine_reads_the_contract_without_fallbacks():
    tree = ast.parse(open(os.path.join(ROOT, "engine.py")).read(), "engine.py")
    bad = []
    for node in ast.walk(tree):
        if isinstance(node, ast.Attribute) and node.attr == "__dict__":
            bad.append((node.lineno, "__dict__"))
        elif isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "getattr":
            owner = node.args[0]
            name = node.args[1].value if len(node.args) > 1 and isinstance(node.args[1], ast.Constant) else None
            if (isinstance(owner, ast.Name) and owner.id == "model") or name in CONTRACT_ATTRS:
                bad.append((node.lineno, f"getattr(..., {name!r})"))
    assert not bad, bad


@pytest.mark.parametrize("family", list(FAMILIES))
def test_cuda_graph_switch_comes_from_the_b200_section(family):
    assert _light(family, B200={"CUDA_GRAPH": False}).cuda_graphs is False
    assert _light(family, B200={"CUDA_GRAPH": True}).cuda_graphs is True


@pytest.mark.parametrize("family", list(FAMILIES))
def test_reference_config_without_b200_section_keeps_cuda_graphs(family):
    refshim = _refshim()
    _, _, yaml, over = FAMILIES[family]
    cfg = refshim.load_cfg(yaml, REF_SMALL + over)
    assert "B200" not in cfg
    torch.manual_seed(0)
    assert _class_of(cfg)(cfg).cuda_graphs is True


@pytest.mark.parametrize("family", ["x3d", "mae", "maskfeat"])
def test_grad_params_are_every_parameter(family):
    model = _light(family)
    assert model.grad_params() == list(model.parameters())
