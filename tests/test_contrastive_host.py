"""MoCo (ContrastiveModel, CONTRASTIVE.TYPE moco) and the MLPHead projection on the engine: module tree, init,
checkpoints, registry and optimizer grouping against the unmodified reference (CPU only)."""
import pytest
import torch

MOCO = "contrastive_ssl/MoCo_SlowR50_8x8.yaml"
# a short queue and kNN memory: the model is the same, the buffers are small
SMALL = ["CONTRASTIVE.QUEUE_LEN", 256, "CONTRASTIVE.LENGTH", 64]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    refshim.install()
    return refshim


def _same_state(mine, ref):
    assert list(mine.keys()) == list(ref.keys())
    for k in ref:
        assert mine[k].shape == ref[k].shape and mine[k].dtype == ref[k].dtype, k
        assert torch.equal(mine[k], ref[k]), k


def test_moco_model_matches_reference_state_and_init():
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    from slowfast_b200.nets.resnet_single import B200ResNet
    cfg = refshim.load_cfg(MOCO, SMALL)
    ref = refshim.build_reference_model(cfg)
    torch.manual_seed(cfg.RNG_SEED)
    mine = B200ContrastiveModel(cfg)
    assert type(mine.backbone) is B200ResNet and type(mine.backbone_hist) is B200ResNet
    assert not any(p.requires_grad for p in mine.backbone_hist.parameters())
    sd = mine.state_dict()
    for k in ("queue_x", "ptr", "iter", "knn_mem.memory", "backbone.head.projection.projection.4.weight"):
        assert k in sd, k
    _same_state(sd, ref.state_dict())
    # the MLP is xavier-initialised (kaiming_uniform a=1 bound sqrt(3 / fan_in)), biases zero
    w = sd["backbone.head.projection.projection.0.weight"]
    assert w.abs().max() <= (3.0 / w.shape[1]) ** 0.5 and w.std() > 0.5 * (1.0 / w.shape[1]) ** 0.5
    assert not sd["backbone.head.projection.projection.2.bias"].any()
    # the wrapper leaves the reference's backbone table as it found it
    import slowfast.models.contrastive as rc
    from slowfast.models.video_model_builder import ResNet
    assert rc._MODEL_TYPES["slow"] is ResNet


@pytest.mark.parametrize("yaml", ["Kinetics/SLOW_8x8_R50.yaml", "Kinetics/SLOWFAST_8x8_R50.yaml"])
@pytest.mark.parametrize("layers", [1, 3])
def test_resnet_family_mlp_head_matches_reference(yaml, layers):
    refshim = _refshim()
    from slowfast_b200.nets.resnet import B200SlowFast
    from slowfast_b200.nets.resnet_single import B200ResNet
    cfg = refshim.load_cfg(yaml, ["CONTRASTIVE.NUM_MLP_LAYERS", layers, "MODEL.NUM_CLASSES", 128])
    ref = refshim.build_reference_model(cfg).state_dict()
    torch.manual_seed(cfg.RNG_SEED)
    mine = (B200SlowFast if "SLOWFAST" in yaml else B200ResNet)(cfg)
    _same_state(mine.state_dict(), ref)
    names = [k for k in ref if k.startswith("head.projection")]
    if layers == 1:
        assert names == ["head.projection.weight", "head.projection.bias"]
    else:
        assert names == [f"head.projection.projection.{i}.{t}" for i in (0, 2, 4) for t in ("weight", "bias")]
        assert [lin.out_features for lin in mine.head.linears()] == [2048, 2048, 128]


def test_moco_checkpoints_load_both_ways():
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    cfg = refshim.load_cfg(MOCO, SMALL)
    ref = refshim.build_reference_model(cfg)
    torch.manual_seed(123)
    mine = B200ContrastiveModel(cfg)
    mine.load_state_dict(ref.state_dict(), strict=True)
    _same_state(mine.state_dict(), ref.state_dict())
    torch.manual_seed(321)
    mine2 = B200ContrastiveModel(cfg)
    ref.load_state_dict(mine2.state_dict(), strict=True)
    _same_state(ref.state_dict(), mine2.state_dict())


def test_build_model_and_optimizer_groups():
    refshim = _refshim()
    import slowfast.models.optimizer as optim
    import slowfast_b200.integration as integ
    from slowfast.models import build_model
    from slowfast.models.build import MODEL_REGISTRY
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    cfg = refshim.load_cfg(MOCO, SMALL)
    ref = refshim.build_reference_model(cfg)
    saved = dict(MODEL_REGISTRY._obj_map)
    try:
        served = integ.register(replace=True)
        assert "B200ContrastiveModel" in served and "ContrastiveModel" in served
        model = build_model(cfg)
        assert type(model) is B200ContrastiveModel
        names = {id(p): n for n, p in model.named_parameters()}
        ref_names = {id(p): n for n, p in ref.named_parameters()}
        mine_groups = optim.construct_optimizer(model, cfg).param_groups
        ref_groups = optim.construct_optimizer(ref, cfg).param_groups
        assert len(mine_groups) == len(ref_groups)
        for g, rg in zip(mine_groups, ref_groups):
            assert [names[id(p)] for p in g["params"]] == [ref_names[id(p)] for p in rg["params"]]
            assert g["weight_decay"] == rg["weight_decay"]
        grouped = {names[id(p)] for g in mine_groups for p in g["params"]}
        assert not any(n.startswith("backbone_hist.") for n in grouped)
        assert any(n.startswith("backbone.head.projection.projection.") for n in grouped)
    finally:
        MODEL_REGISTRY._obj_map.clear()
        MODEL_REGISTRY._obj_map.update(saved)


@pytest.mark.parametrize("kind", ["byol", "simclr", "swav", "mem", "self"])
def test_other_contrastive_types_are_rejected(kind):
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    with pytest.raises(NotImplementedError, match=f"CONTRASTIVE.TYPE '{kind}'"):
        B200ContrastiveModel(refshim.load_cfg(MOCO, SMALL + ["CONTRASTIVE.TYPE", kind]))


def test_moco_without_sequential_is_rejected():
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    with pytest.raises(NotImplementedError, match="CONTRASTIVE.SEQUENTIAL False"):
        B200ContrastiveModel(refshim.load_cfg(MOCO, SMALL + ["CONTRASTIVE.SEQUENTIAL", False]))


def test_contrastive_backbone_heads_pool_globally():
    """Inside ContrastiveModel the reference's ResNet heads use an adaptive 1x1x1 pool (video_model_builder.py:401,630),
    so a test crop larger than the train crop is one global mean, not the windowed train-pool path."""
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    m = B200ContrastiveModel(refshim.load_cfg(MOCO, SMALL))
    assert m.backbone.head.pool_size == [None] and m.backbone_hist.head.pool_size == [None]
    from slowfast_b200.nets.resnet_single import B200ResNet
    assert B200ResNet(refshim.load_cfg("Kinetics/SLOW_8x8_R50.yaml")).head.pool_size == [(8, 7, 7)]


@pytest.mark.parametrize("arch", ["x3d", "mvit"])
def test_non_resnet_backbones_are_rejected(arch):
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    cfg = refshim.load_cfg(MOCO, SMALL)
    cfg.MODEL.ARCH = arch
    with pytest.raises(NotImplementedError, match=f"MODEL.ARCH '{arch}'"):
        B200ContrastiveModel(cfg)


@pytest.mark.parametrize("override,name", [(["CONTRASTIVE.BN_MLP", True], "BN_MLP"),
                                           (["CONTRASTIVE.BN_SYNC_MLP", True], "BN_SYNC_MLP"),
                                           (["CONTRASTIVE.PREDICTOR_DEPTHS", [2]], "PREDICTOR_DEPTHS")])
def test_mlp_head_variants_are_rejected(override, name):
    refshim = _refshim()
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    from slowfast_b200.nets.resnet_single import B200ResNet
    with pytest.raises(NotImplementedError, match=f"CONTRASTIVE.{name}"):
        B200ContrastiveModel(refshim.load_cfg(MOCO, SMALL + override))
    with pytest.raises(NotImplementedError, match=f"CONTRASTIVE.{name}"):
        B200ResNet(refshim.load_cfg("Kinetics/SLOW_8x8_R50.yaml", ["CONTRASTIVE.NUM_MLP_LAYERS", 3] + override))
