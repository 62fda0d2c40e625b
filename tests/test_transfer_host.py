"""CPU: the transfer switches on the engine - MODEL.DETACH_FINAL_FC (linear evaluation), MODEL.HEAD_ACT sigmoid
(multi-label heads) and MODEL.FROZEN_BN (BatchNorm modules in eval inside a training model): module trees and init
against the unmodified reference, the rejected combinations, and the program key that keeps the BN modes apart."""
import pytest
import torch

LINEAR = "contrastive_ssl/linear_k400_Slow_8x8_R50_syn0.yaml"
SMALL = ["DATA.NUM_FRAMES", 4, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64]
HEAD_YAMLS = ["Kinetics/SLOWFAST_8x8_R50.yaml", "Kinetics/X3D_M.yaml", "Kinetics/MVITv2_S_16x4.yaml"]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    refshim.install()
    return refshim


def _engine_class(cfg):
    name = cfg.MODEL.MODEL_NAME
    if name == "SlowFast":
        from slowfast_b200.nets.resnet import B200SlowFast as M
    elif name == "MViT":
        from slowfast_b200.nets.mvit import B200MViT as M
    elif name == "X3D":
        from slowfast_b200.nets.x3d import B200X3D as M
    else:
        from slowfast_b200.nets.resnet_single import B200ResNet as M
    return M


def _engine(cfg):
    torch.manual_seed(cfg.RNG_SEED)
    return _engine_class(cfg)(cfg)


def test_linear_probe_recipe_builds_a_detaching_model_equal_to_the_reference(monkeypatch):
    """``slowfast.models.build_model`` with the engine registered routes the linear-probe recipe to the engine."""
    refshim = _refshim()
    import driver_harness as H
    from slowfast_b200 import subbn
    from slowfast_b200.nets.resnet_single import B200ResNet
    monkeypatch.setattr(subbn, "SUB_BN_CLASS", subbn.SUB_BN_CLASS)  # register() points it at the reference's class
    cfg = refshim.load_cfg(LINEAR)
    assert cfg.MODEL.DETACH_FINAL_FC
    ref = refshim.build_reference_model(cfg)
    try:
        H.use_engine(True)
        from slowfast.models import build_model
        torch.manual_seed(cfg.RNG_SEED)
        mine = build_model(cfg)
    finally:
        H.use_engine(False)
    assert type(mine) is B200ResNet and mine.head.detach_final_fc and ref.head.detach_final_fc
    sd, want = mine.state_dict(), ref.state_dict()
    assert list(sd) == list(want)
    for k in want:
        assert torch.equal(sd[k], want[k]), k
    # the backward writes the projection only: that is the flat gradient bucket, in parameter order
    assert mine.grad_params() == [mine.head.projection.weight, mine.head.projection.bias]


def test_detach_on_the_mvit_head_and_not_on_default_configs():
    refshim = _refshim()
    cfg = refshim.load_cfg("Kinetics/MVITv2_S_16x4.yaml", SMALL + ["MODEL.DETACH_FINAL_FC", True])
    mine = _engine(cfg)
    assert mine.head.detach_final_fc
    assert mine.grad_params() == [mine.head.projection.weight, mine.head.projection.bias]
    plain = _engine(refshim.load_cfg("Kinetics/MVITv2_S_16x4.yaml", SMALL))
    assert not plain.head.detach_final_fc and plain.grad_params() == list(plain.parameters())


@pytest.mark.parametrize("yaml", HEAD_YAMLS)
def test_sigmoid_head_builds(yaml):
    refshim = _refshim()
    cfg = refshim.load_cfg(yaml, SMALL + ["MODEL.HEAD_ACT", "sigmoid"])
    mine = _engine(cfg)
    assert mine.head.act_func == "sigmoid"
    ref = refshim.build_reference_model(cfg)
    assert list(mine.state_dict()) == list(ref.state_dict())


@pytest.mark.parametrize("yaml", HEAD_YAMLS)
def test_unknown_head_activation_is_rejected_by_name(yaml):
    refshim = _refshim()
    cfg = refshim.load_cfg(yaml, SMALL + ["MODEL.HEAD_ACT", "tanh"])
    with pytest.raises(NotImplementedError, match="'tanh'"):
        _engine(cfg)


def test_frozen_bn_with_sub_batchnorm_is_rejected_at_construction():
    refshim = _refshim()
    cfg = refshim.load_cfg("Kinetics/SLOW_8x8_R50.yaml", ["BN.NORM_TYPE", "sub_batchnorm", "BN.NUM_SPLITS", 2,
                                                           "MODEL.FROZEN_BN", True])
    with pytest.raises(NotImplementedError, match="MODEL.FROZEN_BN"):
        _engine(cfg)


def test_program_key_tells_bn_modes_apart():
    refshim = _refshim()
    from slowfast_b200.engine import program_key
    cfg = refshim.load_cfg("Kinetics/SLOW_8x8_R50.yaml", SMALL)
    model = _engine(cfg).train()
    x = [torch.empty(2, 3, 4, 64, 64)]
    key_train = program_key(model, True, x)
    for m in model.s1.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.eval()
    key_part = program_key(model, True, x)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.eval()
    key_frozen = program_key(model, True, x)
    assert len({key_train, key_part, key_frozen}) == 3
    # an eval model's BNs all use running statistics whatever their module modes: one key
    model.eval()
    key_eval = program_key(model, False, x)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.train()
    model.training = False
    assert program_key(model, False, x) == key_eval
