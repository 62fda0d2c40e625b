"""CPU: Non-local recipes (C2D / I3D / Slow / SlowFast NLN) - module tree and init parity with the reference, the
Non-local restatement against the reference's golden vectors, and the configurations the reference rejects."""
import glob
import os

import pytest
import torch

import nonlocal_oracle as NO

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
NLN_YAMLS = ["Kinetics/C2D_NLN_8x8_R50.yaml", "Kinetics/C2D_NLN_8x8_R50_IN1K.yaml", "Kinetics/I3D_NLN_8x8_R50.yaml",
             "Kinetics/I3D_NLN_8x8_R50_IN1K.yaml", "Kinetics/I3D_NLN_8x8_R101.yaml", "Kinetics/SLOW_NLN_4x16_R50.yaml",
             "Kinetics/SLOW_NLN_8x8_R50.yaml", "Kinetics/SLOWFAST_NLN_4x16_R50.yaml",
             "Kinetics/SLOWFAST_NLN_8x8_R50.yaml"]
SMALL = ["i3d_nln_r50_small", "c2d_nln_r50_small", "slow_nln_r50_small", "slowfast_nln_r50_small", "i3d_nln_group2_small"]
ALL = SMALL + ["i3d_nln_r50_224", "slowfast_nln_r50_224"]


def _engine_class(cfg):
    if cfg.MODEL.MODEL_NAME == "SlowFast":
        from slowfast_b200.nets.resnet import B200SlowFast
        return B200SlowFast
    from slowfast_b200.nets.resnet_single import B200ResNet
    return B200ResNet


def _template(gold):
    return {k: torch.empty(shape, dtype=torch.long if k.endswith("num_batches_tracked") else torch.float32)
            for k, shape in gold["keys"]}


@pytest.mark.parametrize("yaml", NLN_YAMLS)
def test_nln_state_dict_and_init_match_reference(yaml):
    """The engine class built from the reference's own CfgNode: same state_dict names / order / shapes, and the same
    values under the same seed (every Non-local conv msra-filled with a zero bias, the block's BN weight zeroed)."""
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    rcfg = refshim.load_cfg(yaml)
    torch.manual_seed(rcfg.RNG_SEED)
    ref = refshim.build_reference_model(rcfg).state_dict()
    torch.manual_seed(rcfg.RNG_SEED)
    mine = _engine_class(rcfg)(rcfg).state_dict()
    assert [(k, tuple(v.shape)) for k, v in mine.items()] == [(k, tuple(v.shape)) for k, v in ref.items()]
    assert all(torch.equal(mine[k], ref[k]) for k in ref)
    assert any(".pathway0_nonlocal" in k for k in ref)


def test_every_shipped_nln_yaml_is_covered():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    root = os.path.join(refshim.REFERENCE_ROOT, "configs")
    shipped = sorted(os.path.relpath(p, root) for p in glob.glob(os.path.join(root, "Kinetics", "*NLN*.yaml")))
    assert shipped == sorted(NLN_YAMLS)


@pytest.mark.parametrize("name", ALL)
def test_nln_state_dict_keys_match_golden(name):
    gold = torch.load(os.path.join(GOLDEN, name + ".pt"))
    cfg = NO.engine_cfg(gold)
    m = _engine_class(cfg)(cfg)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in gold["keys"]]
    assert gold["oracle_check"]["logits"] < 1e-5 and gold["oracle_check"]["grads"] < 1e-4 and \
        gold["oracle_check"]["running"] < 1e-5


@pytest.mark.parametrize("name", ALL)
def test_nonlocal_oracle_reproduces_reference_golden(name):
    from oracle import torch_oracle as TO
    gold = torch.load(os.path.join(GOLDEN, name + ".pt"))
    cfg = NO.engine_cfg(gold)
    state = TO.fixture_state(_template(gold), gold["st_seed"])
    inputs = TO.synthetic_inputs(cfg, gold["batch"], gold["in_seed"])
    dlogits = torch.randn(gold["logits"].shape, generator=torch.Generator().manual_seed(gold["in_seed"] + 1000))
    logits, grads = NO.forward_backward(cfg, state, inputs, dlogits)
    assert ((logits - gold["logits"]).abs().max() / gold["logits"].abs().max()).item() < 1e-5
    floor = gold["grad_norm_floor"]   # (conv_out.bias: an exactly-zero gradient, rounding noise on every host)
    for k, dg in gold["grads"].items():
        g = grads[k].double().flatten()
        assert abs(g.norm().item() - dg["norm"]) / max(dg["norm"], floor, 1e-20) < 1e-3, k
        assert torch.allclose(g[:4], torch.tensor(dg["head"], dtype=torch.float64), rtol=2e-2,
                              atol=1e-3 * max(dg["norm"], 1e-20) + 1e-2 * floor), k


def test_unknown_instantiation_is_rejected_at_construction():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.resnet import B200SlowFast
    from slowfast_b200.nets.resnet_single import B200ResNet
    with pytest.raises(NotImplementedError):
        B200ResNet(get_cfg("I3D_NLN_8x8_R50", NONLOCAL={"INSTANTIATION": "gaussian"}))
    with pytest.raises(NotImplementedError):
        B200SlowFast(get_cfg("SLOWFAST_NLN_8x8_R50", NONLOCAL={"INSTANTIATION": "embedded_gaussian"}))


def test_group_that_does_not_divide_the_frames_is_rejected():
    from slowfast_b200.engine import Act, Ctx
    from slowfast_b200.nets.resnet import NonlocalModule
    ctx = Ctx(3)
    ctx.device = torch.device("cpu")
    m = NonlocalModule("nl", 64, 32, [1, 2, 2], "softmax", 3, ctx)
    x = Act(ctx.storage(("x",), 1, 4, 8, 8, 64))
    with pytest.raises(ValueError, match="GROUP 3 does not divide the 4 frames"):
        m.run_forward(x, Act(ctx.storage(("o",), 1, 4, 8, 8, 64)))


def test_nln_presets_mirror_the_yamls():
    from slowfast_b200.config import get_cfg
    for preset, inst in (("C2D_NLN_8x8_R50", "softmax"), ("I3D_NLN_8x8_R50", "softmax"),
                         ("SLOW_NLN_8x8_R50", "dot_product"), ("SLOWFAST_NLN_8x8_R50", "dot_product")):
        cfg = get_cfg(preset)
        assert cfg.NONLOCAL.INSTANTIATION == inst
        assert cfg.NONLOCAL.LOCATION[1][0] == [1, 3] and cfg.NONLOCAL.LOCATION[2][0] == [1, 3, 5]
        assert cfg.NONLOCAL.POOL[1][0] == [1, 2, 2]
    assert get_cfg("SLOWFAST_NLN_8x8_R50").SLOWFAST.FUSION_KERNEL_SZ == 5
