"""CPU: sub-batch BatchNorm (BN.NORM_TYPE sub_batchnorm, multigrid's long cycle) on the ResNet family - module tree and
init parity with the reference, its aggregation arithmetic, the optimizer grouping, the checkpoint helpers' key renaming
across split counts, and the configurations the engine rejects."""
import copy

import pytest
import torch

from slowfast_b200 import subbn

YAMLS = ["Kinetics/SLOWFAST_8x8_R50.yaml", "Kinetics/SLOW_8x8_R50.yaml", "Kinetics/I3D_8x8_R50.yaml",
         "Kinetics/SLOWFAST_NLN_8x8_R50.yaml"]


def _need_reference():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    return refshim


def _engine_class(cfg):
    if cfg.MODEL.MODEL_NAME == "SlowFast":
        from slowfast_b200.nets.resnet import B200SlowFast
        return B200SlowFast
    from slowfast_b200.nets.resnet_single import B200ResNet
    return B200ResNet


def _cfg(refshim, yaml, splits, extra=()):
    norm = ["BN.NORM_TYPE", "sub_batchnorm", "BN.NUM_SPLITS", splits] if splits else []
    return refshim.load_cfg(yaml, norm + ["RESNET.ZERO_INIT_FINAL_BN", True] + list(extra))


def _engine(cfg):
    torch.manual_seed(cfg.RNG_SEED)
    return _engine_class(cfg)(cfg)


def _bn_sites(model):
    return [name for name, m in model.named_modules() if subbn.is_sub_bn(m)]


@pytest.mark.parametrize("splits", [2, 4])
@pytest.mark.parametrize("yaml", YAMLS)
def test_subbn_state_dict_and_init_match_reference(yaml, splits):
    """Same state_dict keys / order / shapes as the reference under sub_batchnorm, and bit-identical init under the same
    seed: ZERO_INIT_FINAL_BN has no effect on a sub-batch BN (its container is no nn.BatchNorm3d and the inner BNs have no
    weight), so every c_bn.weight stays 1."""
    refshim = _need_reference()
    cfg = _cfg(refshim, yaml, splits)
    ref = refshim.build_reference_model(cfg).state_dict()
    mine = _engine(cfg).state_dict()
    assert [(k, tuple(v.shape)) for k, v in mine.items()] == [(k, tuple(v.shape)) for k, v in ref.items()]
    assert all(torch.equal(mine[k], ref[k]) for k in ref)
    c_bn = [k for k in mine if k.endswith("c_bn.weight")]
    assert c_bn and all(torch.equal(mine[k], torch.ones_like(mine[k])) for k in c_bn)
    assert any(k.endswith("c_bn.split_bn.running_mean") for k in mine)


def test_every_bn_site_is_a_sub_bn():
    """Stems, FuseFastToSlow, a/b/c_bn, branch1_bn and the Non-local bn: no plain BN is left at a BN site."""
    refshim = _need_reference()
    cfg = _cfg(refshim, "Kinetics/SLOWFAST_NLN_8x8_R50.yaml", 2)
    model = _engine(cfg)
    sites = _bn_sites(model)
    for suffix in ("pathway0_stem.bn", "pathway1_stem.bn", "s1_fuse.bn", "s2_fuse.bn", "branch2.a_bn", "branch2.b_bn",
                   "branch2.c_bn", "branch1_bn", "pathway0_nonlocal1.bn"):
        assert any(s.endswith(suffix) for s in sites), suffix
    inner = {id(m.bn) for m in model.modules() if subbn.is_sub_bn(m)} | \
        {id(m.split_bn) for m in model.modules() if subbn.is_sub_bn(m)}
    assert all(id(m) in inner for m in model._all_bns())
    assert len(model._all_bns()) == 2 * len(sites)
    assert len(model._train_bns()) == len(sites)
    assert all(getattr(m, "transform_final_bn", False) for n, m in model.named_modules() if n.endswith("c_bn"))


@pytest.mark.parametrize("splits", [2, 3, 4, 8])
def test_aggregate_stats_equals_reference(splits):
    refshim = _need_reference()
    refshim.install()
    from slowfast.models.batchnorm_helper import SubBatchNorm3d as RefSubBN
    g = torch.Generator().manual_seed(splits)
    c = 24
    mine = subbn.SubBatchNorm3d(num_splits=splits, num_features=c, eps=1e-5, momentum=0.1)
    ref = RefSubBN(num_splits=splits, num_features=c, eps=1e-5, momentum=0.1)
    rm, rv = torch.randn(splits * c, generator=g), torch.rand(splits * c, generator=g) * 3
    for m in (mine, ref):
        m.split_bn.running_mean.copy_(rm)
        m.split_bn.running_var.copy_(rv)
        m.aggregate_stats()
    assert torch.equal(mine.bn.running_mean, ref.bn.running_mean)
    assert torch.equal(mine.bn.running_var, ref.bn.running_var)
    assert [k for k in mine.state_dict()] == [k for k in ref.state_dict()]


def test_aggregate_replaces_the_tensors():
    """aggregate_stats assigns through .data: a captured eval program must see new pointers."""
    m = subbn.SubBatchNorm3d(num_splits=2, num_features=8)
    before = m.bn.running_mean.data_ptr()
    m.aggregate_stats()
    assert m.bn.running_mean.data_ptr() != before


def test_reference_aggregate_finds_engine_modules_after_register(monkeypatch):
    """After integration.register() the engine builds the reference's own container class, so the unmodified
    misc.aggregate_sub_bn_stats (an isinstance check) counts every BN site; the engine's own helper agrees."""
    refshim = _need_reference()
    refshim.install()
    monkeypatch.setattr(subbn, "SUB_BN_CLASS", subbn.SUB_BN_CLASS)
    from slowfast.models.batchnorm_helper import SubBatchNorm3d as RefSubBN
    from slowfast.utils import misc

    from slowfast_b200 import integration
    integration.register()
    assert subbn.SUB_BN_CLASS is RefSubBN
    cfg = _cfg(refshim, "Kinetics/SLOWFAST_NLN_8x8_R50.yaml", 2)
    model = _engine(cfg)
    sites = _bn_sites(model)
    assert all(isinstance(m, RefSubBN) for m in model.modules() if subbn.is_sub_bn(m))
    assert misc.aggregate_sub_bn_stats(model) == len(sites) > 100
    assert subbn.aggregate_sub_bn_stats(model) == len(sites)
    ref = refshim.build_reference_model(cfg)
    assert misc.aggregate_sub_bn_stats(ref) == len(sites)


@pytest.mark.parametrize("yaml", ["Kinetics/SLOWFAST_8x8_R50.yaml", "Kinetics/I3D_8x8_R50.yaml"])
def test_optimizer_groups_match_reference(yaml):
    """construct_optimizer groups BN parameters by _NormBase: the container's weight / bias are not, so they land in the
    SOLVER.WEIGHT_DECAY group - for the reference model, the engine model, and the engine's own grouping."""
    refshim = _need_reference()
    cfg = _cfg(refshim, yaml, 4, ["BN.WEIGHT_DECAY", 0.5, "SOLVER.WEIGHT_DECAY", 1e-4])
    from slowfast.models.optimizer import construct_optimizer

    from slowfast_b200.optim import param_groups_from_cfg

    def named_groups(model, groups):
        names = {id(p): n for n, p in model.named_parameters()}
        return sorted((float(g["weight_decay"]), sorted(names[id(p)] for p in g["params"])) for g in groups)

    ref = refshim.build_reference_model(cfg)
    mine = _engine(cfg)
    want = named_groups(ref, construct_optimizer(ref, cfg).param_groups)
    assert named_groups(mine, construct_optimizer(mine, cfg).param_groups) == want
    assert named_groups(mine, param_groups_from_cfg(mine, cfg)) == want
    decayed = dict((wd, names) for wd, names in want)[1e-4]
    assert any(n.endswith("c_bn.weight") for n in decayed)


def test_checkpoint_round_trip_across_split_counts():
    """A long-cycle phase change: the S=4 model's checkpoint (sub_to_normal_bn on save) loads into an S=2 model and a
    plain-BN model through normal_to_sub_bn, strict."""
    refshim = _need_reference()
    refshim.install()
    from slowfast.utils.checkpoint import normal_to_sub_bn, sub_to_normal_bn
    yaml = "Kinetics/SLOWFAST_8x8_R50.yaml"
    src = _engine(_cfg(refshim, yaml, 4))
    g = torch.Generator().manual_seed(0)
    for m in src.modules():
        if subbn.is_sub_bn(m):
            m.split_bn.running_mean.copy_(torch.randn(m.split_bn.running_mean.shape, generator=g))
            m.split_bn.running_var.copy_(torch.rand(m.split_bn.running_var.shape, generator=g) + 0.5)
            m.weight.data.copy_(torch.randn(m.weight.shape, generator=g))
    subbn.aggregate_sub_bn_stats(src)
    saved = sub_to_normal_bn(src.state_dict())
    assert not any(".split_bn." in k or "bn.bn." in k for k in saved)
    for splits in (2, None):
        dst = _engine(_cfg(refshim, yaml, splits))
        dst.load_state_dict(normal_to_sub_bn(copy.deepcopy(saved), dst.state_dict()), strict=True)
        s_src = dict(src.named_modules())
        for name, m in dst.named_modules():
            if name.endswith("c_bn"):
                want = s_src[name]
                assert torch.equal(m.weight, want.weight)
                have_mean = m.split_bn.running_mean[:m.weight.numel()] if splits else m.running_mean
                assert torch.equal(have_mean, want.bn.running_mean)


def test_sync_batchnorm_is_rejected():
    refshim = _need_reference()
    cfg = refshim.load_cfg("Kinetics/SLOWFAST_8x8_R50.yaml", ["BN.NORM_TYPE", "sync_batchnorm"])
    with pytest.raises(NotImplementedError, match="sync_batchnorm"):
        _engine(cfg)


def test_sub_batchnorm_on_x3d_is_rejected():
    """X3D's channelwise convolutions apply the producer's BN inside their ring: no per-split coefficients there.
    (MViT has no BatchNorm, so BN.NORM_TYPE does not affect it, as in the reference.)"""
    refshim = _need_reference()
    cfg = refshim.load_cfg("Kinetics/X3D_M.yaml", ["BN.NORM_TYPE", "sub_batchnorm", "BN.NUM_SPLITS", 2])
    from slowfast_b200.nets.x3d import B200X3D
    with pytest.raises(AssertionError, match="batchnorm"):
        B200X3D(cfg)


def test_batch_not_divisible_by_splits_is_rejected():
    refshim = _need_reference()
    cfg = _cfg(refshim, "Kinetics/SLOW_8x8_R50.yaml", 2, ["DATA.TRAIN_CROP_SIZE", 64, "DATA.NUM_FRAMES", 4])
    model = _engine(cfg).train()
    with pytest.raises(ValueError, match=r"BN.NUM_SPLITS 2 .*batch size 3"):
        model([torch.zeros(3, 3, 4, 64, 64)])
