"""CPU: the mean-pooled and absolute-position MViT recipes (MaskFeat fine-tuning, MViTv1-B, ViT-B/L/H) - module tree
and init parity with the reference, presets, optimizer grouping, the MaskFeat pre-train -> fine-tune checkpoint path, and
the configurations the engine rejects at construction."""
import pytest
import torch

FT_YAMLS = ["Kinetics/MVIT_B_16x4_CONV.yaml", "masked_ssl/k400_VIT_B_16x4_FT.yaml", "masked_ssl/k400_VIT_L_16x4_FT.yaml",
            "masked_ssl/k400_VIT_H_16x4_FT.yaml", "masked_ssl/k400_MVITv2_S_16x4_FT.yaml",
            "masked_ssl/k400_MVITv2_L_16x4_FT.yaml"]
PRESETS = {"MVIT_B_16x4_CONV": "Kinetics/MVIT_B_16x4_CONV.yaml", "VIT_B_16x4_FT": "masked_ssl/k400_VIT_B_16x4_FT.yaml",
           "MVITv2_S_16x4_FT": "masked_ssl/k400_MVITv2_S_16x4_FT.yaml"}
SMALL = ["DATA.NUM_FRAMES", 8, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    return refshim


@pytest.mark.parametrize("yaml", FT_YAMLS)
def test_state_dict_and_init_match_reference(yaml):
    """The engine class from the reference's own CfgNode: same state_dict names / order / shapes and the same values
    under the same seed (pos_embed_{spatial,temporal,class} drawn after the head and before cls_token)."""
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(yaml)
    with torch.no_grad():
        ref = refshim.build_reference_model(rcfg).state_dict()
        torch.manual_seed(rcfg.RNG_SEED)
        mine = B200MViT(rcfg).state_dict()
    assert [(k, tuple(v.shape)) for k, v in mine.items()] == [(k, tuple(v.shape)) for k, v in ref.items()]
    assert all(torch.equal(mine[k], ref[k]) for k in ref)
    assert ("pos_embed_spatial" in ref) == rcfg.MVIT.USE_ABS_POS


@pytest.mark.parametrize("preset", sorted(PRESETS))
def test_presets_mirror_the_yamls(preset):
    from slowfast_b200.config import get_cfg
    refshim = _refshim()
    rcfg = refshim.load_cfg(PRESETS[preset])
    mine = get_cfg(preset)
    for key, v in mine.MVIT.items():
        if key != "REV":
            want = rcfg.MVIT[key]
            assert (list(v) if isinstance(v, (list, tuple)) else v) == \
                (list(want) if isinstance(want, (list, tuple)) else want), key
    for key in ("NUM_FRAMES", "TRAIN_CROP_SIZE", "TEST_CROP_SIZE", "INPUT_CHANNEL_NUM"):
        assert mine.DATA[key] == rcfg.DATA[key], key
    for key in ("NUM_CLASSES", "ARCH", "MODEL_NAME", "DROPOUT_RATE"):
        assert mine.MODEL[key] == rcfg.MODEL[key], key


@pytest.mark.parametrize("yaml,extra", [
    ("masked_ssl/k400_VIT_B_16x4_FT.yaml", []),                                  # LAYER_DECAY 0.65
    ("masked_ssl/k400_MVITv2_S_16x4_FT.yaml", []),                               # LAYER_DECAY 0.75
    ("Kinetics/MVIT_B_16x4_CONV.yaml", ["MVIT.ZERO_DECAY_POS_CLS", True]),       # plain groups, zero-decay positions
    ("masked_ssl/k400_VIT_B_16x4_FT.yaml", ["MVIT.ZERO_DECAY_POS_CLS", True]),
])
def test_reference_optimizer_groups_match(yaml, extra):
    """slowfast.models.optimizer.construct_optimizer builds the same groups (names, weight decay, layer decay) for the
    engine model as for the reference model: pos_embed_* land in layer 0 and, with ZERO_DECAY_POS_CLS, in a zero group."""
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(yaml, SMALL + ["DATA.NUM_FRAMES", 4] + list(extra))
    import slowfast.models.optimizer as optim
    ref = refshim.build_reference_model(rcfg)
    mine = B200MViT(rcfg)
    assert mine.no_weight_decay() == ref.no_weight_decay()

    def groups(model):
        names = {id(p): n for n, p in model.named_parameters()}
        opt = optim.construct_optimizer(model, rcfg)
        return [(g["weight_decay"], g.get("layer_decay"), [names[id(p)] for p in g["params"]]) for g in opt.param_groups]
    got, want = groups(mine), groups(ref)
    assert got == want
    if rcfg.MVIT.ZERO_DECAY_POS_CLS:
        zero = {n for wd, _, ns in got if wd == 0.0 for n in ns}
        assert {"pos_embed_spatial", "pos_embed_temporal", "pos_embed_class", "cls_token"} <= zero


def test_maskfeat_checkpoint_loads_into_fine_tune_model():
    """MaskFeat pre-training (MaskMViT) -> fine-tuning (MViT with the mean readout): every encoder key of the fine-tune
    model is in the pre-trained state_dict with the same shape; only the classification norm / head are new."""
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    pt = B200MaskMViT(refshim.load_cfg("masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml", SMALL)).state_dict()
    ft = B200MViT(refshim.load_cfg("masked_ssl/k400_MVITv2_S_16x4_FT.yaml", SMALL))
    fsd = ft.state_dict()
    new = [k for k in fsd if k not in pt]
    assert all(k.startswith(("norm.", "head.")) for k in new), new
    # the pre-training recipe keeps block 14's grid at 14x14, so the last block's spatial rel-pos tables differ in
    # length; the reference's checkpoint loader interpolates exactly those (utils/checkpoint.py, "rel_pos")
    mismatched = [k for k in fsd if k in pt and pt[k].shape != fsd[k].shape]
    assert all(".attn.rel_pos_" in k for k in mismatched), mismatched
    missing, unexpected = ft.load_state_dict({k: v for k, v in pt.items() if k in fsd and k not in mismatched},
                                             strict=False)
    assert sorted(missing) == sorted(new + mismatched) and not unexpected


def test_build_model_serves_the_engine_for_every_in_scope_yaml():
    refshim = _refshim()
    refshim.install()
    import slowfast_b200.integration as integ
    from slowfast.models import build_model
    from slowfast.models.build import MODEL_REGISTRY
    from slowfast_b200.nets.mvit import B200MViT
    saved = dict(MODEL_REGISTRY._obj_map)
    try:
        integ.register(replace=True)
        for yaml in ("Kinetics/MVIT_B_16x4_CONV.yaml", "masked_ssl/k400_VIT_B_16x4_FT.yaml",
                     "masked_ssl/k400_MVITv2_S_16x4_FT.yaml", "masked_ssl/k400_MVITv2_L_16x4_FT.yaml",
                     "masked_ssl/k400_VIT_L_16x4_FT.yaml", "masked_ssl/k400_VIT_H_16x4_FT.yaml"):
            assert type(build_model(refshim.load_cfg(yaml, SMALL))) is B200MViT, yaml
        with pytest.raises(NotImplementedError, match=r"pooling kernel \[1, 9, 9\]"):
            build_model(refshim.load_cfg("Kinetics/MVIT_B_32x3_CONV.yaml"))
    finally:
        MODEL_REGISTRY._obj_map.clear()
        MODEL_REGISTRY._obj_map.update(saved)


@pytest.mark.parametrize("override,match", [
    ({"SEP_POS_EMBED": False}, "SEP_POS_EMBED False"),
    ({"USE_FIXED_SINCOS_POS": True}, "USE_FIXED_SINCOS_POS"),
    ({"CLS_EMBED_ON": False}, "CLS_EMBED_ON False"),
    ({"DROPOUT_RATE": 0.1}, "DROPOUT_RATE"),
    ({"PATCH_2D": True}, "PATCH_2D"),
    ({"REV": {"ENABLE": True}}, "REV.ENABLE"),
    ({"POOL_KVQ_KERNEL": None}, r"pooling kernel \[1, 9, 9\]"),   # MVIT_B_32x3_CONV's K/V pools
])
def test_unsupported_options_are_rejected_at_construction(override, match):
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    with pytest.raises(NotImplementedError, match=match):
        B200MViT(get_cfg("MVIT_B_16x4_CONV", MVIT=override))


def test_mvit_b_32x3_yaml_is_rejected_at_construction():
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    with pytest.raises(NotImplementedError, match=r"kv pooling kernel \[1, 9, 9\]"):
        B200MViT(refshim.load_cfg("Kinetics/MVIT_B_32x3_CONV.yaml"))


def test_maskmvit_with_absolute_positions_is_rejected():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    with pytest.raises(NotImplementedError, match="USE_ABS_POS"):
        B200MaskMViT(get_cfg("MVITv2_S_16x4_MaskFeat_PT", MVIT={"USE_ABS_POS": True}))


def test_patch_embedding_path_is_chosen_by_geometry():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    small = {"NUM_FRAMES": 4, "TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64}
    assert B200MViT(get_cfg("VIT_B_16x4_FT", DATA=small, MVIT={"DEPTH": 1})).patchify
    assert not B200MViT(get_cfg("MVIT_B_16x4_CONV", DATA=small)).patchify
    assert not B200MViT(get_cfg("MVITv2_S_16x4_FT", DATA=small)).patchify
