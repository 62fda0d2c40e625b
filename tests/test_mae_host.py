"""CPU: MAE pre-training (k400_VIT_{B,L,H}_16x4_MAE_PT) on the engine - module tree and init parity with the reference's
MaskMViT, weight-decay groups, build_model dispatch, the MAE -> fine-tune checkpoint path, and the rejections."""
import pytest
import torch

MAE_YAMLS = ["masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml", "masked_ssl/k400_VIT_L_16x4_MAE_PT.yaml",
             "masked_ssl/k400_VIT_H_16x4_MAE_PT.yaml"]
SMALL = ["DATA.NUM_FRAMES", 4, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    return refshim


@pytest.mark.parametrize("yaml", MAE_YAMLS)
def test_state_dict_and_init_match_reference(yaml):
    """Same state_dict names / order / shapes and bit-identical values under one seed: the deleted MViT norm / head
    still draw, the decoder blocks' default Linear draws precede the head's trunc_normal, decoder_embed keeps PyTorch's
    default init, mask_token is drawn before decoder_pos_embed."""
    from slowfast_b200.nets.mae import B200MAE
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(yaml)
    with torch.no_grad():
        ref = refshim.build_reference_model(rcfg).state_dict()
        torch.manual_seed(rcfg.RNG_SEED)
        model = B200MaskMViT(rcfg)
        mine = model.state_dict()
    assert type(model) is B200MAE
    assert [(k, tuple(v.shape)) for k, v in mine.items()] == [(k, tuple(v.shape)) for k, v in ref.items()]
    assert all(torch.equal(mine[k], ref[k]) for k in ref)
    assert model.len_keep == 156 and model.n_tokens == 1568


def test_preset_mirrors_the_yaml():
    from slowfast_b200.config import get_cfg
    refshim = _refshim()
    for preset, yaml in (("VIT_B_16x4_MAE_PT", MAE_YAMLS[0]), ("VIT_L_16x4_MAE_PT", MAE_YAMLS[1]),
                         ("VIT_H_16x4_MAE_PT", MAE_YAMLS[2])):
        rcfg = refshim.load_cfg(yaml)
        mine = get_cfg(preset)
        for sect in ("MVIT", "MASK", "AUG"):
            for key, v in mine[sect].items():
                if key == "REV":
                    continue
                want = rcfg[sect][key]
                assert (list(v) if isinstance(v, (list, tuple)) else v) == \
                    (list(want) if isinstance(want, (list, tuple)) else want), (preset, sect, key)
        for key in ("NUM_FRAMES", "TRAIN_CROP_SIZE", "TEST_CROP_SIZE", "INPUT_CHANNEL_NUM"):
            assert mine.DATA[key] == rcfg.DATA[key], key
        for key in ("ARCH", "MODEL_NAME", "LOSS_FUNC", "DROPOUT_RATE"):
            assert mine.MODEL[key] == rcfg.MODEL[key], key


@pytest.mark.parametrize("zero_decay", [False, True])
def test_no_weight_decay_and_optimizer_groups_match(zero_decay):
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(MAE_YAMLS[0], SMALL + ["MVIT.ZERO_DECAY_POS_CLS", zero_decay])
    import slowfast.models.optimizer as optim
    ref = refshim.build_reference_model(rcfg)
    mine = B200MaskMViT(rcfg)
    assert mine.no_weight_decay() == ref.no_weight_decay()
    if zero_decay:
        assert mine.no_weight_decay() == ["pos_embed_decoder", "cls_token"]

    def groups(model):
        names = {id(p): n for n, p in model.named_parameters()}
        opt = optim.construct_optimizer(model, rcfg)
        return [(g["weight_decay"], g.get("layer_decay"), [names[id(p)] for p in g["params"]]) for g in opt.param_groups]
    assert groups(mine) == groups(ref)


def test_build_model_dispatches_on_mae_on():
    refshim = _refshim()
    refshim.install()
    import slowfast_b200.integration as integ
    from slowfast.models import build_model
    from slowfast.models.build import MODEL_REGISTRY
    from slowfast_b200.nets.mae import B200MAE
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    saved = dict(MODEL_REGISTRY._obj_map)
    try:
        integ.register(replace=True)
        for yaml in MAE_YAMLS:
            assert type(build_model(refshim.load_cfg(yaml, SMALL))) is B200MAE, yaml
        for yaml in ("masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml", "masked_ssl/k400_MVITv2_L_16x4_MaskFeat_PT.yaml"):
            assert type(build_model(refshim.load_cfg(yaml, ["DATA.NUM_FRAMES", 8, "DATA.TRAIN_CROP_SIZE", 64,
                                                            "DATA.TEST_CROP_SIZE", 64]))) is B200MaskMViT, yaml
    finally:
        MODEL_REGISTRY._obj_map.clear()
        MODEL_REGISTRY._obj_map.update(saved)


def test_mae_checkpoint_loads_into_fine_tune_model():
    """MAE pre-training -> ViT-B fine-tuning: the engine's and the reference's fine-tune models report the same missing /
    unexpected keys for the same pre-trained state_dict."""
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    pt_cfg = refshim.load_cfg(MAE_YAMLS[0], SMALL)
    ft_cfg = refshim.load_cfg("masked_ssl/k400_VIT_B_16x4_FT.yaml", SMALL)
    pt = B200MaskMViT(pt_cfg).state_dict()
    assert pt.keys() == refshim.build_reference_model(pt_cfg).state_dict().keys()
    results = []
    for ft in (B200MViT(ft_cfg), refshim.build_reference_model(ft_cfg)):
        fsd = ft.state_dict()
        r = ft.load_state_dict({k: v for k, v in pt.items() if k not in fsd or fsd[k].shape == v.shape}, strict=False)
        results.append((sorted(r.missing_keys), sorted(r.unexpected_keys)))
    assert results[0] == results[1]
    assert all(k.startswith(("head.",)) for k in results[0][0]), results[0][0]


def _small(**over):
    from slowfast_b200.config import get_cfg
    cfg = get_cfg("VIT_B_16x4_MAE_PT", DATA={"NUM_FRAMES": 4, "TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64},
                  MVIT={"DEPTH": 1}, MASK={"PRETRAIN_DEPTH": [0], "DECODER_DEPTH": 1})
    return cfg.merge(over)


@pytest.mark.parametrize("override,match", [
    ({"MASK": {"PER_FRAME_MASKING": True}}, "PER_FRAME_MASKING"),
    ({"AUG": {"MASK_TUBE": True}}, "AUG.MASK_TUBE"),
    ({"MASK": {"MAE_RND_MASK": False}}, "without MASK.MAE_RND_MASK"),
    ({"MASK": {"DECODER_SEP_POS_EMBED": True}}, "DECODER_SEP_POS_EMBED"),
    ({"MASK": {"DEC_KV_KERNEL": [3, 3, 3]}}, "DEC_KV_KERNEL"),
    ({"MASK": {"DEC_KV_STRIDE": [1, 2, 2]}}, "DEC_KV_STRIDE"),
    ({"MASK": {"PRED_HOG": True}}, "PRED_HOG"),
    ({"MASK": {"SCALE_INIT_BY_DEPTH": True}}, "SCALE_INIT_BY_DEPTH"),
    ({"VIS_MASK": {"ENABLE": True}}, "VIS_MASK.ENABLE"),
    ({"MVIT": {"USE_ABS_POS": False}}, "USE_ABS_POS False"),
    ({"MVIT": {"SEP_POS_EMBED": False}}, "SEP_POS_EMBED False"),
    ({"MASK": {"PRETRAIN_DEPTH": [0, 0]}}, "more than one prediction depth"),
    ({"DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 448, "TEST_CROP_SIZE": 448}}, "6272 tokens per clip"),
    ({"MVIT": {"REL_POS_SPATIAL": True}}, "relative positions"),
    ({"MVIT": {"POOL_Q_STRIDE": [[0, 1, 2, 2]]}}, "pooling"),
    ({"MVIT": {"DROPPATH_RATE": 0.1}}, "DROPPATH_RATE"),
    ({"MVIT": {"RESIDUAL_POOLING": True}}, "RESIDUAL_POOLING"),
    ({"AUG": {"MASK_RATIO": 0.99}}, "MASK_RATIO"),
])
def test_unsupported_mae_options_are_rejected_at_construction(override, match):
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    with pytest.raises(NotImplementedError, match=match):
        B200MaskMViT(_small(**override))


def test_small_config_builds():
    from slowfast_b200.nets.mae import B200MAE
    m = B200MAE(_small())
    assert (m.n_tokens, m.len_keep, len(m.blocks), len(m.dec_specs)) == (32, 3, 1, 1)
