"""CPU: the ImageNet MViT / ViT recipes (PATCH_2D) - module tree and init parity with the reference, presets, optimizer
grouping, state_dict exchange with the stock model, and the configurations the engine rejects at construction."""
import pytest
import torch

IMAGE_YAMLS = ["ImageNet/MVITv2_T.yaml", "ImageNet/MVITv2_S.yaml", "ImageNet/MVIT_B_16_CONV.yaml",
               "masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml", "masked_ssl/in1k_VIT_L_MaskFeat_FT.yaml"]
# configs/ImageNet/MVITv2_B.yaml does not parse (line 28 is indented by one space); its MVIT block on top of MVITv2_S.yaml
MVITV2_B = ("ImageNet/MVITv2_S.yaml", [
    "MVIT.DEPTH", 24, "MVIT.DIM_MUL", [[2, 2.0], [5, 2.0], [21, 2.0]], "MVIT.HEAD_MUL", [[2, 2.0], [5, 2.0], [21, 2.0]],
    "MVIT.POOL_KV_STRIDE_ADAPTIVE", [1, 4, 4], "MVIT.POOL_KV_STRIDE", [],
    "MVIT.POOL_Q_STRIDE", [[i, 1, 2, 2] if i in (2, 5, 21) else [i, 1, 1, 1] for i in range(24)],
    "MVIT.DROPPATH_RATE", 0.3])
CASES = [(y, []) for y in IMAGE_YAMLS] + [MVITV2_B]
IDS = [y.split("/")[-1] for y in IMAGE_YAMLS] + ["MVITv2_B(composed)"]
PRESETS = {"MVITv2_T": "ImageNet/MVITv2_T.yaml", "MVITv2_S": "ImageNet/MVITv2_S.yaml",
           "VIT_B_IN1K_FT": "masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml"}
SMALL = ["DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    return refshim


@pytest.mark.parametrize("yaml,extra", CASES, ids=IDS)
def test_state_dict_and_init_match_reference(yaml, extra):
    """Same state_dict names / order / shapes and the same values under the same seed: the Conv2d embedding, cls_token
    only with CLS_EMBED_ON, the joint pos_embed drawn after the head and before cls_token, rel_pos_h / rel_pos_w only."""
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(yaml, list(extra))
    with torch.no_grad():
        ref = refshim.build_reference_model(rcfg).state_dict()
        torch.manual_seed(rcfg.RNG_SEED)
        mine = B200MViT(rcfg).state_dict()
    assert [(k, tuple(v.shape)) for k, v in mine.items()] == [(k, tuple(v.shape)) for k, v in ref.items()]
    assert all(torch.equal(mine[k], ref[k]) for k in ref)
    assert mine["patch_embed.proj.weight"].dim() == 4
    assert ("cls_token" in ref) == rcfg.MVIT.CLS_EMBED_ON
    assert ("pos_embed" in ref) == (rcfg.MVIT.USE_ABS_POS and not rcfg.MVIT.SEP_POS_EMBED)
    assert not any(k.endswith("rel_pos_t") for k in ref)


def test_build_model_serves_the_engine_for_every_image_yaml():
    refshim = _refshim()
    refshim.install()
    import slowfast_b200.integration as integ
    from slowfast.models import build_model
    from slowfast.models.build import MODEL_REGISTRY
    from slowfast_b200.nets.mvit import B200MViT
    saved = dict(MODEL_REGISTRY._obj_map)
    try:
        integ.register(replace=True)
        for yaml, extra in CASES:
            assert type(build_model(refshim.load_cfg(yaml, SMALL + list(extra)))) is B200MViT, yaml
    finally:
        MODEL_REGISTRY._obj_map.clear()
        MODEL_REGISTRY._obj_map.update(saved)


@pytest.mark.parametrize("yaml,extra", [
    ("masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml", []),                           # LAYER_DECAY 0.65
    ("masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml", ["MVIT.ZERO_DECAY_POS_CLS", True]),
    ("ImageNet/MVIT_B_16_CONV.yaml", ["MVIT.ZERO_DECAY_POS_CLS", True]),      # joint pos_embed + cls in the zero group
    ("ImageNet/MVITv2_T.yaml", []),
    ("ImageNet/MVITv2_T.yaml", ["MVIT.ZERO_DECAY_POS_CLS", True]),            # rel-pos tables, no cls_token
])
def test_reference_optimizer_groups_match(yaml, extra):
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(yaml, SMALL + list(extra))
    import slowfast.models.optimizer as optim
    ref = refshim.build_reference_model(rcfg)
    mine = B200MViT(rcfg)
    assert mine.no_weight_decay() == ref.no_weight_decay()

    def groups(model):
        names = {id(p): n for n, p in model.named_parameters()}
        opt = optim.construct_optimizer(model, rcfg)
        return [(g["weight_decay"], g.get("layer_decay"), [names[id(p)] for p in g["params"]]) for g in opt.param_groups]
    assert groups(mine) == groups(ref)


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
    for key in ("NUM_FRAMES", "TRAIN_CROP_SIZE", "TEST_CROP_SIZE", "INPUT_CHANNEL_NUM", "MEAN", "STD"):
        assert list(mine.DATA[key]) == list(rcfg.DATA[key]) if isinstance(mine.DATA[key], list) else \
            mine.DATA[key] == rcfg.DATA[key], key
    for key in ("NUM_CLASSES", "ARCH", "MODEL_NAME", "DROPOUT_RATE", "LOSS_FUNC"):
        assert mine.MODEL[key] == rcfg.MODEL[key], key


@pytest.mark.parametrize("yaml", ["ImageNet/MVITv2_T.yaml", "ImageNet/MVIT_B_16_CONV.yaml"])
def test_state_dict_exchanges_with_the_stock_model(yaml):
    """A stock checkpoint loads into the engine model with strict=True and the reverse (the cls-free / spatial-only
    MViTv2-T, and the joint-table MViTv1-B)."""
    from slowfast_b200.nets.mvit import B200MViT
    refshim = _refshim()
    rcfg = refshim.load_cfg(yaml, SMALL)
    torch.manual_seed(1)
    ref = refshim.build_reference_model(rcfg)
    torch.manual_seed(2)
    mine = B200MViT(rcfg)
    mine.load_state_dict(ref.state_dict(), strict=True)
    assert all(torch.equal(a, b) for a, b in zip(mine.state_dict().values(), ref.state_dict().values()))
    torch.manual_seed(3)
    other = B200MViT(rcfg)
    ref.load_state_dict(other.state_dict(), strict=True)
    assert all(torch.equal(a, b) for a, b in zip(other.state_dict().values(), ref.state_dict().values()))


@pytest.mark.parametrize("override,match", [
    ({"PATCH_KERNEL": [1, 7, 7]}, "PATCH_2D"),
    ({"PATCH_STRIDE": [1, 4, 4]}, "PATCH_2D"),
    ({"PATCH_PADDING": [0, 3, 3]}, "PATCH_2D"),
    ({"USE_ABS_POS": True, "SEP_POS_EMBED": True}, "SEP_POS_EMBED with CLS_EMBED_ON False"),
    ({"REL_POS_SPATIAL": False, "REL_POS_TEMPORAL": True}, "REL_POS_TEMPORAL without REL_POS_SPATIAL"),
    ({"USE_FIXED_SINCOS_POS": True}, "USE_FIXED_SINCOS_POS"),
    ({"REV": {"ENABLE": True}}, "REV.ENABLE"),
])
def test_unsupported_image_options_are_rejected_at_construction(override, match):
    """Clean rejections naming the option, never an IndexError from the patch geometry."""
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    with pytest.raises(NotImplementedError, match=match):
        B200MViT(get_cfg("MVITv2_T", MVIT=override))


def test_two_d_patches_need_one_frame():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    with pytest.raises(NotImplementedError, match="NUM_FRAMES"):
        B200MViT(get_cfg("MVITv2_T", DATA={"NUM_FRAMES": 4}))


@pytest.mark.parametrize("yaml", ["masked_ssl/in1k_VIT_B_MaskFeat_PT.yaml", "masked_ssl/in1k_VIT_L_MaskFeat_PT.yaml"])
def test_image_maskfeat_pretraining_is_rejected(yaml):
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    refshim = _refshim()
    with pytest.raises(NotImplementedError, match="USE_ABS_POS"):
        B200MaskMViT(refshim.load_cfg(yaml))


def test_maskmvit_with_2d_patches_is_rejected():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    cfg = get_cfg("MVITv2_S_16x4_MaskFeat_PT", DATA={"NUM_FRAMES": 1},
                  MVIT={"PATCH_2D": True, "PATCH_KERNEL": [7, 7], "PATCH_STRIDE": [4, 4], "PATCH_PADDING": [3, 3]})
    with pytest.raises(NotImplementedError, match="PATCH_2D"):
        B200MaskMViT(cfg)


def test_video_input_to_an_image_model_is_an_error():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    model = B200MViT(get_cfg("MVITv2_T", DATA={"TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64}))
    with pytest.raises(ValueError, match=r"\[B, C, H, W\]"):
        model([torch.zeros(1, 3, 1, 64, 64)])


def test_image_geometry_and_embedding_path():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT, block_specs
    t = get_cfg("MVITv2_T")
    assert [s["size"] for s in block_specs(t)][:2] == [[1, 56, 56], [1, 56, 56]]
    m = B200MViT(t)
    assert (m.T, m.H, m.W, m.ncls, m.patchify) == (1, 56, 56, 0, False)
    assert m._pe_geometry() == ((1, 7, 7), (1, 4, 4), (0, 3, 3))
    v = B200MViT(get_cfg("VIT_B_IN1K_FT", MVIT={"DEPTH": 1}))
    assert (v.T, v.H, v.W, v.ncls, v.patchify) == (1, 14, 14, 1, True)
    assert not hasattr(m.blocks[0].attn, "rel_pos_t") and hasattr(m.blocks[0].attn, "rel_pos_h")
