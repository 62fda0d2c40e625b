"""CPU: host-side geometry / bookkeeping of the model builders (no kernels run)."""
import pytest
import torch


def test_flat_gradient_slots_are_256_byte_aligned():
    from slowfast_b200.engine import FLAT_ALIGN, flat_offsets
    params = [torch.nn.Parameter(torch.zeros(s)) for s in (54, 8, (54, 24, 1, 1, 1), 400, (3, 3), 1)]
    offsets, total = flat_offsets(params)
    assert FLAT_ALIGN * 4 == 256
    assert all(o % FLAT_ALIGN == 0 for o in offsets)
    assert all(b - a >= p.numel() for a, b, p in zip(offsets, offsets[1:] + [total], params))


def test_mvit_block_specs_both_expansion_modes():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import block_specs
    v2 = block_specs(get_cfg("MVITv2_S_16x4"))  # DIM_MUL_IN_ATT True: the block that multiplies owns the wider dim_out
    assert [s["dim_out"] for s in v2] == [96] + [192] * 2 + [384] * 11 + [768] * 2
    assert [s["heads"] for s in v2] == [1] + [2] * 2 + [4] * 11 + [8] * 2
    v1 = block_specs(get_cfg("MVITv2_S_16x4_MaskFeat_PT"))  # shipped MaskFeat yaml: expansion in the previous block's MLP
    assert [s["dim"] for s in v1] == [96] + [192] * 2 + [384] * 11 + [768] * 2
    assert [s["dim_out"] for s in v1] == [192] + [192] + [384] + [384] * 10 + [768] + [768] * 2
    # (size = the block's INPUT token grid) the MaskFeat yaml's q pooling keeps the last stage at 14x14 for the
    # prediction head; the classification yaml pools once more at block 14
    assert v1[-1]["size"] == [8, 14, 14] and v2[-1]["size"] == [8, 7, 7] and v2[-1]["sq"] == [1, 1, 1]


def test_maskfeat_feature_geometry_and_head():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.maskfeat import B200MaskMViT, calc_mvit_feature_geometry
    cfg = get_cfg("MVITv2_S_16x4_MaskFeat_PT")
    size, stride = calc_mvit_feature_geometry(cfg)
    assert size[15] == [8, 14, 14] and stride[15] == [2, 16, 16] and size[0] == [8, 56, 56]
    m = B200MaskMViT(cfg)
    assert m.pred_head.projections[0].out_features == 9 * 4 * 3  # 9 bins x (16/8)^2 cells x RGB
    assert not hasattr(m, "head") and not hasattr(m, "norm")
    assert tuple(m.mask_token.shape) == (1, 1, 96)
    assert m.no_weight_decay() == []  # ZERO_DECAY_POS_CLS False in the yaml


def test_x3d_round_width_and_pool_size():
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.x3d import head_pool_size, round_width
    assert [round_width(12, 2.0), round_width(24, 2.0, divisor=8), round_width(54, 1 / 16, 8, 8)] == [24, 48, 8]
    assert round_width(432, 1 / 16, 8, 8) == 32  # 27 -> 24 is below 0.9 x 27 -> bumped by the divisor
    assert head_pool_size(get_cfg("X3D_M")) == (16, 7, 7)


@pytest.mark.parametrize("preset,spec", [("X3D_M", "slowfast_b200.nets.x3d:B200X3D"),
                                         ("MVITv2_S_16x4", "slowfast_b200.nets.mvit:B200MViT"),
                                         ("C2D_8x8_R50", "slowfast_b200.nets.resnet_single:B200ResNet")])
def test_no_cpu_fallback_other_models(preset, spec):
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    import importlib

    from slowfast_b200.config import get_cfg
    from slowfast_b200.lib import NativeLibraryError
    mod, cls = spec.split(":")
    overrides = dict(DATA={"NUM_FRAMES": 8, "TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64})
    m = getattr(importlib.import_module(mod), cls)(get_cfg(preset, **overrides))
    with pytest.raises(NativeLibraryError):
        m([torch.zeros(1, 3, 8, 64, 64)])

