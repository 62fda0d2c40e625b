"""Stand-alone configuration for the engine's model builders.

The engine classes read the SAME key names as the reference's config tree (slowfast/config/defaults.py) by plain
attribute access, so they accept either the reference's own ``CfgNode`` (drop-in through ``build_model``) or the
light ``Cfg`` objects built here (tests / bench on a box where the reference does not exist).  Only keys that the
hot path consumes are present; defaults and preset values restate slowfast/config/defaults.py and the yaml files
cited per preset.
"""
from __future__ import annotations

import copy
from typing import Any, Dict


class Cfg(dict):
    """dict with attribute access and nested construction."""

    def __init__(self, d: Dict[str, Any] | None = None):
        super().__init__()
        for k, v in (d or {}).items():
            self[k] = Cfg(v) if isinstance(v, dict) else v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def clone(self) -> "Cfg":
        return copy.deepcopy(self)

    def merge(self, other: Dict[str, Any]) -> "Cfg":
        for k, v in other.items():
            if isinstance(v, dict) and isinstance(self.get(k), Cfg):
                self[k].merge(v)
            else:
                self[k] = Cfg(v) if isinstance(v, dict) else v
        return self


# defaults (slowfast/config/defaults.py: BN :99-126, RESNET :296-327, MODEL :393-441, SLOWFAST :637-648,
# DATA :666-716, NONLOCAL :366, DETECTION :950, MULTIGRID :1039)
_DEFAULTS = {
    "BN": {"NORM_TYPE": "batchnorm", "NUM_SPLITS": 1, "NUM_SYNC_DEVICES": 1, "WEIGHT_DECAY": 0.0},
    "RESNET": {
        "TRANS_FUNC": "bottleneck_transform", "NUM_GROUPS": 1, "WIDTH_PER_GROUP": 64, "INPLACE_RELU": True,
        "STRIDE_1X1": False, "ZERO_INIT_FINAL_BN": False, "ZERO_INIT_FINAL_CONV": False, "DEPTH": 50,
        "NUM_BLOCK_TEMP_KERNEL": [[3], [4], [6], [3]], "SPATIAL_STRIDES": [[1], [2], [2], [2]],
        "SPATIAL_DILATIONS": [[1], [1], [1], [1]],
    },
    "NONLOCAL": {"LOCATION": [[[]], [[]], [[]], [[]]], "GROUP": [[1], [1], [1], [1]], "INSTANTIATION": "dot_product",
                 "POOL": [[[1, 2, 2], [1, 2, 2]]] * 4},
    "MODEL": {
        "ARCH": "slowfast", "MODEL_NAME": "SlowFast", "NUM_CLASSES": 400, "LOSS_FUNC": "cross_entropy",
        "DROPOUT_RATE": 0.5, "DROPCONNECT_RATE": 0.0, "FC_INIT_STD": 0.01, "HEAD_ACT": "softmax",
        "ACT_CHECKPOINT": False, "DETACH_FINAL_FC": False, "FROZEN_BN": False,
    },
    "SLOWFAST": {"BETA_INV": 8, "ALPHA": 8, "FUSION_CONV_CHANNEL_RATIO": 2, "FUSION_KERNEL_SZ": 5},
    "DATA": {"NUM_FRAMES": 8, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 256, "INPUT_CHANNEL_NUM": [3, 3],
             "MEAN": [0.45, 0.45, 0.45], "STD": [0.225, 0.225, 0.225], "REVERSE_INPUT_CHANNEL": False},
    "DETECTION": {"ENABLE": False},
    "MULTIGRID": {"SHORT_CYCLE": False},
    "CONTRASTIVE": {"NUM_MLP_LAYERS": 1, "MLP_DIM": 2048, "BN_MLP": False, "BN_SYNC_MLP": False, "PREDICTOR_DEPTHS": []},
    "TRAIN": {"MIXED_PRECISION": False, "BATCH_SIZE": 64},
    "NUM_GPUS": 1,
    "RNG_SEED": 1,
    # MVIT defaults (slowfast/config/defaults.py:450-628)
    "MVIT": {
        "MODE": "conv", "POOL_FIRST": False, "CLS_EMBED_ON": True, "PATCH_KERNEL": [3, 7, 7],
        "PATCH_STRIDE": [2, 4, 4], "PATCH_PADDING": [2, 4, 4], "PATCH_2D": False, "EMBED_DIM": 96, "NUM_HEADS": 1,
        "MLP_RATIO": 4.0, "QKV_BIAS": True, "DROPPATH_RATE": 0.1, "LAYER_SCALE_INIT_VALUE": 0.0, "DEPTH": 16,
        "NORM": "layernorm", "DIM_MUL": [], "HEAD_MUL": [], "POOL_KV_STRIDE": [], "POOL_KV_STRIDE_ADAPTIVE": None,
        "POOL_Q_STRIDE": [], "POOL_KVQ_KERNEL": None, "ZERO_DECAY_POS_CLS": True, "NORM_STEM": False,
        "SEP_POS_EMBED": False, "DROPOUT_RATE": 0.0, "USE_ABS_POS": True, "REL_POS_SPATIAL": False,
        "REL_POS_TEMPORAL": False, "REL_POS_ZERO_INIT": False, "RESIDUAL_POOLING": False, "DIM_MUL_IN_ATT": False,
        "SEPARATE_QKV": False, "HEAD_INIT_SCALE": 1.0, "USE_MEAN_POOLING": False, "USE_FIXED_SINCOS_POS": False,
        "REV": {"ENABLE": False, "RESPATH_FUSE": "concat"},
    },
    # MASK defaults (slowfast/config/defaults.py:563-609)
    "MASK": {"ENABLE": False, "MAE_ON": False, "MAE_RND_MASK": False, "PER_FRAME_MASKING": False,
             "TIME_STRIDE_LOSS": True, "NORM_PRED_PIXEL": True, "SCALE_INIT_BY_DEPTH": False, "DECODER_EMBED_DIM": 512,
             "DECODER_SEP_POS_EMBED": False, "DEC_KV_KERNEL": [], "DEC_KV_STRIDE": [], "PRETRAIN_DEPTH": [15],
             "HEAD_TYPE": "separate", "DECODER_DEPTH": 0, "PRED_HOG": False},
    # AUG / VIS_MASK keys the MAE model reads (slowfast/config/defaults.py:214-234)
    "AUG": {"MASK_TUBE": False, "MASK_RATIO": 0.0},
    "VIS_MASK": {"ENABLE": False},
    # X3D defaults (slowfast/config/defaults.py:333-358)
    "X3D": {"WIDTH_FACTOR": 1.0, "DEPTH_FACTOR": 1.0, "BOTTLENECK_FACTOR": 1.0, "DIM_C5": 2048, "DIM_C1": 12,
            "SCALE_RES2": False, "BN_LIN5": False, "CHANNELWISE_3x3x3": True},
    # engine-side knobs (not in the reference): operand precision of the tensor-core kernels
    "B200": {"NSPLIT": 3, "CUDA_GRAPH": True},
}

_PRESETS = {
    # configs/Kinetics/SLOWFAST_8x8_R50.yaml
    "SLOWFAST_8x8_R50": {
        "DATA": {"NUM_FRAMES": 32, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 256, "INPUT_CHANNEL_NUM": [3, 3]},
        "SLOWFAST": {"ALPHA": 4, "BETA_INV": 8, "FUSION_CONV_CHANNEL_RATIO": 2, "FUSION_KERNEL_SZ": 7},
        "RESNET": {"ZERO_INIT_FINAL_BN": True, "WIDTH_PER_GROUP": 64, "NUM_GROUPS": 1, "DEPTH": 50,
                   "NUM_BLOCK_TEMP_KERNEL": [[3, 3], [4, 4], [6, 6], [3, 3]],
                   "SPATIAL_STRIDES": [[1, 1], [2, 2], [2, 2], [2, 2]],
                   "SPATIAL_DILATIONS": [[1, 1], [1, 1], [1, 1], [1, 1]]},
        "NONLOCAL": {"LOCATION": [[[], []], [[], []], [[], []], [[], []]], "GROUP": [[1, 1], [1, 1], [1, 1], [1, 1]]},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "slowfast", "MODEL_NAME": "SlowFast", "DROPOUT_RATE": 0.5},
        "TRAIN": {"BATCH_SIZE": 64},
        "RNG_SEED": 0,
    },
    # configs/Kinetics/MVITv2_S_16x4.yaml
    "MVITv2_S_16x4": {
        "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": {"ZERO_DECAY_POS_CLS": False, "USE_ABS_POS": False, "REL_POS_SPATIAL": True, "REL_POS_TEMPORAL": True,
                 "DEPTH": 16, "NUM_HEADS": 1, "EMBED_DIM": 96, "PATCH_KERNEL": [3, 7, 7], "PATCH_STRIDE": [2, 4, 4],
                 "PATCH_PADDING": [1, 3, 3], "MLP_RATIO": 4.0, "QKV_BIAS": True, "DROPPATH_RATE": 0.2,
                 "NORM": "layernorm", "MODE": "conv", "CLS_EMBED_ON": True,
                 "DIM_MUL": [[1, 2.0], [3, 2.0], [14, 2.0]], "HEAD_MUL": [[1, 2.0], [3, 2.0], [14, 2.0]],
                 "POOL_KVQ_KERNEL": [3, 3, 3], "POOL_KV_STRIDE_ADAPTIVE": [1, 8, 8],
                 "POOL_Q_STRIDE": [[0, 1, 1, 1], [1, 1, 2, 2], [2, 1, 1, 1], [3, 1, 2, 2], [4, 1, 1, 1], [5, 1, 1, 1],
                                   [6, 1, 1, 1], [7, 1, 1, 1], [8, 1, 1, 1], [9, 1, 1, 1], [10, 1, 1, 1],
                                   [11, 1, 1, 1], [12, 1, 1, 1], [13, 1, 1, 1], [14, 1, 2, 2], [15, 1, 1, 1]],
                 "DROPOUT_RATE": 0.0, "DIM_MUL_IN_ATT": True, "RESIDUAL_POOLING": True},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "mvit", "MODEL_NAME": "MViT", "DROPOUT_RATE": 0.5},
        "TRAIN": {"BATCH_SIZE": 16},
        "RNG_SEED": 0,
    },
    # configs/masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml
    "MVITv2_S_16x4_MaskFeat_PT": {
        "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": {"ZERO_DECAY_POS_CLS": False, "USE_ABS_POS": False, "SEP_POS_EMBED": True, "REL_POS_SPATIAL": True,
                 "REL_POS_TEMPORAL": True, "DEPTH": 16, "NUM_HEADS": 1, "EMBED_DIM": 96, "PATCH_KERNEL": [3, 7, 7],
                 "PATCH_STRIDE": [2, 4, 4], "PATCH_PADDING": [1, 3, 3], "QKV_BIAS": True, "DROPPATH_RATE": 0.0,
                 "MODE": "conv", "CLS_EMBED_ON": True,
                 "DIM_MUL": [[1, 2.0], [3, 2.0], [14, 2.0]], "HEAD_MUL": [[1, 2.0], [3, 2.0], [14, 2.0]],
                 "POOL_KVQ_KERNEL": [3, 3, 3], "POOL_KV_STRIDE_ADAPTIVE": [1, 8, 8],
                 # [14, 1, 1, 1] (not [14, 1, 2, 2]) keeps the last stage at 14x14 for the prediction head
                 "POOL_Q_STRIDE": [[0, 1, 1, 1], [1, 1, 2, 2], [2, 1, 1, 1], [3, 1, 2, 2], [4, 1, 1, 1], [5, 1, 1, 1],
                                   [6, 1, 1, 1], [7, 1, 1, 1], [8, 1, 1, 1], [9, 1, 1, 1], [10, 1, 1, 1],
                                   [11, 1, 1, 1], [12, 1, 1, 1], [13, 1, 1, 1], [14, 1, 1, 1], [15, 1, 1, 1]],
                 "DIM_MUL_IN_ATT": False, "RESIDUAL_POOLING": True},
        "MASK": {"ENABLE": True, "PRETRAIN_DEPTH": [15], "HEAD_TYPE": "separate", "PRED_HOG": True},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "maskmvit", "MODEL_NAME": "MaskMViT", "LOSS_FUNC": "multi_mse",
                  "DROPOUT_RATE": 0.0},
        "TRAIN": {"BATCH_SIZE": 32},
        "RNG_SEED": 0,
    },
    # configs/Kinetics/MVITv2_B_32x3.yaml
    "MVITv2_B_32x3": {
        "DATA": {"NUM_FRAMES": 32, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": {"ZERO_DECAY_POS_CLS": False, "USE_ABS_POS": False, "REL_POS_SPATIAL": True, "REL_POS_TEMPORAL": True,
                 "DEPTH": 24, "NUM_HEADS": 1, "EMBED_DIM": 96, "PATCH_KERNEL": [3, 7, 7], "PATCH_STRIDE": [2, 4, 4],
                 "PATCH_PADDING": [1, 3, 3], "MLP_RATIO": 4.0, "QKV_BIAS": True, "DROPPATH_RATE": 0.3,
                 "NORM": "layernorm", "MODE": "conv", "CLS_EMBED_ON": True,
                 "DIM_MUL": [[2, 2.0], [5, 2.0], [21, 2.0]], "HEAD_MUL": [[2, 2.0], [5, 2.0], [21, 2.0]],
                 "POOL_KVQ_KERNEL": [3, 3, 3], "POOL_KV_STRIDE_ADAPTIVE": [1, 8, 8],
                 "POOL_Q_STRIDE": [[i, 1, 2, 2] if i in (2, 5, 21) else [i, 1, 1, 1] for i in range(24)],
                 "DROPOUT_RATE": 0.0, "DIM_MUL_IN_ATT": True, "RESIDUAL_POOLING": True},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "mvit", "MODEL_NAME": "MViT", "DROPOUT_RATE": 0.5},
        "TRAIN": {"BATCH_SIZE": 16},
        "RNG_SEED": 0,
    },
    # BASELINE.json configs[4]: "MViTv2-B MaskFeat pretrain 32x224x224 (masked_ssl config)".  The reference ships no
    # MViTv2-B MaskFeat yaml (configs/masked_ssl has S and L): composed as SURVEY.md section 3.5 describes - the MVIT block of
    # configs/Kinetics/MVITv2_B_32x3.yaml with the last Q stride [21,1,2,2] -> [21,1,1,1] (14x14 output grid for the
    # prediction head, as the S file does for its block 14) and PRETRAIN_DEPTH [23], plus the MASK / MODEL blocks of
    # configs/masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml (mask cube window 16x7x7 for the 16 temporal tokens).
    "MVITv2_B_32x3_MaskFeat_PT": {
        "DATA": {"NUM_FRAMES": 32, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": {"ZERO_DECAY_POS_CLS": False, "USE_ABS_POS": False, "SEP_POS_EMBED": True, "REL_POS_SPATIAL": True,
                 "REL_POS_TEMPORAL": True, "DEPTH": 24, "NUM_HEADS": 1, "EMBED_DIM": 96, "PATCH_KERNEL": [3, 7, 7],
                 "PATCH_STRIDE": [2, 4, 4], "PATCH_PADDING": [1, 3, 3], "MLP_RATIO": 4.0, "QKV_BIAS": True,
                 "DROPPATH_RATE": 0.0, "NORM": "layernorm", "MODE": "conv", "CLS_EMBED_ON": True,
                 "DIM_MUL": [[2, 2.0], [5, 2.0], [21, 2.0]], "HEAD_MUL": [[2, 2.0], [5, 2.0], [21, 2.0]],
                 "POOL_KVQ_KERNEL": [3, 3, 3], "POOL_KV_STRIDE_ADAPTIVE": [1, 8, 8],
                 "POOL_Q_STRIDE": [[i, 1, 2, 2] if i in (2, 5) else [i, 1, 1, 1] for i in range(24)],
                 "DROPOUT_RATE": 0.0, "DIM_MUL_IN_ATT": True, "RESIDUAL_POOLING": True},
        "MASK": {"ENABLE": True, "PRETRAIN_DEPTH": [23], "HEAD_TYPE": "separate", "PRED_HOG": True},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "maskmvit", "MODEL_NAME": "MaskMViT", "LOSS_FUNC": "multi_mse",
                  "DROPOUT_RATE": 0.0},
        "TRAIN": {"BATCH_SIZE": 32},
        "RNG_SEED": 0,
    },
    # configs/Kinetics/X3D_M.yaml
    "X3D_M": {
        "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 256, "INPUT_CHANNEL_NUM": [3]},
        "X3D": {"WIDTH_FACTOR": 2.0, "DEPTH_FACTOR": 2.2, "BOTTLENECK_FACTOR": 2.25, "DIM_C5": 2048, "DIM_C1": 12},
        "RESNET": {"ZERO_INIT_FINAL_BN": True, "TRANS_FUNC": "x3d_transform", "STRIDE_1X1": False, "DEPTH": 50,
                   "NUM_GROUPS": 1, "WIDTH_PER_GROUP": 64},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "x3d", "MODEL_NAME": "X3D", "DROPOUT_RATE": 0.5},
        "TRAIN": {"BATCH_SIZE": 128},
        "RNG_SEED": 0,
    },
    # configs/Kinetics/SLOW_8x8_R50.yaml
    "SLOW_8x8_R50": {
        "DATA": {"NUM_FRAMES": 8, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 256, "INPUT_CHANNEL_NUM": [3]},
        "RESNET": {"ZERO_INIT_FINAL_BN": True, "WIDTH_PER_GROUP": 64, "NUM_GROUPS": 1, "DEPTH": 50,
                   "NUM_BLOCK_TEMP_KERNEL": [[3], [4], [6], [3]]},
        "NONLOCAL": {"LOCATION": [[[]], [[]], [[]], [[]]], "GROUP": [[1], [1], [1], [1]]},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "slow", "MODEL_NAME": "ResNet", "DROPOUT_RATE": 0.5},
        "RNG_SEED": 0,
    },
    # configs/Kinetics/I3D_8x8_R50.yaml
    "I3D_8x8_R50": {
        "DATA": {"NUM_FRAMES": 8, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 256, "INPUT_CHANNEL_NUM": [3]},
        "RESNET": {"ZERO_INIT_FINAL_BN": True, "WIDTH_PER_GROUP": 64, "NUM_GROUPS": 1, "DEPTH": 50,
                   "NUM_BLOCK_TEMP_KERNEL": [[3], [4], [6], [3]]},
        "NONLOCAL": {"LOCATION": [[[]], [[]], [[]], [[]]], "GROUP": [[1], [1], [1], [1]]},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "i3d", "MODEL_NAME": "ResNet", "DROPOUT_RATE": 0.5},
        "RNG_SEED": 0,
    },
    # configs/Kinetics/C2D_8x8_R50.yaml
    "C2D_8x8_R50": {
        "DATA": {"NUM_FRAMES": 8, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 256, "INPUT_CHANNEL_NUM": [3]},
        "RESNET": {"ZERO_INIT_FINAL_BN": True, "WIDTH_PER_GROUP": 64, "NUM_GROUPS": 1, "DEPTH": 50,
                   "NUM_BLOCK_TEMP_KERNEL": [[3], [4], [6], [3]]},
        "NONLOCAL": {"LOCATION": [[[]], [[]], [[]], [[]]], "GROUP": [[1], [1], [1], [1]], "INSTANTIATION": "softmax"},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "c2d", "MODEL_NAME": "ResNet", "DROPOUT_RATE": 0.5},
        "RNG_SEED": 0,
    },
}
_MVIT_B_POOL = {"DIM_MUL": [[1, 2.0], [3, 2.0], [14, 2.0]], "HEAD_MUL": [[1, 2.0], [3, 2.0], [14, 2.0]],
                 "POOL_KVQ_KERNEL": [3, 3, 3], "POOL_KV_STRIDE_ADAPTIVE": [1, 8, 8]}
_PRESETS.update({
    # configs/Kinetics/MVIT_B_16x4_CONV.yaml (MViTv1-B: separable absolute positions, cls readout)
    "MVIT_B_16x4_CONV": {
        "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": dict(_MVIT_B_POOL, ZERO_DECAY_POS_CLS=False, SEP_POS_EMBED=True, DEPTH=16, NUM_HEADS=1, EMBED_DIM=96,
                     PATCH_KERNEL=[3, 7, 7], PATCH_STRIDE=[2, 4, 4], PATCH_PADDING=[1, 3, 3], MLP_RATIO=4.0,
                     QKV_BIAS=True, DROPPATH_RATE=0.2, NORM="layernorm", MODE="conv", CLS_EMBED_ON=True,
                     POOL_Q_STRIDE=[[1, 1, 2, 2], [3, 1, 2, 2], [14, 1, 2, 2]], DROPOUT_RATE=0.0),
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "mvit", "MODEL_NAME": "MViT", "DROPOUT_RATE": 0.5},
        "TRAIN": {"BATCH_SIZE": 16},
        "RNG_SEED": 0,
    },
    # configs/masked_ssl/k400_VIT_B_16x4_FT.yaml (ViT-B: 2x16x16 patches, separable positions, mean readout)
    "VIT_B_16x4_FT": {
        "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": {"ZERO_DECAY_POS_CLS": False, "SEP_POS_EMBED": True, "PATCH_KERNEL": [2, 16, 16],
                 "PATCH_STRIDE": [2, 16, 16], "PATCH_PADDING": [0, 0, 0], "EMBED_DIM": 768, "NUM_HEADS": 12,
                 "MLP_RATIO": 4.0, "QKV_BIAS": True, "NORM": "layernorm", "DEPTH": 12, "MODE": "conv",
                 "DROPPATH_RATE": 0.1, "LAYER_SCALE_INIT_VALUE": 0.0, "USE_MEAN_POOLING": True,
                 "HEAD_INIT_SCALE": 0.001},
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "mvit", "MODEL_NAME": "MViT", "DROPOUT_RATE": 0.3},
        "TRAIN": {"BATCH_SIZE": 1},
        "RNG_SEED": 0,
    },
    # configs/masked_ssl/k400_MVITv2_S_16x4_FT.yaml (MaskFeat fine-tuning: MViTv2-S with the mean readout)
    "MVITv2_S_16x4_FT": {
        "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
        "MVIT": dict(_MVIT_B_POOL, DEPTH=16, NUM_HEADS=1, EMBED_DIM=96, PATCH_KERNEL=[3, 7, 7], PATCH_STRIDE=[2, 4, 4],
                     PATCH_PADDING=[1, 3, 3], ZERO_DECAY_POS_CLS=False, QKV_BIAS=True,
                     POOL_Q_STRIDE=[[i, 1, 2, 2] if i in (1, 3, 14) else [i, 1, 1, 1] for i in range(16)],
                     CLS_EMBED_ON=True, USE_ABS_POS=False, SEP_POS_EMBED=True, REL_POS_SPATIAL=True,
                     REL_POS_TEMPORAL=True, RESIDUAL_POOLING=True, MODE="conv", DROPPATH_RATE=0.1,
                     LAYER_SCALE_INIT_VALUE=0.0, USE_MEAN_POOLING=True, HEAD_INIT_SCALE=0.001),
        "MODEL": {"NUM_CLASSES": 400, "ARCH": "mvit", "MODEL_NAME": "MViT", "DROPOUT_RATE": 0.0},
        "TRAIN": {"BATCH_SIZE": 16},
        "RNG_SEED": 0,
    },
})
# configs/masked_ssl/k400_VIT_{B,L,H}_16x4_MAE_PT.yaml (MAE pre-training: 90 % of the 2x16x16 patches removed, a 4-block
# 512-wide decoder predicting normalised pixels)
_VIT_MAE = {
    "DATA": {"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3]},
    "MVIT": {"ZERO_DECAY_POS_CLS": False, "SEP_POS_EMBED": True, "PATCH_KERNEL": [2, 16, 16], "PATCH_STRIDE": [2, 16, 16],
             "PATCH_PADDING": [0, 0, 0], "EMBED_DIM": 768, "NUM_HEADS": 12, "MLP_RATIO": 4.0, "QKV_BIAS": True,
             "NORM": "layernorm", "DEPTH": 12, "DROPPATH_RATE": 0.0, "MODE": "conv", "CLS_EMBED_ON": True},
    "MASK": {"ENABLE": True, "MAE_ON": True, "MAE_RND_MASK": True, "PRETRAIN_DEPTH": [11], "HEAD_TYPE": "separate_xformer",
             "DECODER_DEPTH": 4, "DECODER_EMBED_DIM": 512},
    "AUG": {"MASK_RATIO": 0.9},
    "MODEL": {"NUM_CLASSES": 400, "ARCH": "maskmvit", "MODEL_NAME": "MaskMViT", "LOSS_FUNC": "multi_mse",
              "DROPOUT_RATE": 0.0},
    "TRAIN": {"BATCH_SIZE": 64},
    "RNG_SEED": 0,
}
_PRESETS.update({
    "VIT_B_16x4_MAE_PT": _VIT_MAE,
    "VIT_L_16x4_MAE_PT": dict(copy.deepcopy(_VIT_MAE), MVIT=dict(_VIT_MAE["MVIT"], EMBED_DIM=1024, NUM_HEADS=16, DEPTH=24),
                              MASK=dict(_VIT_MAE["MASK"], PRETRAIN_DEPTH=[23]), TRAIN={"BATCH_SIZE": 32}),
    "VIT_H_16x4_MAE_PT": dict(copy.deepcopy(_VIT_MAE), MVIT=dict(_VIT_MAE["MVIT"], EMBED_DIM=1280, NUM_HEADS=16, DEPTH=32),
                              MASK=dict(_VIT_MAE["MASK"], PRETRAIN_DEPTH=[31]), TRAIN={"BATCH_SIZE": 32}),
})
# ImageNet recipes (PATCH_2D: one-frame [B, 3, H, W] inputs)
_IN1K_DATA = {"NUM_FRAMES": 1, "TRAIN_CROP_SIZE": 224, "TEST_CROP_SIZE": 224, "INPUT_CHANNEL_NUM": [3],
              "MEAN": [0.485, 0.456, 0.406], "STD": [0.229, 0.224, 0.225]}
_IN1K_MODEL = {"NUM_CLASSES": 1000, "ARCH": "mvit", "MODEL_NAME": "MViT", "LOSS_FUNC": "soft_cross_entropy",
               "DROPOUT_RATE": 0.0}
# configs/ImageNet/MVITv2_T.yaml (no cls token, spatial rel-pos, norm-then-mean readout)
_MVITv2_T = {
    "DATA": _IN1K_DATA,
    "MVIT": {"PATCH_2D": True, "ZERO_DECAY_POS_CLS": False, "MODE": "conv", "CLS_EMBED_ON": False,
             "PATCH_KERNEL": [7, 7], "PATCH_STRIDE": [4, 4], "PATCH_PADDING": [3, 3], "EMBED_DIM": 96, "NUM_HEADS": 1,
             "MLP_RATIO": 4.0, "QKV_BIAS": True, "DROPPATH_RATE": 0.1, "DEPTH": 10, "NORM": "layernorm",
             "DIM_MUL": [[1, 2.0], [3, 2.0], [8, 2.0]], "HEAD_MUL": [[1, 2.0], [3, 2.0], [8, 2.0]],
             "POOL_KVQ_KERNEL": [1, 3, 3],
             "POOL_KV_STRIDE": [[0, 1, 4, 4], [1, 1, 2, 2], [2, 1, 2, 2]] + [[i, 1, 1, 1] for i in range(3, 10)],
             "POOL_Q_STRIDE": [[i, 1, 2, 2] if i in (1, 3, 8) else [i, 1, 1, 1] for i in range(10)],
             "RESIDUAL_POOLING": True, "USE_ABS_POS": False, "REL_POS_SPATIAL": True, "DIM_MUL_IN_ATT": True},
    "MODEL": _IN1K_MODEL,
    "RNG_SEED": 0,
}
_PRESETS.update({
    "MVITv2_T": _MVITv2_T,
    # configs/ImageNet/MVITv2_S.yaml (MViTv2-T at depth 16, the last stage from block 14)
    "MVITv2_S": dict(copy.deepcopy(_MVITv2_T), MVIT=dict(
        _MVITv2_T["MVIT"], DEPTH=16, DIM_MUL=[[1, 2.0], [3, 2.0], [14, 2.0]], HEAD_MUL=[[1, 2.0], [3, 2.0], [14, 2.0]],
        POOL_KV_STRIDE=[[0, 1, 4, 4], [1, 1, 2, 2], [2, 1, 2, 2]] + [[i, 1, 1, 1] for i in range(3, 16)],
        POOL_Q_STRIDE=[[i, 1, 2, 2] if i in (1, 3, 14) else [i, 1, 1, 1] for i in range(16)])),
    # configs/masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml (ViT-B/16: 196 patches + cls, a joint pos_embed, mean readout)
    "VIT_B_IN1K_FT": {
        "DATA": _IN1K_DATA,
        "MVIT": {"PATCH_2D": True, "ZERO_DECAY_POS_CLS": False, "MODE": "conv", "CLS_EMBED_ON": True,
                 "PATCH_KERNEL": [16, 16], "PATCH_STRIDE": [16, 16], "PATCH_PADDING": [0, 0], "EMBED_DIM": 768,
                 "NUM_HEADS": 12, "MLP_RATIO": 4.0, "QKV_BIAS": True, "DROPPATH_RATE": 0.1,
                 "LAYER_SCALE_INIT_VALUE": 0.0, "DEPTH": 12, "NORM": "layernorm", "HEAD_INIT_SCALE": 0.001,
                 "USE_MEAN_POOLING": True},
        "MODEL": _IN1K_MODEL,
        "RNG_SEED": 0,
    },
})
# Non-local recipes (Wang et al., arXiv:1711.07971): the same backbones with Non-local blocks after res3 blocks 1, 3 and
# res4 blocks 1, 3, 5 (slow pathway only for SlowFast); NONLOCAL.POOL keeps its default [1, 2, 2]
_NLN_R50 = {"LOCATION": [[[]], [[1, 3]], [[1, 3, 5]], [[]]], "GROUP": [[1], [1], [1], [1]]}
_PRESETS.update({
    # configs/Kinetics/C2D_NLN_8x8_R50.yaml
    "C2D_NLN_8x8_R50": dict(copy.deepcopy(_PRESETS["C2D_8x8_R50"]), NONLOCAL=dict(_NLN_R50, INSTANTIATION="softmax")),
    # configs/Kinetics/I3D_NLN_8x8_R50.yaml
    "I3D_NLN_8x8_R50": dict(copy.deepcopy(_PRESETS["I3D_8x8_R50"]), NONLOCAL=dict(_NLN_R50, INSTANTIATION="softmax")),
    # configs/Kinetics/SLOW_NLN_8x8_R50.yaml
    "SLOW_NLN_8x8_R50": dict(copy.deepcopy(_PRESETS["SLOW_8x8_R50"]),
                             NONLOCAL=dict(_NLN_R50, INSTANTIATION="dot_product")),
    # configs/Kinetics/SLOWFAST_NLN_8x8_R50.yaml (FUSION_KERNEL_SZ 5, not the 7 of SLOWFAST_8x8_R50.yaml)
    "SLOWFAST_NLN_8x8_R50": dict(
        copy.deepcopy(_PRESETS["SLOWFAST_8x8_R50"]),
        SLOWFAST={"ALPHA": 4, "BETA_INV": 8, "FUSION_CONV_CHANNEL_RATIO": 2, "FUSION_KERNEL_SZ": 5},
        NONLOCAL={"LOCATION": [[[], []], [[1, 3], []], [[1, 3, 5], []], [[], []]],
                  "GROUP": [[1, 1], [1, 1], [1, 1], [1, 1]], "INSTANTIATION": "dot_product"}),
})


def get_cfg(preset: str | None = None, **overrides) -> Cfg:
    """Defaults (+ a named preset) (+ nested overrides, e.g. ``MODEL={"DROPOUT_RATE": 0.0}``)."""
    cfg = Cfg(copy.deepcopy(_DEFAULTS))
    if preset is not None:
        if preset not in _PRESETS:
            raise KeyError(f"unknown preset {preset!r}; have {sorted(_PRESETS)}")
        cfg.merge(copy.deepcopy(_PRESETS[preset]))
    cfg.merge(overrides)
    return cfg


def presets():
    return sorted(_PRESETS)


def nsplit_of(cfg) -> int:
    """Operand precision mode: 3 = split-bf16 (fp32-class, parity mode), 1 = plain bf16 (fast mode)."""
    b = getattr(cfg, "B200", None)
    if b is None:
        return 3
    return int(getattr(b, "NSPLIT", 3)) if not isinstance(b, dict) else int(b.get("NSPLIT", 3))
