"""TEST INFRASTRUCTURE: the engine config of a golden fixture (tests/golden/*.pt): the preset its yaml names plus the
model overrides it was generated with."""
from __future__ import annotations

PRESET = {"Kinetics/SLOWFAST_8x8_R50.yaml": "SLOWFAST_8x8_R50", "Kinetics/C2D_8x8_R50.yaml": "C2D_8x8_R50",
          "Kinetics/SLOW_8x8_R50.yaml": "SLOW_8x8_R50", "Kinetics/I3D_8x8_R50.yaml": "I3D_8x8_R50",
          "Kinetics/MVITv2_S_16x4.yaml": "MVITv2_S_16x4", "Kinetics/MVITv2_B_32x3.yaml": "MVITv2_B_32x3",
          "Kinetics/X3D_M.yaml": "X3D_M",
          "masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml": "MVITv2_S_16x4_MaskFeat_PT"}


def engine_cfg(gold, nsplit=3):
    from slowfast_b200.config import get_cfg
    preset = PRESET[gold["yaml"]]
    if gold["case"].startswith("maskfeat_b"):   # composed config (BASELINE config 5, SURVEY.md section 3.5)
        preset = "MVITv2_B_32x3_MaskFeat_PT"
    cfg = get_cfg(preset, B200={"NSPLIT": nsplit})
    ov = gold["overrides"]
    for k, v in zip(ov[0::2], ov[1::2]):
        sec, key = k.split(".")
        if sec == "AUG":
            continue  # loader-side keys (mask window) are not read by the model
        cfg[sec][key] = v
    return cfg
