"""GPU probe: training throughput of the ImageNet recipes at 224^2 (images/s and peak memory).

Recipes: MViTv2-T, MViTv2-S (no cls token, spatial rel-pos, norm-then-mean readout) and in1k ViT-B/16 (joint pos_embed,
mean readout).  For each it times, in one process and alternating the leg order between repeats, SGD training steps
(forward, cross-entropy, backward, torch.optim.SGD step) of
  * the engine model in parity mode (split-bf16) and fast mode (bf16), CUDA graphs on;
  * the unmodified reference model (oracle/_ref, fp32 PyTorch, TF32 off) on the same GPU, when build() installed it.
Every leg warms up, then runs for at least --seconds of wall time ended by a device synchronise.  Prints one JSON object
(images/s and peak memory per leg, GPU name and power limit).

    python tests/probes/image_bench.py [--batch 64] [--seconds 3] [--repeats 3] [--out image_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "probes"))

from vit_bench import gpu_info, time_leg  # noqa: E402

RECIPES = {
    # name: (engine preset, reference yaml)
    "mvitv2_t": ("MVITv2_T", "ImageNet/MVITv2_T.yaml"),
    "mvitv2_s": ("MVITv2_S", "ImageNet/MVITv2_S.yaml"),
    "vit_b_in1k": ("VIT_B_IN1K_FT", "masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml"),
}


def build_leg(recipe: str, kind: str, batch: int, dev):
    """(model, inputs, labels) of one leg; kind = parity | fast | reference."""
    import torch
    from oracle import torch_oracle as TO
    preset, yaml = RECIPES[recipe]
    if kind == "reference":
        from oracle import refshim
        cfg = refshim.load_cfg(yaml, ["MODEL.DROPOUT_RATE", 0.0])
        model = refshim.build_reference_model(cfg)
    else:
        from slowfast_b200.config import get_cfg
        from slowfast_b200.nets.mvit import B200MViT
        cfg = get_cfg(preset, MODEL={"DROPOUT_RATE": 0.0}, B200={"NSPLIT": 3 if kind == "parity" else 1})
        model = B200MViT(cfg)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 5))
    model = model.to(dev).train()
    crop = cfg.DATA.TRAIN_CROP_SIZE
    inputs = [torch.randn(batch, 3, crop, crop, generator=torch.Generator().manual_seed(11)).to(dev)]
    labels = torch.randint(0, cfg.MODEL.NUM_CLASSES, (batch,), generator=torch.Generator().manual_seed(12)).to(dev)
    return model, inputs, labels


def main() -> None:
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--recipes", default=",".join(RECIPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_bench needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    from oracle import refshim
    kinds = ["parity", "fast"] + (["reference"] if refshim.reference_available() else [])
    result = dict(gpu_info(), batch=args.batch, crop=224, seconds_per_leg=args.seconds, torch=torch.__version__, legs={})
    for rep in range(args.repeats):
        for recipe in args.recipes.split(","):
            for kind in (kinds if rep % 2 == 0 else list(reversed(kinds))):
                model, inputs, labels = build_leg(recipe, kind, args.batch, dev)
                r = time_leg(model, inputs, labels, args.seconds)
                r["images_per_s"] = r.pop("clips_per_s")
                result["legs"].setdefault(f"{recipe}/{kind}", []).append(r)
                print(f"[rep {rep}] {recipe}/{kind}: {r}", file=sys.stderr, flush=True)
                del model, inputs, labels
                gc.collect()
                torch.cuda.empty_cache()
    summary = {}
    for leg, rs in result["legs"].items():
        v = sorted(r["images_per_s"] for r in rs)
        summary[leg] = {"images_per_s_median": v[len(v) // 2], "min": v[0], "max": v[-1],
                        "peak_mem_gib": max(r["peak_mem_gib"] for r in rs)}
    result["summary"] = summary
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
