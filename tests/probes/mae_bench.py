"""GPU probe: training throughput of the MAE pre-training recipes (ViT-B / ViT-L, 16x224^2, 90 % of the patches removed).

The recipe's per-GPU batch is 8 videos x TRAIN_CROP_NUM_TEMPORAL 4 = 32 clips.  For each recipe it times, in one process
and alternating, AdamW training steps (forward, MSE loss against the pixel targets, backward, torch.optim.AdamW step) of
  * the engine model in parity mode (split-bf16) and fast mode (bf16), CUDA graphs on;
  * the unmodified reference model (oracle/_ref, fp32 PyTorch) on the same GPU, when build() installed it.
Every leg warms up, then runs for at least --seconds of wall time ended by a device synchronise; all legs are repeated
--repeats times, alternating their order.  A separate torch.profiler run of the ViT-B parity step (graphs off) lists the
CUDA-time share of the batched attention GEMMs and the softmax kernels.  Prints one JSON object (clips/s and peak memory
per leg, the profile, GPU name and power limit).

    python tests/probes/mae_bench.py [--batch 32] [--seconds 3] [--repeats 3] [--out mae_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "probes"))

from vit_bench import gpu_info  # noqa: E402

RECIPES = {
    "vit_b_mae": ("VIT_B_16x4_MAE_PT", "masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml"),
    "vit_l_mae": ("VIT_L_16x4_MAE_PT", "masked_ssl/k400_VIT_L_16x4_MAE_PT.yaml"),
}


def build_leg(recipe: str, kind: str, batch: int, dev, graphs: bool = True):
    import torch
    from oracle import torch_oracle as TO
    preset, yaml = RECIPES[recipe]
    if kind == "reference":
        from oracle import refshim
        cfg = refshim.load_cfg(yaml)
        model = refshim.build_reference_model(cfg)
    else:
        from slowfast_b200.config import get_cfg
        from slowfast_b200.nets.maskfeat import B200MaskMViT
        cfg = get_cfg(preset, B200={"NSPLIT": 3 if kind == "parity" else 1, "CUDA_GRAPH": graphs})
        model = B200MaskMViT(cfg)
    torch.manual_seed(0)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 5))
    model = model.to(dev).train()
    return model, TO.synthetic_inputs(cfg, batch, 11)[0].to(dev)


def _stepper(model, x):
    import torch
    opt = torch.optim.AdamW(model.parameters(), lr=1e-5)

    def step():
        opt.zero_grad(set_to_none=True)
        preds, labels = model([x])
        torch.nn.functional.mse_loss(preds[0], labels[0][0]).backward()
        opt.step()
    return step


def time_leg(model, x, seconds: float, warmup: int = 4) -> dict:
    import torch
    step = _stepper(model, x)
    for _ in range(warmup):          # (the engine captures its CUDA graphs on the third call)
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    steps, t0 = 0, time.perf_counter()
    while True:
        step()
        steps += 1
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= seconds and steps >= 2:
            break
    return {"clips_per_s": round(steps * x.shape[0] / dt, 2), "steps": steps, "seconds": round(dt, 3),
            "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def profile(batch: int, dev, steps: int = 2) -> dict:
    """CUDA-time shares of the ViT-B MAE parity step (torch.profiler, graphs off)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as prof_
    model, x = build_leg("vit_b_mae", "parity", batch, dev, graphs=False)
    step = _stepper(model, x)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with prof_(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    rows = []
    total = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += t
        rows.append((t, ev.key))
    rows.sort(reverse=True)
    groups = {"gemm_batched (attention)": "gemm_batched_kernel", "softmax": "softmax_relpos",
              "conv_igemm (Linear fwd / dgrad)": "igemm", "conv_wgrad (Linear wgrad)": "wgrad",
              "layernorm": "ln_", "mae kernels": ("mae_", "assemble", "scatter", "gather", "pixel_targets")}
    shares = {}
    for name, pat in groups.items():
        pats = pat if isinstance(pat, tuple) else (pat,)
        shares[name] = round(sum(t for t, k in rows if any(p in k for p in pats)) / total, 3)
    del model, x
    return {"profiled_steps": steps, "cuda_ms_per_step": round(total / steps / 1e3, 2), "shares": shares,
            "top": [(k[:80], round(t / steps / 1e3, 2)) for t, k in rows[:12]]}


def main() -> None:
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--recipes", default=",".join(RECIPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mae_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    from oracle import refshim
    kinds = ["parity", "fast"] + (["reference"] if refshim.reference_available() else [])
    result = dict(gpu_info(), batch=args.batch, crop=224, frames=16, seconds_per_leg=args.seconds,
                  torch=torch.__version__, legs={})
    for rep in range(args.repeats):
        for recipe in args.recipes.split(","):
            order = kinds if rep % 2 == 0 else list(reversed(kinds))
            for kind in order:
                model, x = build_leg(recipe, kind, args.batch, dev)
                r = time_leg(model, x, args.seconds)
                result["legs"].setdefault(f"{recipe}/{kind}", []).append(r)
                print(f"[rep {rep}] {recipe}/{kind}: {r}", file=sys.stderr, flush=True)
                del model, x
                gc.collect()
                torch.cuda.empty_cache()
    summary = {}
    for leg, rs in result["legs"].items():
        v = [r["clips_per_s"] for r in rs]
        summary[leg] = {"clips_per_s_median": sorted(v)[len(v) // 2], "min": min(v), "max": max(v),
                        "peak_mem_gib": max(r["peak_mem_gib"] for r in rs)}
    result["summary"] = summary
    if "vit_b_mae" in args.recipes.split(","):
        result["vit_b_mae_profile"] = profile(args.batch, dev)
        print(f"profile: {result['vit_b_mae_profile']}", file=sys.stderr, flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
