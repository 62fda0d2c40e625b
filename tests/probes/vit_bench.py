"""GPU probe: training throughput of the absolute-position / mean-readout MViT recipes at 224^2.

Recipes: ViT-B 16x4 (MaskFeat fine-tuning recipe), MViTv1-B 16x4 and MViTv2-S fine-tuning.  For each it times, in one
process and alternating, SGD training steps (forward, cross-entropy, backward, torch.optim.SGD step) of
  * the engine model in parity mode (split-bf16) and fast mode (bf16), CUDA graphs on;
  * the unmodified reference model (oracle/_ref, fp32 PyTorch) on the same GPU, when build() installed it.
Every leg warms up, then runs for at least --seconds of wall time ended by a device synchronise; all legs are repeated
--repeats times, alternating their order, to show the spread.  A separate torch.profiler run of the ViT-B parity step
(graphs off, so every kernel is listed) gives the share of CUDA time spent in the attention score / output GEMMs
(gemm_batched_kernel) and the softmax kernels.  Prints one JSON object (clips/s and peak memory per leg, the profile
shares, GPU name and power limit).

    python tests/probes/vit_bench.py [--batch 8] [--seconds 3] [--repeats 2] [--out vit_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

RECIPES = {
    # name: (engine preset, reference yaml)
    "vit_b_16x4": ("VIT_B_16x4_FT", "masked_ssl/k400_VIT_B_16x4_FT.yaml"),
    "mvit_b_16x4": ("MVIT_B_16x4_CONV", "Kinetics/MVIT_B_16x4_CONV.yaml"),
    "mvitv2_s_16x4_ft": ("MVITv2_S_16x4_FT", "masked_ssl/k400_MVITv2_S_16x4_FT.yaml"),
}


def gpu_info() -> dict:
    """Card name and power limit (read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"gpu": None, "power_limit": None, "query_error": repr(e)}


def build_leg(recipe: str, kind: str, batch: int, dev, graphs: bool = True):
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
        cfg = get_cfg(preset, MODEL={"DROPOUT_RATE": 0.0},
                      B200={"NSPLIT": 3 if kind == "parity" else 1, "CUDA_GRAPH": graphs})
        model = B200MViT(cfg)
    torch.manual_seed(0)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 5))
    model = model.to(dev).train()
    inputs = [t.to(dev) for t in TO.synthetic_inputs(cfg, batch, 11)]
    labels = torch.randint(0, cfg.MODEL.NUM_CLASSES, (batch,), generator=torch.Generator().manual_seed(12)).to(dev)
    return model, inputs, labels


def _stepper(model, inputs, labels):
    import torch
    opt = torch.optim.SGD(model.parameters(), lr=1e-5, momentum=0.9)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.cross_entropy(model([x for x in inputs]), labels)
        loss.backward()
        opt.step()
    return step


def time_leg(model, inputs, labels, seconds: float, warmup: int = 4) -> dict:
    import torch
    step = _stepper(model, inputs, labels)
    for _ in range(warmup):          # (the engine captures its CUDA graphs on the third call)
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    steps, t0 = 0, time.perf_counter()
    while True:
        step()
        steps += 1
        if steps % 2 == 0:
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if dt >= seconds:
                break
    batch = inputs[0].shape[0]
    return {"clips_per_s": round(steps * batch / dt, 2), "steps": steps, "seconds": round(dt, 3),
            "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def attention_share(batch: int, dev, steps: int = 3) -> dict:
    """CUDA-time share of gemm_batched_kernel and the softmax kernels in the ViT-B parity step (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    model, inputs, labels = build_leg("vit_b_16x4", "parity", batch, dev, graphs=False)
    step = _stepper(model, inputs, labels)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    total, bgemm, soft = 0.0, 0.0, 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += t
        if "gemm_batched_kernel" in ev.key:
            bgemm += t
        elif "softmax_relpos" in ev.key:
            soft += t
    del model, inputs, labels
    return {"profiled_steps": steps, "cuda_ms_per_step": round(total / steps / 1e3, 2),
            "gemm_batched_share": round(bgemm / total, 3), "softmax_share": round(soft / total, 3)}


def main() -> None:
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--recipes", default=",".join(RECIPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vit_bench needs a CUDA device")
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    from oracle import refshim
    kinds = ["parity", "fast"] + (["reference"] if refshim.reference_available() else [])
    result = dict(gpu_info(), batch=args.batch, crop=224, frames=16, seconds_per_leg=args.seconds,
                  torch=torch.__version__, legs={})
    for rep in range(args.repeats):
        for recipe in args.recipes.split(","):
            order = kinds if rep % 2 == 0 else list(reversed(kinds))
            for kind in order:
                model, inputs, labels = build_leg(recipe, kind, args.batch, dev)
                r = time_leg(model, inputs, labels, args.seconds)
                result["legs"].setdefault(f"{recipe}/{kind}", []).append(r)
                print(f"[rep {rep}] {recipe}/{kind}: {r}", file=sys.stderr, flush=True)
                del model, inputs, labels
                gc.collect()
                torch.cuda.empty_cache()
    summary = {}
    for leg, rs in result["legs"].items():
        v = [r["clips_per_s"] for r in rs]
        summary[leg] = {"clips_per_s_median": sorted(v)[len(v) // 2], "min": min(v), "max": max(v),
                        "peak_mem_gib": max(r["peak_mem_gib"] for r in rs)}
    result["summary"] = summary
    if "vit_b_16x4" in args.recipes.split(","):
        result["vit_b_profile"] = attention_share(args.batch, dev)
        print(f"profile: {result['vit_b_profile']}", file=sys.stderr, flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
