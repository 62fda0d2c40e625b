"""GPU probe: one MoCo pre-training step of configs/contrastive_ssl/MoCo_SlowR50_8x8.yaml at the recipe's per-GPU shape
(8 clips of 8 x 224^2, TRAIN_CROP_NUM_TEMPORAL 4, CONTRASTIVE.SEQUENTIAL: 4 key-encoder forwards, then forward + backward
per query clip, the enqueue, and a torch.optim.SGD step), full queue (65536) and kNN memory.

Legs, alternating in one process:
  * the engine (B200ContrastiveModel), parity mode (split-bf16) and fast mode (bf16), CUDA graphs on;
  * the unmodified reference ContrastiveModel (oracle/_ref, fp32 PyTorch) on the same GPU, when build() installed it.
Every leg warms up, then runs for at least --seconds of wall time ended by a device synchronise.  Also times the
key-encoder momentum update alone (CUDA events over 50 calls): the engine's one in-place launch against the reference's
per-parameter `p.data = q * (1 - m) + p * m`.  Prints one JSON object with the GPU name and power limit.

    python tests/probes/moco_bench.py [--seconds 5] [--repeats 2] [--out moco_bench.json]
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
sys.path.insert(0, str(Path(__file__).resolve().parent))

from nln_bench import gpu_info  # noqa: E402

YAML = "contrastive_ssl/MoCo_SlowR50_8x8.yaml"
BATCH, CROPS = 8, 4


def build_leg(kind: str, dev):
    import torch
    from oracle import refshim
    from oracle import torch_oracle as TO
    cfg = refshim.load_cfg(YAML, ["NUM_GPUS", 1, "TRAIN.BATCH_SIZE", BATCH])
    if kind == "reference":
        model = refshim.build_reference_model(cfg)
    else:
        from slowfast_b200.nets.contrastive import B200ContrastiveModel
        cfg["B200"] = {"NSPLIT": 3 if kind == "parity" else 1, "CUDA_GRAPH": True}
        torch.manual_seed(cfg.RNG_SEED)
        model = B200ContrastiveModel(cfg)
    sd = model.state_dict()
    sd.update({k: v for k, v in TO.fixture_state(sd, 5).items() if k.startswith("backbone")})
    model.load_state_dict(sd)
    model = model.to(dev).train()
    clips = [[t.to(dev) for t in TO.synthetic_inputs(cfg, BATCH, 20 + i)] for i in range(CROPS)]
    return cfg, model, clips


def run_step(model, cfg, clips, opt, epoch):
    import torch
    from slowfast.models.contrastive import contrastive_forward

    class _NoScale:
        @staticmethod
        def scale(loss):
            return loss

    index = torch.arange(BATCH, device=clips[0][0].device)
    tm = torch.zeros(BATCH, CROPS, 1, device=clips[0][0].device)
    opt.zero_grad(set_to_none=True)
    contrastive_forward(model, cfg, clips, index, tm, epoch, _NoScale())
    opt.step()


def time_leg(kind, dev, seconds):
    import torch
    cfg, model, clips = build_leg(kind, dev)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-4, momentum=0.9)
    for i in range(3):
        run_step(model, cfg, clips, opt, 0.01 * i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    steps, t0 = 0, time.perf_counter()
    while True:
        run_step(model, cfg, clips, opt, 0.01 * steps)
        steps += 1
        if steps >= 3 and time.perf_counter() - t0 >= seconds:
            torch.cuda.synchronize()
            if time.perf_counter() - t0 >= seconds:
                break
    dt = time.perf_counter() - t0
    # the momentum update alone
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        model._update_history()
    e0.record()
    for _ in range(50):
        model._update_history()
    e1.record()
    torch.cuda.synchronize()
    out = {"steps": steps, "seconds": round(dt, 3), "clips_per_s": round(steps * BATCH / dt, 2),
           "step_ms": round(1e3 * dt / steps, 2), "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "momentum_update_ms": round(e0.elapsed_time(e1) / 50, 4)}
    del model, clips, opt
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main() -> None:
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=5.0)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moco_bench needs a CUDA device")
    from oracle import refshim
    if not refshim.reference_available():
        raise SystemExit("moco_bench needs the reference tree (build() copies it into oracle/_ref)")
    refshim.install()
    dev = torch.device("cuda:0")
    kinds = ["parity", "fast"] + ([] if args.no_reference else ["reference"])
    result = dict(gpu_info(), seconds_per_leg=args.seconds, torch=torch.__version__, batch=BATCH, crops=CROPS, legs={})
    for rep in range(args.repeats):
        for kind in (kinds if rep % 2 == 0 else list(reversed(kinds))):
            r = time_leg(kind, dev, args.seconds)
            result["legs"].setdefault(kind, []).append(r)
            print(f"[rep {rep}] {kind}: {r}", file=sys.stderr, flush=True)
    result["summary"] = {k: {"clips_per_s_runs": [r["clips_per_s"] for r in rs],
                             "peak_mem_gib": max(r["peak_mem_gib"] for r in rs),
                             "momentum_update_ms": min(r["momentum_update_ms"] for r in rs)}
                         for k, rs in result["legs"].items()}
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
