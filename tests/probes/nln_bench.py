"""GPU probe: training throughput of the Non-local recipes (I3D-NLN-8x8-R50, SlowFast-NLN-8x8-R50) at 224^2.

For each recipe it times, in one process and alternating, SGD training steps (forward, cross-entropy, backward,
torch.optim.SGD step) of
  * the engine model with its Non-local blocks, parity mode (split-bf16) and fast mode (bf16), CUDA graphs on;
  * the same engine model without Non-local blocks (NONLOCAL.LOCATION emptied): the difference is the blocks' cost;
  * the unmodified reference model (oracle/_ref, fp32 PyTorch) on the same GPU, when build() installed it.
Every leg warms up, then runs for at least --seconds of wall time ended by a device synchronise; all legs are repeated
--repeats times to show the spread.  Prints one JSON object (clips/s and peak memory per leg, GPU name and power limit).

    python tests/probes/nln_bench.py [--batch 8] [--seconds 3] [--repeats 2] [--out nln_bench.json]
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
    "i3d_nln_8x8_r50": ("I3D_NLN_8x8_R50", "Kinetics/I3D_NLN_8x8_R50.yaml"),
    "slowfast_nln_8x8_r50": ("SLOWFAST_NLN_8x8_R50", "Kinetics/SLOWFAST_NLN_8x8_R50.yaml"),
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


def build_leg(recipe: str, kind: str, batch: int, dev):
    """(model, inputs, labels) of one leg; kind = nl_parity | nl_fast | base_parity | base_fast | reference."""
    import torch
    from oracle import torch_oracle as TO
    preset, yaml = RECIPES[recipe]
    if kind == "reference":
        from oracle import refshim
        cfg = refshim.load_cfg(yaml, ["MODEL.DROPOUT_RATE", 0.0])
        model = refshim.build_reference_model(cfg)
    else:
        from slowfast_b200.config import get_cfg
        over = dict(MODEL={"DROPOUT_RATE": 0.0}, B200={"NSPLIT": 3 if kind.endswith("parity") else 1, "CUDA_GRAPH": True})
        if kind.startswith("base"):
            over["NONLOCAL"] = {"LOCATION": [[[] for _ in p] for p in get_cfg(preset).NONLOCAL.LOCATION]}
        cfg = get_cfg(preset, **over)
        if cfg.MODEL.MODEL_NAME == "SlowFast":
            from slowfast_b200.nets.resnet import B200SlowFast as M
        else:
            from slowfast_b200.nets.resnet_single import B200ResNet as M
        model = M(cfg)
    torch.manual_seed(0)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 5))
    model = model.to(dev).train()
    inputs = [t.to(dev) for t in TO.synthetic_inputs(cfg, batch, 11)]
    labels = torch.randint(0, cfg.MODEL.NUM_CLASSES, (batch,), generator=torch.Generator().manual_seed(12)).to(dev)
    return model, inputs, labels


def time_leg(model, inputs, labels, seconds: float, warmup: int = 4) -> dict:
    import torch
    opt = torch.optim.SGD(model.parameters(), lr=1e-5, momentum=0.9)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.cross_entropy(model([x for x in inputs]), labels)
        loss.backward()
        opt.step()

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
        raise SystemExit("nln_bench needs a CUDA device")
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    from oracle import refshim
    kinds = ["nl_parity", "base_parity", "nl_fast", "base_fast"] + (["reference"] if refshim.reference_available() else [])
    result = dict(gpu_info(), batch=args.batch, crop=224, seconds_per_leg=args.seconds, torch=torch.__version__,
                  legs={})
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
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
