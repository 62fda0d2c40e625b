"""GPU probe: SlowFast-8x8-R50 training throughput at the long-cycle base shapes of the stepwise-multigrid recipe
(configs/Kinetics/SLOWFAST_8x8_R50_stepwise_multigrid.yaml: 8 clips per GPU, MULTIGRID.BN_BASE_SIZE 8).

Shapes, as (batch, fast frames, crop, NUM_SPLITS): (64, 8, 158, 8), (32, 16, 158, 4), (16, 16, 224, 2), (8, 32, 224, plain BN).
For each shape it times, in one process and alternating, SGD training steps (forward, cross-entropy, backward,
torch.optim.SGD step) of
  * the engine with sub-batch BN, parity mode (split-bf16) and fast mode (bf16), CUDA graphs on;
  * the engine at the same shape with plain BN: the difference is the cost of the per-split statistics pass;
  * the unmodified reference model (oracle/_ref, fp32 PyTorch, its own SubBatchNorm3d) on the same GPU, when build()
    installed it.
The short cycle's adaptive head pool is on (MULTIGRID.SHORT_CYCLE), as in the recipe.  Every leg warms up, then runs for
at least --seconds of wall time ended by a device synchronise; all legs are repeated --repeats times to show the spread.
Prints one JSON object (clips/s and peak memory per leg, GPU name and power limit read in the same process).

    python tests/probes/subbn_bench.py [--seconds 3] [--repeats 2] [--shapes 0,1,2,3] [--out subbn_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from nln_bench import gpu_info, time_leg  # noqa: E402  (same timing loop and card query)

SHAPES = [(64, 8, 158, 8), (32, 16, 158, 4), (16, 16, 224, 2), (8, 32, 224, 1)]


def build_leg(shape, kind: str, dev):
    """(model, inputs, labels); kind = sub_parity | plain_parity | sub_fast | plain_fast | reference."""
    import torch
    from oracle import torch_oracle as TO
    batch, frames, crop, splits = shape
    sub = splits > 1 and not kind.startswith("plain")
    if kind == "reference":
        from oracle import refshim
        over = ["MODEL.DROPOUT_RATE", 0.0, "DATA.NUM_FRAMES", frames, "DATA.TRAIN_CROP_SIZE", crop,
                "MULTIGRID.SHORT_CYCLE", True]
        if sub:
            over += ["BN.NORM_TYPE", "sub_batchnorm", "BN.NUM_SPLITS", splits]
        cfg = refshim.load_cfg("Kinetics/SLOWFAST_8x8_R50.yaml", over)
        model = refshim.build_reference_model(cfg)
    else:
        from slowfast_b200.config import get_cfg
        from slowfast_b200.nets.resnet import B200SlowFast
        bn = {"NORM_TYPE": "sub_batchnorm", "NUM_SPLITS": splits} if sub else {"NORM_TYPE": "batchnorm"}
        cfg = get_cfg("SLOWFAST_8x8_R50", MODEL={"DROPOUT_RATE": 0.0}, DATA={"NUM_FRAMES": frames, "TRAIN_CROP_SIZE": crop},
                      MULTIGRID={"SHORT_CYCLE": True}, BN=bn,
                      B200={"NSPLIT": 3 if kind.endswith("parity") else 1, "CUDA_GRAPH": True})
        model = B200SlowFast(cfg)
    torch.manual_seed(0)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 5))
    model = model.to(dev).train()
    inputs = [t.to(dev) for t in TO.synthetic_inputs(cfg, batch, 11)]
    labels = torch.randint(0, cfg.MODEL.NUM_CLASSES, (batch,), generator=torch.Generator().manual_seed(12)).to(dev)
    return model, inputs, labels


def main() -> None:
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--shapes", default="0,1,2,3")
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("subbn_bench needs a CUDA device")
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    from oracle import refshim
    with_ref = refshim.reference_available() and not args.no_reference
    result = dict(gpu_info(), seconds_per_leg=args.seconds, torch=torch.__version__, legs={})
    for rep in range(args.repeats):
        for si in (int(s) for s in args.shapes.split(",")):
            shape = SHAPES[si]
            kinds = (["sub_parity", "plain_parity", "sub_fast", "plain_fast"] if shape[3] > 1
                     else ["plain_parity", "plain_fast"]) + (["reference"] if with_ref else [])
            for kind in (kinds if rep % 2 == 0 else list(reversed(kinds))):
                name = "b{}_t{}_s{}_S{}/{}".format(*shape, kind)
                model, inputs, labels = build_leg(shape, kind, dev)
                r = time_leg(model, inputs, labels, args.seconds)
                result["legs"].setdefault(name, []).append(r)
                print(f"[rep {rep}] {name}: {r}", file=sys.stderr, flush=True)
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
