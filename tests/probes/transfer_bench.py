"""GPU probe: the three transfer steps of a Slow-R50 (configs/Kinetics/SLOW_8x8_R50.yaml, 8 clips of 8 x 224^2):
  * finetune  - every BN in training mode, the whole network trains;
  * frozen_bn - MODEL.FROZEN_BN: ``misc.frozen_bn_stats`` after ``.train()``, every BN on its running statistics;
  * linear    - MODEL.DETACH_FINAL_FC (contrastive_ssl/linear_k400_Slow_8x8_R50_syn0.yaml): the projection trains only.
Each step is forward, cross-entropy, backward and a torch.optim.SGD step, timed on the engine (parity mode, split-bf16,
CUDA graphs on) and on the unmodified reference (oracle/_ref, fp32 PyTorch) on the same GPU, legs alternating.  Every leg
warms up, then runs for at least --seconds of wall time, bracketed by CUDA events.  Prints one JSON object with the GPU
name and power limit.

    python tests/probes/transfer_bench.py [--seconds 5] [--repeats 2] [--out transfer_bench.json]
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

BATCH = 8
STEPS = {"finetune": ("Kinetics/SLOW_8x8_R50.yaml", False), "frozen_bn": ("Kinetics/SLOW_8x8_R50.yaml", True),
         "linear": ("contrastive_ssl/linear_k400_Slow_8x8_R50_syn0.yaml", False)}


def build_leg(impl: str, step: str, dev):
    import torch
    from oracle import refshim
    from oracle import torch_oracle as TO
    from slowfast.utils import misc
    yaml, frozen = STEPS[step]
    cfg = refshim.load_cfg(yaml, ["NUM_GPUS", 1, "TRAIN.BATCH_SIZE", BATCH, "DATA.NUM_FRAMES", 8,
                                  "DATA.TRAIN_CROP_SIZE", 224, "MODEL.DROPOUT_RATE", 0.0, "MODEL.FROZEN_BN", frozen])
    if impl == "reference":
        model = refshim.build_reference_model(cfg)
    else:
        from slowfast_b200.nets.resnet_single import B200ResNet
        cfg["B200"] = {"NSPLIT": 3, "CUDA_GRAPH": True}
        torch.manual_seed(cfg.RNG_SEED)
        model = B200ResNet(cfg)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 5))
    model = model.to(dev).train()
    if cfg.MODEL.FROZEN_BN:
        misc.frozen_bn_stats(model)  # as tools/train_net.py:72-73 does after model.train()
    x = [t.to(dev) for t in TO.synthetic_inputs(cfg, BATCH, 20)]
    y = torch.randint(0, cfg.MODEL.NUM_CLASSES, (BATCH,), generator=torch.Generator().manual_seed(21)).to(dev)
    return model, x, y


def time_leg(impl, step, dev, seconds):
    import torch
    model, x, y = build_leg(impl, step, dev)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-4, momentum=0.9)

    def run():
        opt.zero_grad(set_to_none=True)
        torch.nn.functional.cross_entropy(model(x), y).backward()
        opt.step()

    for _ in range(4):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps, t0 = 0, time.perf_counter()
    e0.record()
    while steps < 3 or time.perf_counter() - t0 < seconds:
        run()
        steps += 1
        if steps % 8 == 0:
            torch.cuda.synchronize()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    out = {"steps": steps, "step_ms": round(ms / steps, 2), "clips_per_s": round(1e3 * steps * BATCH / ms, 2)}
    del model, x, y, opt
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
        raise SystemExit("transfer_bench needs a CUDA device")
    from oracle import refshim
    if not refshim.reference_available():
        raise SystemExit("transfer_bench needs the reference tree (build() copies it into oracle/_ref)")
    refshim.install()
    dev = torch.device("cuda:0")
    legs = [(impl, step) for step in STEPS for impl in (["engine"] + ([] if args.no_reference else ["reference"]))]
    result = dict(gpu_info(), seconds_per_leg=args.seconds, torch=torch.__version__, batch=BATCH, legs={})
    for rep in range(args.repeats):
        for impl, step in (legs if rep % 2 == 0 else list(reversed(legs))):
            r = time_leg(impl, step, dev, args.seconds)
            result["legs"].setdefault(f"{impl}/{step}", []).append(r)
            print(f"[rep {rep}] {impl} {step}: {r}", file=sys.stderr, flush=True)
    result["summary"] = {k: [r["step_ms"] for r in rs] for k, rs in result["legs"].items()}
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
