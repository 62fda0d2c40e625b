"""TEST INFRASTRUCTURE: the reference's own bf16 error class for tests/test_gpu_models.py's fast-mode test.

Runs the UNMODIFIED reference modules (oracle/refshim.py) under torch.autocast(bfloat16) on the fixtures that test
builds (same golden configs, weights, clips and upstream gradient) and writes their error against the fp32 oracle,
logits rel-L2 and median parameter-gradient rel-L2, to tests/golden/fast_mode_reference_error.json.  The test reads
it when the reference tree is not installed, so the comparison holds on any checkout.

    python -m oracle.make_fast_mode_bounds [--out FILE]      (on the GPU: CUDA autocast, as the test runs it live)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
OUT = os.path.join(GOLDEN, "fast_mode_reference_error.json")
CASES = {"mvit": "mvitv2_s_small", "slowfast": "slowfast_r50_small"}


def reference_error(family: str, device: str) -> dict:
    from oracle import refshim, torch_oracle as TO
    from oracle.golden_cfg import engine_cfg

    gold = torch.load(os.path.join(GOLDEN, CASES[family] + ".pt"))
    cfg = engine_cfg(gold, nsplit=1)
    template = {k: torch.empty(shape, dtype=torch.long if k.endswith("num_batches_tracked") else torch.float32)
                for k, shape in gold["keys"]}
    state = TO.fixture_state(template, 91)
    if family == "slowfast":
        for k in state:
            if k.endswith("c_bn.weight"):
                state[k] = state[k] * 0.1
    inputs = TO.synthetic_inputs(cfg, 2, 92)
    dlogits = torch.randn(2, 400, generator=torch.Generator().manual_seed(93))
    o_logits, o_grads = TO.forward_backward(cfg, state, inputs, dlogits)
    rcfg = refshim.load_cfg(gold["yaml"], ["NUM_GPUS", 1 if device == "cuda" else 0] + list(gold["overrides"]))
    model = refshim.build_reference_model(rcfg)
    model.load_state_dict(state, strict=True)
    model = model.to(device).train()
    with torch.autocast(device, dtype=torch.bfloat16):
        r_logits = model([t.to(device) for t in inputs])
    r_logits.float().backward(dlogits.to(device))
    r_log = ((r_logits.float().cpu() - o_logits).norm() / o_logits.norm()).item()
    rper = sorted(((p.grad.float().cpu() - o_grads[k]).norm() / o_grads[k].norm().clamp_min(1e-20)).item()
                  for k, p in model.named_parameters() if k in o_grads)
    return dict(logits_rel_l2=r_log, median_grad_rel_l2=rper[len(rper) // 2], autocast_device=device)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", default="cuda", choices=["cpu", "cuda"])
    ap.add_argument("--out", default=OUT)
    args = ap.parse_args()
    out = {family: reference_error(family, args.device) for family in CASES}
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
