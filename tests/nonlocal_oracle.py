"""TEST INFRASTRUCTURE: plain-PyTorch restatement of the Non-local recipes (C2D / I3D / Slow / SlowFast NLN) and the
generator of their golden files.

The restatement extends ``oracle/torch_oracle.py`` (whose stems, bottleneck blocks, lateral fusions and head it reuses
unchanged) with the Non-local block exactly as the reference evaluates it: ``nonlocal_helper.py:103-144`` in its own
order (theta, pool, phi / g, the Nq x Nk affinity, softmax or 1/Nk scaling, the second einsum, conv_out, bn, residual)
around the temporal group fold of ``resnet_helper.py:704-722``.

Goldens: run in a tree where the unmodified reference is available (``oracle/_ref`` or $SLOWFAST_REFERENCE_ROOT):

    python tests/nonlocal_oracle.py [case ...]

For every case it builds the reference model, loads the seeded fixture state, runs forward + backward on CPU (fp32),
checks this restatement against it and writes ``tests/golden/<case>.pt`` in the format of ``oracle/make_golden.py``.
"""
from __future__ import annotations

import os
import sys
from typing import List

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import torch_oracle as TO  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

# golden yaml -> engine preset (slowfast_b200.config)
PRESET = {"Kinetics/C2D_NLN_8x8_R50.yaml": "C2D_NLN_8x8_R50", "Kinetics/I3D_NLN_8x8_R50.yaml": "I3D_NLN_8x8_R50",
          "Kinetics/SLOW_NLN_8x8_R50.yaml": "SLOW_NLN_8x8_R50",
          "Kinetics/SLOWFAST_NLN_8x8_R50.yaml": "SLOWFAST_NLN_8x8_R50"}

_SMALL = ["DATA.NUM_FRAMES", 8, "DATA.TRAIN_CROP_SIZE", 64, "MODEL.DROPOUT_RATE", 0.0]
CASES = {
    # name: (yaml, overrides, batch, input seed, state seed)
    "i3d_nln_r50_small": ("Kinetics/I3D_NLN_8x8_R50.yaml", _SMALL, 2, 71, 72),
    "c2d_nln_r50_small": ("Kinetics/C2D_NLN_8x8_R50.yaml", _SMALL, 2, 73, 74),
    "slow_nln_r50_small": ("Kinetics/SLOW_NLN_8x8_R50.yaml", _SMALL, 2, 75, 76),
    # the Non-local after the last res3 slow block writes the channel slice of the lateral-concat storage
    "slowfast_nln_r50_small": ("Kinetics/SLOWFAST_NLN_8x8_R50.yaml",
                               ["DATA.NUM_FRAMES", 16, "DATA.TRAIN_CROP_SIZE", 64, "MODEL.DROPOUT_RATE", 0.0], 2, 77, 78),
    # T folded into the batch (GROUP 2) and the grouped T/2 pooled in time (POOL [2, 2, 2])
    "i3d_nln_group2_small": ("Kinetics/I3D_NLN_8x8_R50.yaml",
                             _SMALL + ["NONLOCAL.GROUP", [[1], [2], [2], [1]], "NONLOCAL.POOL", [[[2, 2, 2]]] * 4],
                             2, 79, 80),
    # the real geometry (Nq 3136 / Nk 784 softmax; Nq 6272 / Nk 1568 dot_product on the slow pathway)
    "i3d_nln_r50_224": ("Kinetics/I3D_NLN_8x8_R50.yaml", ["MODEL.DROPOUT_RATE", 0.0], 1, 81, 82),
    "slowfast_nln_r50_224": ("Kinetics/SLOWFAST_NLN_8x8_R50.yaml", ["MODEL.DROPOUT_RATE", 0.0], 1, 83, 84),
}
# cases that also store sampled gradients and the reference's own fp32-vs-fp64 envelope (as oracle/make_golden.SAMPLED)
SAMPLED = {"i3d_nln_r50_224", "slowfast_nln_r50_224"}


def nonlocal_block(x, sd: TO.SD, prefix: str, pool, instantiation: str, group: int, training: bool):
    """ResStage's group fold (resnet_helper.py:704-722) around Nonlocal.forward (nonlocal_helper.py:103-144)."""
    b, c, t, h, w = x.shape
    if group > 1:
        x = x.permute(0, 2, 1, 3, 4).reshape(b * group, t // group, c, h, w).permute(0, 2, 1, 3, 4)
    x_identity = x
    n, _, tt, hh, ww = x.size()
    theta = F.conv3d(x, sd[prefix + ".conv_theta.weight"], sd[prefix + ".conv_theta.bias"])
    if pool is not None and any(s > 1 for s in pool):
        x = F.max_pool3d(x, list(pool), list(pool), [0, 0, 0])
    phi = F.conv3d(x, sd[prefix + ".conv_phi.weight"], sd[prefix + ".conv_phi.bias"])
    g = F.conv3d(x, sd[prefix + ".conv_g.weight"], sd[prefix + ".conv_g.bias"])
    d = theta.shape[1]
    theta, phi, g = theta.view(n, d, -1), phi.view(n, d, -1), g.view(n, d, -1)
    theta_phi = torch.einsum("nct,ncp->ntp", (theta, phi))
    if instantiation == "softmax":
        theta_phi = theta_phi * (d ** -0.5)
        theta_phi = F.softmax(theta_phi, dim=2)
    elif instantiation == "dot_product":
        theta_phi = theta_phi / theta_phi.shape[2]
    else:
        raise NotImplementedError(instantiation)
    theta_phi_g = torch.einsum("ntg,ncg->nct", (theta_phi, g)).view(n, d, tt, hh, ww)
    p = F.conv3d(theta_phi_g, sd[prefix + ".conv_out.weight"], sd[prefix + ".conv_out.bias"])
    p = TO._bn(p, sd, prefix + ".bn", training)
    out = x_identity + p
    if group > 1:
        out = out.permute(0, 2, 1, 3, 4).reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4)
    return out


def _stage(cfg, stage: int, xs: List[torch.Tensor], sd: TO.SD, prefix: str, depth: int, strides, training: bool):
    """ResStage.forward (resnet_helper.py:697-726) with its Non-local blocks."""
    out = []
    for p, x in enumerate(xs):
        for i in range(depth):
            x = TO._res_block(x, sd, f"{prefix}.pathway{p}_res{i}", strides[p] if i == 0 else 1, training)
            nl = f"{prefix}.pathway{p}_nonlocal{i}"
            if nl + ".conv_theta.weight" in sd:
                x = nonlocal_block(x, sd, nl, cfg.NONLOCAL.POOL[stage][p], cfg.NONLOCAL.INSTANTIATION,
                                   cfg.NONLOCAL.GROUP[stage][p], training)
        out.append(x)
    return out


def slowfast_forward(cfg, sd: TO.SD, inputs, training: bool = True):
    """oracle/torch_oracle.slowfast_forward with Non-local stages."""
    depth = TO.STAGE_DEPTH[cfg.RESNET.DEPTH]
    alpha = cfg.SLOWFAST.ALPHA
    xs, xf = inputs
    xs = TO._stem(xs, sd, "s1.pathway0_stem", training)
    xf = TO._stem(xf, sd, "s1.pathway1_stem", training)
    xs, xf = TO._fuse(xs, xf, sd, "s1_fuse", alpha, training)
    for i in range(4):
        xs, xf = _stage(cfg, i, [xs, xf], sd, f"s{i + 2}", depth[i], cfg.RESNET.SPATIAL_STRIDES[i], training)
        if i < 3:
            xs, xf = TO._fuse(xs, xf, sd, f"s{i + 2}_fuse", alpha, training)
    c32 = cfg.DATA.TRAIN_CROP_SIZE // 32
    pools = None if cfg.MULTIGRID.SHORT_CYCLE else [[cfg.DATA.NUM_FRAMES // alpha, c32, c32],
                                                     [cfg.DATA.NUM_FRAMES, c32, c32]]
    return TO._basic_head([xs, xf], sd, training, cfg.MODEL.DROPOUT_RATE, cfg.MODEL.HEAD_ACT, pools)


def resnet_forward(cfg, sd: TO.SD, inputs, training: bool = True):
    """oracle/torch_oracle.resnet_forward with Non-local stages."""
    depth = TO.STAGE_DEPTH[cfg.RESNET.DEPTH]
    pool1 = {"2d": 1, "c2d": 2, "slow_c2d": 1, "i3d": 2, "slow_i3d": 1, "slow": 1}[cfg.MODEL.ARCH]
    (x,) = inputs
    x = TO._stem(x, sd, "s1.pathway0_stem", training)
    for i in range(4):
        (x,) = _stage(cfg, i, [x], sd, f"s{i + 2}", depth[i], cfg.RESNET.SPATIAL_STRIDES[i], training)
        if i == 0 and pool1 > 1:
            x = F.max_pool3d(x, (pool1, 1, 1), (pool1, 1, 1), 0)
    c32 = cfg.DATA.TRAIN_CROP_SIZE // 32
    pools = None if cfg.MULTIGRID.SHORT_CYCLE else [[cfg.DATA.NUM_FRAMES // pool1, c32, c32]]
    return TO._basic_head([x], sd, training, cfg.MODEL.DROPOUT_RATE, cfg.MODEL.HEAD_ACT, pools)


def forward(cfg, sd: TO.SD, inputs, training: bool = True):
    fn = slowfast_forward if cfg.MODEL.MODEL_NAME in ("SlowFast", "B200SlowFast") else resnet_forward
    return fn(cfg, sd, inputs, training)


def forward_backward(cfg, sd: TO.SD, inputs, dlogits):
    """logits and the gradient of sum(logits * dlogits) w.r.t. every parameter (train mode)."""
    names = [k for k, v in sd.items() if v.is_floating_point() and "running_" not in k]
    work = {k: (v.clone() if "running_" in k else v) for k, v in sd.items()}
    leaves = {k: sd[k].detach().clone().requires_grad_(True) for k in names}
    work.update(leaves)
    logits = forward(cfg, work, inputs, True)
    grads = torch.autograd.grad(logits, [leaves[k] for k in names], dlogits, allow_unused=True)
    return logits.detach(), {k: g for k, g in zip(names, grads) if g is not None}


def engine_cfg(gold, nsplit: int = 3):
    """The engine config of a golden file: its preset plus the overrides it was generated with."""
    from slowfast_b200.config import get_cfg
    cfg = get_cfg(PRESET[gold["yaml"]], B200={"NSPLIT": nsplit})
    ov = gold["overrides"]
    for k, v in zip(ov[0::2], ov[1::2]):
        sec, key = k.split(".")
        cfg[sec][key] = v
    return cfg


# ------------------------------------------------------------------------------------------------ golden generation
def _digest(t: torch.Tensor):
    f = t.detach().double().flatten()
    return dict(norm=f.norm().item(), sum=f.sum().item(), head=f[:4].tolist(), numel=f.numel())


def sample_idx(numel: int, k: int = 256) -> torch.Tensor:
    return torch.linspace(0, numel - 1, min(numel, k)).round().long()


def run_case(name, yaml, overrides, batch, in_seed, st_seed):
    from oracle import refshim
    cfg = refshim.load_cfg(yaml, overrides)
    model = refshim.build_reference_model(cfg)
    state = TO.fixture_state(model.state_dict(), st_seed)
    model.load_state_dict(state, strict=True)
    model.train()
    inputs = TO.synthetic_inputs(cfg, batch, in_seed)
    logits = model([t.clone() for t in inputs])
    dlogits = torch.randn(logits.shape, generator=torch.Generator().manual_seed(in_seed + 1000))
    logits.backward(dlogits)
    ref_grads = {k: p.grad for k, p in model.named_parameters()}
    ref_state = model.state_dict()
    # ---- pin the restatement against the reference itself (the bounds of oracle/make_golden.py)
    o_logits, o_grads = forward_backward(cfg, state, inputs, dlogits)
    work = {k: v.clone() for k, v in state.items()}
    forward(cfg, work, inputs, True)
    err_logits = (o_logits - logits.detach()).abs().max().item() / logits.detach().abs().max().item()
    norms = sorted(g.norm().item() for g in ref_grads.values())
    floor = 1e-2 * norms[len(norms) // 2]
    err_grad = max(((o_grads[k] - ref_grads[k]).norm() / ref_grads[k].norm().clamp_min(floor)).item() for k in ref_grads)
    err_rs = max([((work[k] - ref_state[k]).abs().max() / ref_state[k].abs().max().clamp_min(1e-20)).item()
                  for k in ref_state if "running_" in k] + [0.0])
    print(f"[{name}] oracle vs reference: logits rel {err_logits:.2e}  worst param-grad rel-L2 {err_grad:.2e}  "
          f"running stats rel {err_rs:.2e}")
    assert err_logits < 1e-5 and err_grad < 1e-4 and err_rs < 1e-5, "Non-local restatement disagrees with the reference"
    gold = dict(
        case=name, yaml=yaml, overrides=overrides, batch=batch, in_seed=in_seed, st_seed=st_seed,
        logits=logits.detach().clone(),
        grads={k: _digest(g) for k, g in ref_grads.items()},
        grad_norm_floor=floor,
        running={k: _digest(v) for k, v in ref_state.items() if "running_" in k},
        keys=[(k, tuple(v.shape)) for k, v in ref_state.items()],
        oracle_check=dict(logits=err_logits, grads=err_grad, running=err_rs),
        torch=str(torch.__version__),
    )
    # the reference's OWN fp32 rounding error: same modules, same state, run in fp64 (logits for every case; sampled
    # gradients for SAMPLED)
    model64 = refshim.build_reference_model(cfg).double()
    model64.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in state.items()})
    model64.train()
    l64 = model64([t.double() for t in inputs])
    gold["logits_env"] = ((logits.detach().double() - l64.detach()).abs().max() / l64.detach().abs().max()).item()
    print(f"[{name}] reference fp32 vs fp64 logits: {gold['logits_env']:.2e}")
    if name in SAMPLED:
        l64.backward(dlogits.double())
        g64 = {k: p.grad for k, p in model64.named_parameters()}
        gold["grad_samples"] = {k: g.flatten()[sample_idx(g.numel())].clone() for k, g in ref_grads.items()}
        env = {}
        for k, g in ref_grads.items():
            i = sample_idx(g.numel())
            a, b = g.flatten()[i].double(), g64[k].flatten()[i]
            env[k] = ((a - b).norm() / b.norm().clamp_min(1e-30)).item()
        gold["grad_env"] = env
        e = sorted(env.values())
        print(f"[{name}] reference fp32 vs fp64: logits {gold['logits_env']:.2e}; sampled-gradient rel-L2 median "
              f"{e[len(e) // 2]:.2e} max {e[-1]:.2e}")
    out = os.path.join(GOLDEN, name + ".pt")
    torch.save(gold, out)
    print(f"[{name}] wrote {out} ({os.path.getsize(out) / 1024:.1f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    for case in sys.argv[1:] or list(CASES):
        run_case(case, *CASES[case])
