"""GPU: the transfer switches on the engine against the unmodified reference on the same GPU.

  * MODEL.FROZEN_BN (``misc.frozen_bn_stats`` after ``model.train()``): every BN site normalises with its running
    statistics and keeps its buffers, while the convolutions train.  Held to the fp64 reference with the engine's ReLU
    masks and max-pool routes pinned (tests/test_gpu_resnet_pinned.py), with all BNs frozen and with a hand-frozen
    subset, and under CUDA-graph replay alternating frozen and training steps.
  * MODEL.DETACH_FINAL_FC (linear evaluation): nothing before the detach gets a gradient, and the backward program
    runs the projection only.
  * MODEL.HEAD_ACT sigmoid: the kernel against fp64, the eval outputs of the three head kinds against the reference.
"""
import time

import pytest
import torch
import torch.nn as nn

from test_gpu_replay import _build, _inputs
from test_gpu_resnet_pinned import BOUNDS, SOFTMAX_NLN_BOUNDS, engine_pins, install_pins
from test_gpu_vit import _rel

pytestmark = pytest.mark.gpu

TOL = 1e-3  # outputs against the reference (tests/test_gpu_models.py)

# The softmax Non-local cases are ill-conditioned: their attention logits are differences of large dot products, so
# the operand rounding of split-bf16 moves the attention weights far more than the logits.  For them the test also runs
# the pinned fp64 reference with every conv / einsum / linear operand rounded to split-bf16 (hi + lo, forward only) and
# holds the engine's worst gradient to EMULATION_FACTOR x that emulation's, where this exceeds SOFTMAX_NLN_BOUNDS.  The
# emulation rounds the forward operands only; the engine also rounds those of the backward GEMMs.  Measured (H100 80GB
# HBM3, 700 W), stock I3D-NLN on frozen BN: emulation 4.2e-3 logits / 0.13 worst gradient, engine 6.9e-3 / 0.34.
EMULATION_FACTOR = 4.0

FROZEN_CASES = [  # (id, yaml, frames, crop, batch)
    ("slowfast-64", "Kinetics/SLOWFAST_8x8_R50.yaml", 16, 64, 2),
    ("slow-64", "Kinetics/SLOW_8x8_R50.yaml", 8, 64, 2),
    ("i3d-nln-64", "Kinetics/I3D_NLN_8x8_R50.yaml", 8, 64, 2),
    ("x3d-m-64", "Kinetics/X3D_M.yaml", 4, 64, 2),
]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    refshim.install()
    return refshim


def _engine_class(cfg):
    name = cfg.MODEL.MODEL_NAME
    if name == "SlowFast":
        from slowfast_b200.nets.resnet import B200SlowFast as M
    elif name == "MViT":
        from slowfast_b200.nets.mvit import B200MViT as M
    elif name == "X3D":
        from slowfast_b200.nets.x3d import B200X3D as M
    else:
        from slowfast_b200.nets.resnet_single import B200ResNet as M
    return M


def _bns(model):
    return [(n, m) for n, m in model.named_modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]


def _bn_buffers(model):
    """{state_dict key: clone} of every BN buffer, with the module it belongs to."""
    out = {}
    for n, m in _bns(model):
        for b in ("running_mean", "running_var", "num_batches_tracked"):
            out[f"{n}.{b}"] = (m, getattr(m, b).detach().clone())
    return out


def _stat_err(v, ref):
    """Running-statistics agreement as tests/test_gpu_models.py holds it: the sums, relative to the reference's norm."""
    v, ref = v.double().flatten(), ref.double().flatten()
    return abs(v.sum().item() - ref.sum().item()) / max(abs(ref.sum().item()), ref.norm().item(), 1e-20)


def _fit_running_stats(ref, cfg, batch, dev, dtype):
    """Running statistics that fit the weights (random ones make an unnormalised 50-layer stack drift): one
    momentum-1.0 training forward of the reference on a second clip batch, as precise-BN takes them."""
    from oracle import torch_oracle as TO
    saved = [(m, m.momentum) for _, m in _bns(ref)]
    for m, _ in saved:
        m.momentum = 1.0
    ref.train()
    with torch.no_grad():
        ref([x.to(dev, dtype) for x in TO.synthetic_inputs(cfg, batch, 11)])
    for m, mmt in saved:
        m.momentum = mmt


def _split(x):
    """x rounded to the split-bf16 pair hi + lo the engine's tensor-core operands carry (fp64 result)."""
    hi = x.to(torch.bfloat16).to(x.dtype)
    return hi + (x - hi).to(torch.bfloat16).to(x.dtype)


def _rounded(x):
    """Forward: the split-bf16 value of x; backward: identity (the emulation rounds the forward operands only)."""
    return x + (_split(x.detach()) - x.detach())


class split_bf16_operands:
    """Context in which F.conv3d, torch.einsum and F.linear see split-bf16-rounded operands."""

    def __enter__(self):
        F = torch.nn.functional
        self.saved = (F.conv3d, torch.einsum, F.linear)
        conv3d, einsum, linear = self.saved
        F.conv3d = lambda x, w, b=None, *a, **k: conv3d(_rounded(x), _rounded(w), b, *a, **k)
        # (nonlocal_helper.py passes the operands as one tuple)
        torch.einsum = lambda eq, *ops: einsum(eq, *[_rounded(o) for o in
                                                     (ops[0] if len(ops) == 1 and isinstance(ops[0], tuple) else ops)])
        F.linear = lambda x, w, b=None: linear(_rounded(x), _rounded(w), b)
        return self

    def __exit__(self, *exc):
        F = torch.nn.functional
        F.conv3d, torch.einsum, F.linear = self.saved


def _freeze_all(model):
    from slowfast.utils import misc
    misc.frozen_bn_stats(model)


def _freeze_stem(model):
    for n, m in _bns(model):
        if n.startswith("s1."):
            m.eval()


def _frozen_run(yaml, frames, crop, batch, fixture, freeze, dev):
    """Engine against the pinned fp64 reference, both ``.train()`` then ``freeze``; returns the errors and checks
    the BN buffers: frozen ones bitwise unchanged in both models, the others updated as the reference updates them."""
    refshim = _refshim()
    from oracle import torch_oracle as TO
    t0 = time.time()
    cfg = refshim.load_cfg(yaml, ["DATA.NUM_FRAMES", frames, "DATA.TRAIN_CROP_SIZE", crop, "DATA.TEST_CROP_SIZE", crop,
                                  "MODEL.DROPOUT_RATE", 0.0])
    ref = refshim.build_reference_model(cfg)
    state = TO.fixture_state(ref.state_dict(), 7)
    if fixture == "gentle":
        for k in state:
            if k.endswith("c_bn.weight"):
                state[k] = state[k] * 0.1
    ref.load_state_dict(state)
    ref = ref.to(dev).double()
    _fit_running_stats(ref, cfg, batch, dev, torch.float64)
    state = {k: (v.float() if v.is_floating_point() else v).cpu() for k, v in ref.state_dict().items()}
    ref.load_state_dict(state)
    mine = _engine_class(cfg)(cfg)
    mine.load_state_dict(state)
    mine = mine.to(dev).train()
    freeze(ref)
    freeze(mine)
    before, before_ref = _bn_buffers(mine), _bn_buffers(ref)
    xs = [x.to(dev) for x in TO.synthetic_inputs(cfg, batch, 4)]
    dl = torch.randn(batch, cfg.MODEL.NUM_CLASSES, generator=torch.Generator().manual_seed(5)).to(dev)
    lm = mine(xs)
    torch.cuda.synchronize()
    pins, _ = engine_pins(mine)
    lm.backward(dl)
    install_pins(ref, pins)
    lr = ref([x.double() for x in xs])
    lr.backward(dl.double())
    torch.cuda.synchronize()
    rel = _rel(lm.double(), lr)
    g64 = {k: p.grad.detach().clone() for k, p in ref.named_parameters()}
    bad = [k for k, g in g64.items() if not torch.isfinite(g).all()]
    assert not bad, f"non-finite reference gradients: {bad}"
    bad = [k for k, p in mine.named_parameters() if not torch.isfinite(p.grad).all()]
    assert not bad, f"non-finite engine gradients: {bad}"
    med = sorted(g.norm().item() for g in g64.values())[len(g64) // 2]
    zero = {k for k, g in g64.items() if g.norm().item() < 1e-6 * med}
    per = {k: _rel(p.grad.double(), g64[k]) for k, p in mine.named_parameters() if k not in zero}
    worst = max(per, key=per.get)
    after, after_ref = _bn_buffers(mine), _bn_buffers(ref)
    softmax_nln = cfg.NONLOCAL.INSTANTIATION == "softmax" and any(l for st in cfg.NONLOCAL.LOCATION for l in st)
    emulated = ""
    if softmax_nln:
        # what split-bf16 operand rounding alone does to this fixture (same pins, frozen BN, fp64 otherwise)
        ref.zero_grad(set_to_none=True)
        with split_bf16_operands():
            le = ref([x.double() for x in xs])
            le.backward(dl.double())
        torch.cuda.synchronize()
        e_logits = _rel(le.detach(), lr.detach())
        e_per = {k: _rel(p.grad, g64[k]) for k, p in ref.named_parameters() if k not in zero}
        e_worst = max(e_per.values())
        emulated = f"; split-bf16 emulation of the reference: logits {e_logits:.2e} grad max {e_worst:.2e}"
    frozen = 0
    for k, (m, v) in before.items():
        if not m.training:
            frozen += 1
            assert torch.equal(after[k][1], v), k
            assert torch.equal(after_ref[k][1], before_ref[k][1]), k
        elif k.endswith("num_batches_tracked"):
            assert int(after[k][1]) == int(v) + 1 == int(after_ref[k][1]), k
        else:
            assert not torch.equal(after[k][1], v), k
            assert _stat_err(after[k][1], after_ref[k][1]) < 1e-3, k
    print(f"[frozen BN {yaml.split('/')[-1]} {frames}x{crop}^2, {fixture}, {frozen} of {len(before)} BN buffers frozen] "
          f"logits rel-L2 {rel:.2e}; grad rel-L2 median {sorted(per.values())[len(per) // 2]:.2e} max {per[worst]:.2e} "
          f"({worst}){emulated}; {time.time() - t0:.1f} s")
    b_logits, b_grad = (SOFTMAX_NLN_BOUNDS if softmax_nln else BOUNDS)[fixture]
    if softmax_nln:
        b_logits, b_grad = max(b_logits, EMULATION_FACTOR * e_logits), max(b_grad, EMULATION_FACTOR * e_worst)
    assert rel < b_logits and torch.equal(lm.argmax(1), lr.argmax(1)), rel
    assert per[worst] < b_grad, (worst, per[worst])
    for k in zero:
        assert mine.get_parameter(k).grad.norm().item() < 1e-3 * med, k
    return frozen, len(before)


@pytest.mark.parametrize("fixture", ["gentle", "stock"])
@pytest.mark.parametrize("yaml,frames,crop,batch", [c[1:] for c in FROZEN_CASES], ids=[c[0] for c in FROZEN_CASES])
def test_frozen_bn_matches_reference_fp64_with_pinned_routing(yaml, frames, crop, batch, fixture, cuda_device):
    frozen, total = _frozen_run(yaml, frames, crop, batch, fixture, _freeze_all, cuda_device)
    assert frozen == total


@pytest.mark.parametrize("fixture", ["gentle", "stock"])
def test_partly_frozen_bn_is_per_site(fixture, cuda_device):
    """Only the two stem BNs frozen: they keep their buffers, every other BN trains as in the reference."""
    frozen, total = _frozen_run("Kinetics/SLOWFAST_8x8_R50.yaml", 16, 64, 2, fixture, _freeze_stem, cuda_device)
    assert frozen == 6 and total > frozen


def test_replay_alternating_frozen_and_training_steps(cuda_device):
    """CUDA graphs on: frozen and training SGD steps alternate three times each.  Each BN mode is captured once and
    replayed by its own steps only; logits, BN buffers and parameters follow the eager sequence."""
    def run(graphs):
        cfg, model, _, batch = _build("slowfast", graphs, cuda_device)
        model.graph_warmup = 1  # steps 1-2 eager, 3-4 capture, 5-6 replay
        opt = torch.optim.SGD(model.parameters(), lr=0.002, momentum=0.9)
        outs, keys = [], []
        for s in range(6):
            frozen = s % 2 == 0
            for _, m in _bns(model):
                m.train(not frozen)
            x, y = _inputs(cfg, batch, 100 + s)
            before = {k: v[1] for k, v in _bn_buffers(model).items()}
            opt.zero_grad(set_to_none=True)
            logits = model([t.to(cuda_device) for t in x])
            torch.nn.functional.cross_entropy(logits, y.to(cuda_device)).backward()
            opt.step()
            after = {k: v[1] for k, v in _bn_buffers(model).items()}
            assert all(torch.equal(after[k], before[k]) == frozen for k in before), s
            outs.append(logits.detach().cpu())
            keys.append(dict(model._graphs))
        torch.cuda.synchronize()
        return model, outs, keys

    mg, og, kg = run(True)
    _, oe, _ = run(False)
    _, oe2, _ = run(False)
    assert len(mg._graphs) == 2
    k_frozen, k_train = sorted(mg._graphs, key=lambda k: -len(k[-1]))
    assert k_frozen[-1] and not k_train[-1] and k_frozen[:-1] == k_train[:-1]
    assert not kg[1] and set(kg[2]) == {k_frozen} and set(kg[3]) == {k_frozen, k_train}
    # steps 5 and 6 replay the programs captured at steps 3 and 4
    assert kg[5][k_frozen] is kg[2][k_frozen] and kg[5][k_train] is kg[3][k_train]
    for s in range(6):
        rel = ((og[s] - oe[s]).abs().max() / oe[s].abs().max()).item()
        noise = ((oe2[s] - oe[s]).abs().max() / oe[s].abs().max()).item()
        print(f"step {s} ({'frozen' if s % 2 == 0 else 'training'} BN): logits replay vs eager {rel:.2e} "
              f"(eager vs eager {noise:.2e})")
        assert rel < max(2e-4, 5 * noise), (s, rel, noise)


@pytest.mark.parametrize("case", ["slow-linear", "mvit-s"])
def test_detach_final_fc_trains_the_head_only(case, cuda_device):
    refshim = _refshim()
    from oracle import torch_oracle as TO
    from slowfast_b200 import ops
    if case == "slow-linear":
        cfg = refshim.load_cfg("contrastive_ssl/linear_k400_Slow_8x8_R50_syn0.yaml",
                               ["DATA.NUM_FRAMES", 8, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64])
    else:
        cfg = refshim.load_cfg("Kinetics/MVITv2_S_16x4.yaml",
                               ["DATA.NUM_FRAMES", 8, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64,
                                "MODEL.DROPOUT_RATE", 0.0, "MVIT.DROPPATH_RATE", 0.0, "MODEL.DETACH_FINAL_FC", True])
    assert cfg.MODEL.DETACH_FINAL_FC
    ref = refshim.build_reference_model(cfg)
    state = TO.fixture_state(ref.state_dict(), 21)
    ref.load_state_dict(state)
    ref = ref.to(cuda_device).train()
    mine = _engine_class(cfg)(cfg)
    mine.load_state_dict(state)
    mine = mine.to(cuda_device).train()
    xs = [x.to(cuda_device) for x in TO.synthetic_inputs(cfg, 2, 22)]
    dl = torch.randn(2, cfg.MODEL.NUM_CLASSES, generator=torch.Generator().manual_seed(23)).to(cuda_device)
    lm = mine(xs)
    n0 = ops.launches()
    lm.backward(dl)
    torch.cuda.synchronize()
    bwd_launches = ops.launches() - n0
    lr = ref(xs)
    lr.backward(dl)
    torch.cuda.synchronize()
    head = {"head.projection.weight", "head.projection.bias"}
    for k, p in ref.named_parameters():
        assert (p.grad is None) == (k not in head), k
    for k, p in mine.named_parameters():
        assert (p.grad is None) == (k not in head), k
    rel = ((lm - lr).abs().max() / lr.abs().max()).item()
    errs = {k: _rel(mine.get_parameter(k).grad, ref.get_parameter(k).grad) for k in head}
    print(f"[detach {case}] logits rel {rel:.2e}, head grads {errs}, backward launches {bwd_launches}")
    assert rel < TOL and all(e < TOL for e in errs.values()), (rel, errs)
    # the backward is the projection's weight / bias gradient kernel: one launch, whatever the depth
    assert bwd_launches == 1
    sm, sr = mine.state_dict(), ref.state_dict()
    for k in sr:
        if "running_" in k:
            assert _stat_err(sm[k], sr[k]) < 1e-3, k
        elif k.endswith("num_batches_tracked"):
            assert int(sm[k]) == int(sr[k]), k


def test_row_sigmoid_kernel_against_fp64(cuda_device):
    from slowfast_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(37, 401, generator=g) * 8
    x[0, :8] = torch.tensor([0.0, -0.0, 88.0, -88.0, 104.0, -104.0, 1e4, -1e4])
    x[1, :4] = torch.tensor([1e-8, -1e-8, 20.0, -20.0])
    y = x.to(cuda_device)
    ops.row_sigmoid(y)
    want = torch.sigmoid(x.double())
    got = y.cpu().double()
    assert torch.isfinite(got).all()
    err = (got - want).abs().max().item()
    normal = want >= torch.finfo(torch.float32).tiny  # below it fp32 flushes towards 0, as torch.sigmoid does
    rel = ((got - want).abs() / want)[normal].max().item()
    assert (got[~normal] <= torch.finfo(torch.float32).tiny).all()
    print(f"row_sigmoid vs fp64: max abs {err:.2e}, max rel {rel:.2e}")
    assert err < 2e-7 and rel < 1e-6


SIGMOID_CASES = [  # (id, yaml, frames, train crop, test crop, overrides)
    ("slowfast-windowed", "Kinetics/SLOWFAST_8x8_R50.yaml", 16, 64, 96, []),
    ("x3d-m", "Kinetics/X3D_M.yaml", 4, 64, 64, []),
    ("mvitv2-s", "Kinetics/MVITv2_S_16x4.yaml", 8, 64, 64, ["MVIT.DROPPATH_RATE", 0.0]),
]


@pytest.mark.parametrize("yaml,frames,crop,test_crop,extra", [c[1:] for c in SIGMOID_CASES],
                         ids=[c[0] for c in SIGMOID_CASES])
def test_sigmoid_head_eval_outputs_match_reference(yaml, frames, crop, test_crop, extra, cuda_device):
    refshim = _refshim()
    from oracle import torch_oracle as TO
    cfg = refshim.load_cfg(yaml, ["DATA.NUM_FRAMES", frames, "DATA.TRAIN_CROP_SIZE", crop, "DATA.TEST_CROP_SIZE",
                                  test_crop, "MODEL.HEAD_ACT", "sigmoid", "MODEL.DROPOUT_RATE", 0.0] + extra)
    ref = refshim.build_reference_model(cfg)
    ref.load_state_dict(TO.fixture_state(ref.state_dict(), 61))
    ref = ref.to(cuda_device)
    _fit_running_stats(ref, cfg, 2, cuda_device, torch.float32)
    state = {k: v.cpu() for k, v in ref.state_dict().items()}
    ref.eval()
    mine = _engine_class(cfg)(cfg)
    mine.load_state_dict(state)
    mine = mine.to(cuda_device).eval()
    xs = [x.to(cuda_device) for x in TO.synthetic_inputs(cfg, 2, 62, crop=test_crop)]
    with torch.no_grad():
        pm, pr = mine(xs), ref(xs)
    rel = ((pm - pr).abs().max() / pr.abs().max()).item()
    print(f"[sigmoid eval {yaml.split('/')[-1]} {frames}x{test_crop}^2] outputs rel {rel:.2e}")
    assert rel < TOL, rel
    assert (pm >= 0).all() and (pm <= 1).all() and not torch.allclose(pm.sum(1), torch.ones_like(pm[:, 0]))
    # train mode returns the logits
    if test_crop == crop:
        mine.train()
        ref.train()
        xs = [x.to(cuda_device) for x in TO.synthetic_inputs(cfg, 2, 63)]
        with torch.no_grad():
            lm, lr = mine(xs), ref(xs)
        assert ((lm - lr).abs().max() / lr.abs().max()).item() < TOL
        assert ((lm < 0) | (lm > 1)).any()


def test_flat_optimizer_and_allreduce_leave_the_detached_backbone_alone(cuda_device):
    """Under MODEL.DETACH_FINAL_FC the flat bucket is the projection's: FlatOptimizer steps it (and nothing else, weight
    decay and momentum included) and allreduce_gradients exchanges exactly that bucket."""
    import socket

    import torch.distributed as dist
    refshim = _refshim()
    from oracle import torch_oracle as TO
    from slowfast_b200.engine import flat_offsets
    from slowfast_b200.optim import FlatOptimizer, param_groups_from_cfg
    cfg = refshim.load_cfg("contrastive_ssl/linear_k400_Slow_8x8_R50_syn0.yaml",
                           ["DATA.NUM_FRAMES", 8, "DATA.TRAIN_CROP_SIZE", 64, "DATA.TEST_CROP_SIZE", 64,
                            "SOLVER.WEIGHT_DECAY", 1e-4, "BN.WEIGHT_DECAY", 1e-4])
    model = _engine_class(cfg)(cfg)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 31))
    model = model.to(cuda_device).train()
    head = model.grad_params()
    assert [id(p) for p in head] == [id(model.head.projection.weight), id(model.head.projection.bias)]
    opt = FlatOptimizer(model, "sgd", param_groups_from_cfg(model, cfg), lr=0.1, momentum=0.9, nesterov=True)
    before = {k: p.detach().clone() for k, p in model.named_parameters()}
    xs = [x.to(cuda_device) for x in TO.synthetic_inputs(cfg, 2, 32)]
    for step in range(2):
        opt.zero_grad()
        model(xs).square().sum().backward()
        assert model.ctx.flat_grad.numel() == flat_offsets(head)[1]
        opt.step()
    torch.cuda.synchronize()
    for k, p in model.named_parameters():
        if k.startswith("head.projection."):
            assert not torch.equal(p, before[k]), k
        else:
            assert torch.equal(p, before[k]), k
            assert p.grad is None, k
    # one-process NCCL group: the exchange covers the head-only bucket and re-points the head's .grad at it
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        flat = model.ctx.flat_grad
        want = flat.clone()
        model.allreduce_gradients()
        torch.cuda.synchronize()
        assert torch.equal(flat, want)
        offs, total = flat_offsets(head)
        assert flat.numel() == total
        for p, off in zip(head, offs):
            assert p.grad.data_ptr() == flat.data_ptr() + 4 * off
        assert all(p.grad is None for k, p in model.named_parameters() if not k.startswith("head.projection."))
    finally:
        dist.destroy_process_group()


def test_frozen_inner_sub_bn_is_rejected_at_forward(cuda_device):
    refshim = _refshim()
    from oracle import torch_oracle as TO
    cfg = refshim.load_cfg("Kinetics/SLOW_8x8_R50.yaml", ["DATA.NUM_FRAMES", 4, "DATA.TRAIN_CROP_SIZE", 64,
                                                           "DATA.TEST_CROP_SIZE", 64, "BN.NORM_TYPE", "sub_batchnorm",
                                                           "BN.NUM_SPLITS", 2])
    model = _engine_class(cfg)(cfg).to(cuda_device).train()
    model.s3.pathway0_res1.branch2.b_bn.split_bn.eval()
    with pytest.raises(NotImplementedError, match="MODEL.FROZEN_BN"):
        model([x.to(cuda_device) for x in TO.synthetic_inputs(cfg, 2, 3)])


# ------------------------------------------------------------------------------------------------ unmodified drivers
def _driver_harness():
    import driver_harness as H
    if H.setup_reference() is None:
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    return H


def _assert_driver_losses(en, st, what):
    assert len(en["train"]) == len(st["train"]) > 0
    for i, (a, b) in enumerate(zip(en["train"], st["train"])):
        rel = abs(a["loss"] - b["loss"]) / abs(b["loss"])
        print(f"{what}: iter {i} loss engine {a['loss']:.6f} stock {b['loss']:.6f} (rel {rel:.1e})")
        assert rel < (1e-3 if i == 0 else 1e-2), (i, a["loss"], b["loss"])   # test_gpu_drivers.py's bounds
    assert len(en["val"]) == len(st["val"]) > 0


def _last_checkpoint(out_dir, task=""):
    """model_state of the last checkpoint ``save_checkpoint`` wrote for ``task`` (get_path_to_checkpoint's names)."""
    import glob
    import os
    name = f"{task}_checkpoint_epoch_*.pyth" if task else "checkpoint_epoch_*.pyth"
    return torch.load(sorted(glob.glob(os.path.join(out_dir, "checkpoints", name)))[-1], map_location="cpu",
                      weights_only=False)["model_state"]


def test_moco_checkpoint_linear_probe_through_the_unmodified_driver(cuda_device, tmp_path):
    """An engine MoCo checkpoint (cu.save_checkpoint of a built B200ContrastiveModel) is linear-probed by the unmodified
    tools/train_net.train with TASK ssl_eval_k400: the ssl_eval branch (train_net.py:544) loads it with
    CHECKPOINT_CLEAR_NAME_PATTERN ("backbone.",).  Engine and stock model: losses within the driver bounds, every backbone
    parameter after the epoch bitwise the loaded one, the head moved."""
    import shutil

    H = _driver_harness()
    import slowfast.models.optimizer as optim
    import slowfast.utils.checkpoint as cu
    from oracle import torch_oracle as TO
    from slowfast.models import build_model
    moco_dir = tmp_path / "moco"
    try:
        H.use_engine(True)
        mcfg = H.driver_cfg("contrastive_ssl/MoCo_SlowR50_8x8.yaml", 1,
                            ["CONTRASTIVE.QUEUE_LEN", 64, "CONTRASTIVE.LENGTH", 16, "DATA.NUM_FRAMES", 8],
                            out_dir=str(moco_dir))
        moco = build_model(mcfg)
        assert type(moco).__name__ == "B200ContrastiveModel"
        sd = moco.state_dict()
        sd.update({k: v for k, v in TO.fixture_state(sd, 41).items() if k.startswith("backbone.")})
        moco.load_state_dict(sd)
        ckpt = cu.save_checkpoint(str(moco_dir), moco, optim.construct_optimizer(moco, mcfg), 0, mcfg)
        saved = torch.load(ckpt, map_location="cpu", weights_only=False)["model_state"]
        del moco
        recs, loaded, final = {}, {}, {}
        orig = cu.load_checkpoint
        for engine in (False, True):
            H.use_engine(engine)
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            out = tmp_path / ("engine" if engine else "stock")
            (out / "checkpoints").mkdir(parents=True)
            shutil.copy(ckpt, out / "checkpoints")
            cfg = H.driver_cfg("contrastive_ssl/linear_k400_Slow_8x8_R50_syn0.yaml", 1,
                               ["TRAIN.AUTO_RESUME", True, "DATA.NUM_FRAMES", 8, "SOLVER.BASE_LR", 0.05],
                               out_dir=str(out))
            assert cfg.TASK == "ssl_eval_k400" and cfg.MODEL.DETACH_FINAL_FC
            params = set()

            def recording_load(path, model, *a, **k):
                epoch = orig(path, model, *a, **k)
                m = getattr(model, "module", model)
                params.update(n for n, _ in m.named_parameters())
                loaded[engine] = {n: v.detach().cpu().clone() for n, v in m.state_dict().items()}
                assert type(m).__name__ == ("B200ResNet" if engine else "ResNet")
                return epoch

            cu.load_checkpoint = recording_load
            try:
                recs[engine], _ = H.run_train(cfg)
            finally:
                cu.load_checkpoint = orig
            final[engine] = _last_checkpoint(str(out), cfg.TASK)
        _assert_driver_losses(recs[True], recs[False], "linear probe")
        backbone = sorted(k for k in params if not k.startswith("head."))
        assert backbone and all("backbone." + k in saved for k in backbone)
        for engine in (False, True):
            for k in backbone:
                assert torch.equal(loaded[engine][k], saved["backbone." + k]), (engine, k)
                assert torch.equal(final[engine][k], loaded[engine][k]), (engine, k)
            for k in ("head.projection.weight", "head.projection.bias"):
                assert not torch.equal(final[engine][k], loaded[engine][k]), (engine, k)
    finally:
        H.use_engine(False)


def test_frozen_bn_through_the_unmodified_driver(cuda_device, tmp_path):
    """MODEL.FROZEN_BN on a shrunk Slow-R50 through tools/train_net.train (frozen_bn_stats inside train_epoch, the
    eval epoch, CUDA graphs on): losses within the driver bounds of the stock model, every BN buffer bitwise its initial
    value after the epoch."""
    H = _driver_harness()
    from slowfast.models import build_model
    recs, final, init = {}, {}, {}
    try:
        for engine in (False, True):
            H.use_engine(engine)
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            out = tmp_path / ("engine" if engine else "stock")
            out.mkdir()
            cfg = H.driver_cfg("Kinetics/SLOW_8x8_R50.yaml", 1,
                               ["MODEL.FROZEN_BN", True, "MODEL.DROPOUT_RATE", 0.0, "SOLVER.BASE_LR", 0.002],
                               out_dir=str(out), frames=8)
            built = build_model(cfg)
            assert type(built).__name__ == ("B200ResNet" if engine else "ResNet")
            init[engine] = {k: v.cpu() for k, v in built.state_dict().items()
                            if "running_" in k or k.endswith("num_batches_tracked")}
            del built
            recs[engine], _ = H.run_train(cfg)
            final[engine] = _last_checkpoint(str(out), cfg.TASK)
        _assert_driver_losses(recs[True], recs[False], "frozen BN")
        for engine in (False, True):
            assert len(init[engine]) > 100
            for k, v in init[engine].items():
                assert torch.equal(final[engine][k], v), (engine, k)
    finally:
        H.use_engine(False)
