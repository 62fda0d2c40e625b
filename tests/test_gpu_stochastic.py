"""GPU tests of the stochastic operators every bench leg runs (head dropout 0.5, MViT stochastic depth 0.2) and no parity
test could pin (parity runs switch them off because the reference's Philox stream cannot be reproduced):

  * kernel level: keep rate, 1/keep scaling, saved mask == what the forward applied, backward uses the saved mask,
    the device-side step counter advances so that CUDA-graph replays draw fresh masks;
  * model level: with the step counter reset to the same value the forward is reproducible (so mask(fwd) is a pure
    function of (seed, counter)), consecutive replays differ, and a central finite difference of the loss along a random
    parameter direction - evaluated with the SAME mask - equals <grad, direction>: the backward applied the forward's mask.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_dropout_kernel_statistics_and_mask_identity(cuda_device):
    from slowfast_b200 import ops
    n, p = 1 << 20, 0.5
    for p in (0.5, 0.1):
        x = torch.full((n,), 2.0, device=cuda_device)
        mask = torch.empty(n, dtype=torch.uint8, device=cuda_device)
        step = torch.zeros(1, dtype=torch.int64, device=cuda_device)
        ops.dropout_fwd(x, mask, p, 1234, step)
        keep = mask.float().mean().item()
        assert abs(keep - (1 - p)) < 5 * math.sqrt(p * (1 - p) / n), (p, keep)
        assert set(mask.unique().tolist()) <= {0, 1}
        assert torch.equal(x != 0, mask.bool())
        assert torch.allclose(x[mask.bool()], torch.full_like(x[mask.bool()], 2.0 / (1 - p)))
        assert int(step.item()) == 1
        # backward: dx <- dx * mask / (1 - p) with the SAVED mask
        dx = torch.randn(n, device=cuda_device)
        want = dx * mask.float() / (1 - p)
        ops.dropout_bwd(dx, mask, p)
        assert torch.allclose(dx, want)
        # the counter makes the next call (a graph replay) draw another mask; the same counter reproduces the mask
        x2 = torch.full((n,), 2.0, device=cuda_device)
        mask2 = torch.empty_like(mask)
        ops.dropout_fwd(x2, mask2, p, 1234, step)
        frac_same = (mask2 == mask).float().mean().item()
        assert abs(frac_same - (p * p + (1 - p) * (1 - p))) < 0.01, frac_same  # independent draws
        step.zero_()
        x3 = torch.full((n,), 2.0, device=cuda_device)
        mask3 = torch.empty_like(mask)
        ops.dropout_fwd(x3, mask3, p, 1234, step)
        assert torch.equal(mask3, mask)


def test_droppath_scales_kernel(cuda_device):
    from slowfast_b200 import ops
    b = 8192
    rates = torch.tensor([0.0, 0.1, 0.2, 0.5], device=cuda_device)
    out = torch.empty(4, b, device=cuda_device)
    step = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    ops.droppath_scales(out, rates, 99, step)
    first = out.clone()
    assert torch.all(first[0] == 1.0)  # rate 0: exact identity
    for i, r in enumerate(rates.tolist()[1:], start=1):
        keep = 1.0 - r
        vals = first[i]
        kept = vals != 0
        assert torch.allclose(vals[kept], torch.full_like(vals[kept], 1.0 / keep))  # x / keep * floor(keep + U)
        frac = kept.float().mean().item()
        assert abs(frac - keep) < 5 * math.sqrt(keep * r / b), (r, frac)
    ops.droppath_scales(out, rates, 99, step)
    assert int(step.item()) == 2
    assert (out[3] != first[3]).float().mean().item() > 0.3  # a different draw per step
    step.zero_()
    ops.droppath_scales(out, rates, 99, step)
    assert torch.equal(out, first)


def _mvit(dev, graphs):
    from oracle import torch_oracle as TO
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    cfg = get_cfg("MVITv2_S_16x4", DATA={"NUM_FRAMES": 8, "TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64},
                  MODEL={"DROPOUT_RATE": 0.5}, MVIT={"DROPPATH_RATE": 0.3}, B200={"NSPLIT": 3, "CUDA_GRAPH": graphs})
    torch.manual_seed(0)
    m = B200MViT(cfg)
    m.load_state_dict(TO.fixture_state(m.state_dict(), 5))
    return cfg, m.to(dev).train()


def _reset_counters(m):
    for name in ("_dp_counter", "_drop_counter"):
        c = getattr(m, name, None)
        if c is not None:
            c.zero_()


def test_mvit_stochastic_depth_and_dropout_forward_backward_consistency(cuda_device):
    from oracle import torch_oracle as TO
    cfg, m = _mvit(cuda_device, graphs=False)
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, 4, 3)]
    y = torch.randint(0, 400, (4,), generator=torch.Generator().manual_seed(1)).to(cuda_device)
    loss_fn = torch.nn.functional.cross_entropy

    def loss_at():
        _reset_counters(m)  # same (seed, counter) -> same masks
        return loss_fn(m(x), y)

    l0 = loss_at()            # first call creates the counters (value 0) and uses them
    l0b = loss_at()
    assert torch.equal(l0, l0b) or abs(l0.item() - l0b.item()) < 1e-6 * abs(l0.item())
    l_next = loss_fn(m(x), y)  # counters advanced: another mask
    assert abs(l_next.item() - l0.item()) > 1e-4 * abs(l0.item()), "drop-path / dropout masks did not change between steps"
    sc = m.ctx.arena.bufs[("dp.scales",)].clone()
    assert (sc == 0).any() and (sc > 1).any(), "no dropped / rescaled sample in the stochastic-depth scales"
    # gradient with the counter-0 masks
    m.zero_grad(set_to_none=True)
    loss_at().backward()
    params = [p for p in m.parameters()]
    grads = [p.grad.detach().clone() for p in params]
    g = torch.Generator(device="cpu").manual_seed(11)
    dirs = [torch.randn(p.shape, generator=g).to(cuda_device) * p.detach().abs().mean().clamp_min(1e-3) for p in params]
    dd = sum((gr * d).sum().item() for gr, d in zip(grads, dirs))
    eps = 2e-2
    with torch.no_grad():
        for p, d in zip(params, dirs):
            p.add_(eps * d)
        lp = loss_at().item()
        for p, d in zip(params, dirs):
            p.sub_(2 * eps * d)
        lm = loss_at().item()
        for p, d in zip(params, dirs):
            p.add_(eps * d)
    fd = (lp - lm) / (2 * eps)
    print(f"mvit stochastic: <grad, d> = {dd:.5e}, central difference = {fd:.5e}")
    assert abs(fd - dd) < 0.05 * max(abs(dd), abs(fd)) + 1e-6, (fd, dd)


def test_mvit_masks_differ_between_graph_replays(cuda_device):
    from oracle import torch_oracle as TO
    cfg, m = _mvit(cuda_device, graphs=True)
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, 4, 3)]
    y = torch.randint(0, 400, (4,), generator=torch.Generator().manual_seed(1)).to(cuda_device)
    scales, losses = [], []
    for i in range(6):
        m.zero_grad(set_to_none=True)
        loss = torch.nn.functional.cross_entropy(m(x), y)
        loss.backward()
        torch.cuda.synchronize()
        scales.append(m.ctx.arena.bufs[("dp.scales",)].clone())
        losses.append(loss.item())
    assert len(m._graphs) == 1
    for i in range(3, 6):  # calls 3.. are replays
        assert not torch.equal(scales[i], scales[i - 1]), "replayed graph reused the previous stochastic-depth draw"
    assert len({round(l, 6) for l in losses}) == len(losses)
    assert int(m._dp_counter.item()) == 6 and int(m._drop_counter.item()) == 6


def test_slowfast_head_dropout_backward_uses_forward_mask(cuda_device):
    """Logits are linear in head.projection: with the dropout mask pinned (counter reset) the finite difference along a
    projection-weight direction is exact, so it equals <grad, direction> iff backward used the forward's mask."""
    from oracle import torch_oracle as TO
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.resnet import B200SlowFast
    cfg = get_cfg("SLOWFAST_8x8_R50", DATA={"NUM_FRAMES": 16, "TRAIN_CROP_SIZE": 64}, MODEL={"DROPOUT_RATE": 0.5},
                  B200={"CUDA_GRAPH": False})
    torch.manual_seed(0)
    m = B200SlowFast(cfg)
    m.load_state_dict(TO.fixture_state(m.state_dict(), 8))
    m = m.to(cuda_device).train()
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, 2, 4)]
    dl = torch.randn(2, 400, device=cuda_device)

    def f():
        if getattr(m, "_drop_counter", None) is not None:
            m._drop_counter.zero_()
        return (m(x) * dl).sum()

    f()
    m.zero_grad(set_to_none=True)
    f().backward()
    w = m.head.projection.weight
    gw = w.grad.detach().clone()
    assert (m._drop_mask == 0).any() and (m._drop_mask == 1).any()
    d = torch.randn_like(w) * 0.01
    with torch.no_grad():
        w.add_(d)
        lp = f().item()
        w.sub_(2 * d)
        lm = f().item()
        w.add_(d)
    fd, dd = (lp - lm) / 2, (gw * d).sum().item()
    print(f"slowfast head dropout: <grad, d> = {dd:.5e}, central difference = {fd:.5e}")
    assert abs(fd - dd) < 2e-3 * max(abs(dd), abs(fd)) + 1e-6
