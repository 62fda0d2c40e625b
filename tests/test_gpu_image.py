"""GPU: the ImageNet MViT / ViT recipes (PATCH_2D) on the engine - the cls-free token layout, spatial-only relative
positions, the joint position table and the norm-then-mean readout.

  * kernels at the image geometries against fp64 (or bitwise against the reference's fp32 arithmetic where the kernel
    does exactly that arithmetic), with determinism where the kernel promises it;
  * whole models against the unmodified reference (fp32 and fp64, same GPU, same fixture weights and images);
  * CUDA-graph replay against eager over AdamW steps (within the eager-vs-eager noise), and the unmodified train / test
    drivers on a synthetic image set.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _planes_value(hi, lo):
    return hi.double() + (lo.double() if lo is not None else 0.0)


# ============================================================================================ kernels
@pytest.mark.parametrize("name,kern,stride,out", [("kv", (1, 3, 3), (1, 4, 4), 14), ("q", (1, 3, 3), (1, 2, 2), 28),
                                                  ("q1", (1, 3, 3), (1, 1, 1), 56)])
def test_dwpool_without_cls_matches_fp64(name, kern, stride, out, cuda_device):
    """Depthwise pooling of MViTv2-T's first stage (56^2 tokens, one head of 96) with no cls row: forward, data gradient
    (both the gather and the scatter form) and weight gradient against fp64 conv3d."""
    from slowfast_b200 import ops
    B, Hn, hd, side = 2, 1, 96, 56
    Ltok, A = side * side, Hn * hd
    g = torch.Generator().manual_seed(out)
    src = torch.randn(B, Ltok, 3 * A, generator=g)
    bias = torch.randn(3 * A, generator=g)
    w = torch.randn(hd, 1, *kern, generator=g) * 0.3
    dout = torch.randn(B, Hn, out * out, hd, generator=g)
    s_d, b_d, w_d, do_d = (v.to(cuda_device) for v in (src, bias, w, dout))
    o = torch.full((B, Hn, out * out, hd), float("nan"), device=cuda_device)
    dsrc = torch.zeros(B, Ltok, 3 * A, device=cuda_device)
    geom = (B, Hn, hd, (1, side, side), (1, out, out), kern, stride)
    ops.dwpool_fwd(s_d, A, b_d, w_d, *geom, o, cls=False)
    x = (src[:, :, A:2 * A] + bias[A:2 * A]).double().view(B, side, side, Hn, hd).permute(0, 3, 4, 1, 2)
    x = x.reshape(B * Hn, hd, 1, side, side).requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    y = F.conv3d(x, w64, stride=stride, padding=[k // 2 for k in kern], groups=hd)
    want = y.reshape(B, Hn, hd, out * out).permute(0, 1, 3, 2)
    assert _rel(o.cpu().double(), want) < 1e-6
    dw = torch.full_like(w_d, float("nan"))
    wp = torch.empty(ops.dwpool_wgrad_blocks(B, Hn, (1, out, out)) * hd * math.prod(kern), device=cuda_device)
    ops.dwpool_bwd(s_d, A, b_d, w_d, *geom, do_d, dsrc, dw=dw, wpartials=wp, cls=False)
    want.backward(dout.double())
    gx = x.grad.view(B, Hn, hd, side * side).permute(0, 3, 1, 2).reshape(B, Ltok, A)
    got = dsrc.cpu().double()
    assert _rel(got[:, :, A:2 * A], gx) < 1e-6
    assert got[:, :, :A].abs().max() == 0 and got[:, :, 2 * A:].abs().max() == 0
    assert _rel(dw.cpu().double(), w64.grad) < 1e-5


def _bias_only(RQ, q_shape, k_shape, Lh):
    """fp64 RQ[q, ih] + RQ[q, Lh + iw] with the reference's index rule (attention.py:64-105), no cls row."""
    _, qh, qw = q_shape
    _, kh, kw = k_shape
    def dist(qn, kn):
        qr, kr = max(kn / qn, 1.0), max(qn / kn, 1.0)
        return (torch.arange(qn)[:, None] * qr - torch.arange(kn)[None, :] * kr + (kn - 1) * kr).long()
    ih, iw = dist(qh, kh), dist(qw, kw)
    BH = RQ.shape[0]
    rq = RQ.view(BH, qh, qw, -1)
    bh_ = torch.gather(rq[..., :Lh], 3, ih.view(1, qh, 1, kh).expand(BH, qh, qw, kh))
    bw_ = torch.gather(rq[..., Lh:], 3, iw.view(1, 1, qw, kw).expand(BH, qh, qw, kw))
    return (bh_[..., :, None] + bw_[..., None, :]).reshape(BH, qh * qw, kh * kw)


@pytest.mark.parametrize("cls", [0, 1])
def test_softmax_spatial_relpos_matches_fp64(cls, cuda_device):
    """MViTv2-T's first block: Nq 3136 (56^2) queries over Nk 196 (14^2) pooled keys with the spatial terms only (no Rt
    table).  Forward P and backward dS / dRQ against fp64 autograd of the same bias; with a cls row (cls = 1, the video
    spatial-only layout) the cls row / column carry no bias.  The fp64 formulation is checked against the reference's
    cal_rel_pos_spatial first."""
    from oracle import refshim
    from slowfast_b200 import ops
    BH, side, kside, hd = 2, 56, 14, 96
    Lq, Lk = side * side, kside * kside
    Nq, Nk = Lq + cls, Lk + cls
    Nkp = (Nk + 7) // 8 * 8
    Lh = Lw = 2 * side - 1
    Ltp = (Lh + Lw + 7) // 8 * 8
    g = torch.Generator().manual_seed(11 + cls)
    S = torch.randn(BH, Nq, Nk, generator=g, dtype=torch.float64)
    q = torch.randn(BH, Lq, hd, generator=g, dtype=torch.float64) * 0.3
    Rh, Rw = (torch.randn(Lh, hd, generator=g, dtype=torch.float64) * 0.3 for _ in range(2))
    RQ = torch.cat([q @ Rh.t(), q @ Rw.t()], -1)
    dP = torch.randn(BH, Nq, Nk, generator=g, dtype=torch.float64)
    if refshim.reference_available():
        refshim.install()
        from slowfast.models.attention import cal_rel_pos_spatial
        qr = torch.cat([torch.zeros(BH, cls, hd, dtype=torch.float64), q], 1).view(1, BH, Nq, hd)
        a = cal_rel_pos_spatial(S.clone().view(1, BH, Nq, Nk), qr, None, bool(cls), [1, side, side],
                                [1, kside, kside], Rh, Rw).view(BH, Nq, Nk)[:, cls:, cls:]
        torch.testing.assert_close(a, S[:, cls:, cls:] + _bias_only(RQ, (1, side, side), (1, kside, kside), Lh))
    rq_leaf = RQ.clone().requires_grad_(True)
    S_leaf = S.clone().requires_grad_(True)
    full = S_leaf + F.pad(_bias_only(rq_leaf, (1, side, side), (1, kside, kside), Lh), (cls, 0, cls, 0))
    P64 = torch.softmax(full, -1)
    P64.backward(dP)
    Sd = torch.zeros(BH, Nq, Nkp, device=cuda_device)
    Sd[..., :Nk] = S.float().to(cuda_device)
    rqd = torch.zeros(BH * Lq, Ltp, device=cuda_device)
    rqd[:, :Lh + Lw] = RQ.float().view(BH * Lq, -1).to(cuda_device)
    ph, plo = (torch.empty(BH, Nq, Nkp, dtype=torch.bfloat16, device=cuda_device) for _ in range(2))
    grids = dict(q_thw=(1, side, side), k_thw=(1, kside, kside), cls=bool(cls), spatial_only=True)
    P_planes = ops.Planes(ph, plo, 1, 1, 1, BH * Nq, Nkp)
    ops.softmax_relpos_fwd(Sd, P_planes, BH, Nq, Nk, rq=rqd, **grids)
    P = _planes_value(ph, plo).cpu()
    assert _rel(P[..., :Nk], P64.detach()) < 3e-5   # split-bf16 planes carry ~16 mantissa bits
    assert P[..., Nk:].abs().max() == 0
    dPd = torch.zeros(BH, Nq, Nkp, device=cuda_device)
    dPd[..., :Nk] = dP.float().to(cuda_device)
    dsh, dsl = (torch.empty(BH, Nq, Nkp, dtype=torch.bfloat16, device=cuda_device) for _ in range(2))
    drq = torch.full((BH * Lq, Ltp), float("nan"), device=cuda_device)
    ops.softmax_relpos_bwd(P_planes, dPd, ops.Planes(dsh, dsl, 1, 1, 1, BH * Nq, Nkp), BH, Nq, Nk, drq=drq, **grids)
    dS = _planes_value(dsh, dsl).cpu()
    assert _rel(dS[..., :Nk], S_leaf.grad) < 5e-5
    got = drq.cpu().double()
    assert _rel(got[:, :Lh + Lw], rq_leaf.grad.view(BH * Lq, -1)) < 5e-5
    assert got[:, Lh + Lw:].abs().max() == 0


@pytest.mark.parametrize("cls,pos", [(True, True), (False, True), (False, False)])
@pytest.mark.parametrize("b,l,e", [(2, 3136, 96), (3, 196, 768), (1, 5, 8)])
def test_tokens_assemble_joint_is_bitwise_the_reference_arithmetic(b, l, e, cls, pos, cuda_device):
    from slowfast_b200 import ops
    g = torch.Generator().manual_seed(l + e)
    y, bias, c = torch.randn(b, l, e, generator=g), torch.randn(e, generator=g), torch.randn(e, generator=g)
    p = torch.randn(1, l + int(cls), e, generator=g)
    yd, bd, cd, pd = (v.to(cuda_device) for v in (y, bias, c, p))
    out = torch.full((b, l + int(cls), e), float("nan"), device=cuda_device)
    ops.tokens_assemble_joint(yd, bd, cd if cls else None, pd if pos else None, b, l, e, out)
    want = y + bias                                                        # the patch embedding's conv + bias
    if cls:
        want = torch.cat([c.view(1, 1, e).expand(b, 1, e), want], 1)      # cat(cls_tokens, x)
    if pos:
        want = want + p                                                    # x += pos_embed
    assert torch.equal(out.cpu(), want)


@pytest.mark.parametrize("b,n,e", [(64, 3137, 96), (64, 197, 768), (3, 7, 8)])
def test_pos_embed_joint_bwd_matches_fp64_and_is_deterministic(b, n, e, cuda_device):
    from slowfast_b200 import ops
    dx = torch.randn(b, n, e, generator=torch.Generator().manual_seed(n))
    d = dx.to(cuda_device)
    outs = []
    for _ in range(2):
        dp = torch.full((n, e), float("nan"), device=cuda_device)
        ops.pos_embed_joint_bwd(d, b, n, e, dp)
        outs.append(dp.cpu())
    assert _rel(outs[0].double(), dx.double().sum(0)) < 1e-6
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("b,n,c", [(8, 49, 768), (2, 3136, 96), (3, 1, 8)])
def test_norm_then_mean_readout_forward_backward(b, n, c, cuda_device):
    """The default readout without cls (video_model_builder.py:1239-1241): LayerNorm on all b*n rows, per-image mean, and
    its backward (dmean / n to every row, then LayerNorm backward) against fp64 autograd; the mean is deterministic."""
    from slowfast_b200 import ops
    g = torch.Generator().manual_seed(n * c)
    x, dm = torch.randn(b, n, c, generator=g) * 2 + 0.3, torch.randn(b, c, generator=g)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    xd, dmd, gd, bd = (v.to(cuda_device) for v in (x, dm, gamma, beta))
    rows = b * n
    y = torch.empty(rows, c, device=cuda_device)
    mean, rstd = torch.empty(rows, device=cuda_device), torch.empty(rows, device=cuda_device)
    ops.layernorm_fwd(xd, c, rows, c, gd, bd, 1e-6, mean, rstd, out_f32=y)
    part = torch.empty(b * ops.segment_slabs(b, n) * c, device=cuda_device)
    outs = []
    for _ in range(2):
        o = torch.full((b, c), float("nan"), device=cuda_device)
        ops.token_mean_fwd(y, b, n, c, o, part, cls=False)
        outs.append(o.cpu())
    assert torch.equal(outs[0], outs[1])
    dn = torch.full((rows, c), float("nan"), device=cuda_device)
    ops.token_mean_bwd(dmd, b, n, c, dn, cls=False)
    dx, dg, db = (torch.empty(s, device=cuda_device) for s in ((rows, c), (c,), (c,)))
    lp = torch.empty(ops.colsum_blocks(rows) * 2 * c, device=cuda_device)
    ops.layernorm_bwd(dn, c, xd, c, rows, c, gd, mean, rstd, dx, c, dg, db, lp)
    xr = x.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    out = F.layer_norm(xr, (c,), gr, br, 1e-6).mean(1)
    out.backward(dm.double())
    assert _rel(outs[0].double(), out.detach()) < 1e-6
    assert _rel(dx.cpu().double().view(b, n, c), xr.grad) < 1e-5
    assert _rel(dg.cpu().double(), gr.grad) < 1e-5 and _rel(db.cpu().double(), br.grad) < 1e-5


def test_token_maxpool_without_cls_matches_max_pool(cuda_device):
    """The skip path of a Q-pooled block (kernel 3x3, stride 2 over 56^2 tokens) with no pass-through row."""
    from slowfast_b200 import ops
    B, C_, side, o = 2, 96, 56, 28
    x = torch.randn(B, side * side, C_, generator=torch.Generator().manual_seed(5))
    dout = torch.randn(B, o * o, C_, generator=torch.Generator().manual_seed(6))
    xd, dd = x.to(cuda_device), dout.to(cuda_device)
    out = torch.empty(B, o * o, C_, device=cuda_device)
    am = torch.empty(B, o * o, C_, dtype=torch.uint8, device=cuda_device)
    dx = torch.full((B, side * side, C_), float("nan"), device=cuda_device)
    geom = (B, C_, (1, side, side), (1, o, o), (1, 3, 3), (1, 2, 2))
    ops.token_maxpool_fwd(xd, *geom, out, am, cls=False)
    ops.token_maxpool_bwd(dd, am, *geom, dx, cls=False)
    xr = x.double().view(B, side, side, C_).permute(0, 3, 1, 2).requires_grad_(True)
    y = F.max_pool2d(xr, 3, 2, 1)
    assert torch.equal(out.cpu().double(), y.detach().permute(0, 2, 3, 1).reshape(B, o * o, C_))
    y.backward(dout.double().view(B, o, o, C_).permute(0, 3, 1, 2))
    assert _rel(dx.cpu().double(), xr.grad.permute(0, 2, 3, 1).reshape(B, side * side, C_)) < 1e-6


# ============================================================================================ whole models vs reference
def _fixture(template, seed=3):
    from oracle import torch_oracle as TO
    state = TO.fixture_state(template, seed)
    for i, k in enumerate(template):   # position tables at the scale of the cls token, so they matter to the output
        if k.startswith("pos_embed"):
            state[k] = torch.randn(template[k].shape, generator=torch.Generator().manual_seed(seed * 7919 + i)) * 0.2
    return state


def _images(batch, crop, seed):
    return [torch.randn(batch, 3, crop, crop, generator=torch.Generator().manual_seed(seed))]


_B_MVIT = ["MVIT.DEPTH", 24, "MVIT.DIM_MUL", [[2, 2.0], [5, 2.0], [21, 2.0]],
           "MVIT.HEAD_MUL", [[2, 2.0], [5, 2.0], [21, 2.0]], "MVIT.POOL_KV_STRIDE_ADAPTIVE", [1, 4, 4],
           "MVIT.POOL_KV_STRIDE", [], "MVIT.POOL_Q_STRIDE",
           [[i, 1, 2, 2] if i in (2, 5, 21) else [i, 1, 1, 1] for i in range(24)]]
MODEL_CASES = [  # (yaml, crop, extra overrides)
    ("ImageNet/MVITv2_T.yaml", 224, []),
    ("ImageNet/MVITv2_S.yaml", 224, []),
    ("ImageNet/MVITv2_S.yaml", 64, _B_MVIT),                 # the composed MViTv2-B, all 24 blocks, at 64^2
    ("ImageNet/MVIT_B_16_CONV.yaml", 224, []),               # joint pos_embed [1, 1 + 56*56, 96], cls readout
    ("masked_ssl/in1k_VIT_B_MaskFeat_FT.yaml", 224, []),     # 197 tokens, joint pos_embed, mean readout
    ("masked_ssl/in1k_VIT_L_MaskFeat_FT.yaml", 224, ["MVIT.DEPTH", 2]),
]
MODEL_IDS = ["mvitv2_t", "mvitv2_s", "mvitv2_b_composed", "mvit_b_16", "vit_b_in1k", "vit_l_in1k_2blk"]


@pytest.mark.parametrize("fast", [False, True], ids=["parity", "fast"])
@pytest.mark.parametrize("yaml,crop,extra", MODEL_CASES, ids=MODEL_IDS)
def test_image_model_step_and_eval_match_reference(yaml, crop, extra, fast, cuda_device):
    """One training step and an eval forward of the engine and of the unmodified reference (fp32, same GPU, same fixture
    weights and images), with test_gpu_vit.py's bounds: parity mode logits within 1e-3 max-abs relative with argmax
    exact and gradients against fp64 within max(8x the reference's own fp32 error, 0.15) per parameter; fast mode
    within 2x the reference's bf16-autocast error (floor 1e-2)."""
    import copy
    from oracle import refshim
    from slowfast_b200.nets.mvit import B200MViT
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    cfg = refshim.load_cfg(yaml, ["DATA.TRAIN_CROP_SIZE", crop, "DATA.TEST_CROP_SIZE", crop, "MODEL.DROPOUT_RATE", 0.0,
                                  "MVIT.DROPPATH_RATE", 0.0] + list(extra))
    if fast:
        cfg["B200"] = {"NSPLIT": 1}
    batch = 2
    ref = refshim.build_reference_model(cfg)
    state = _fixture(ref.state_dict())
    ref.load_state_dict(state)
    ref = ref.to(cuda_device).train()
    mine = B200MViT(cfg)
    mine.load_state_dict(state)
    mine = mine.to(cuda_device).train()
    x = [t.to(cuda_device) for t in _images(batch, crop, 4)]
    dl = torch.randn(batch, cfg.MODEL.NUM_CLASSES, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    lr = ref([t.clone() for t in x])
    lr.backward(dl)
    lm = mine(x)
    lm.backward(dl)
    torch.cuda.synchronize()
    rel_max = ((lm - lr).abs().max() / lr.abs().max()).item()
    rm = dict(ref.named_parameters())
    per = {k: _rel(p.grad.double(), rm[k].grad.double()) for k, p in mine.named_parameters()}
    worst = max(per, key=per.get)
    if not fast:
        r64 = copy.deepcopy(ref).double()
        r64.zero_grad(set_to_none=True)
        r64([t.double() for t in x]).backward(dl.double())
        g64 = {k: p.grad for k, p in r64.named_parameters()}
        del r64
        med = sorted(g.norm().item() for g in g64.values())[len(g64) // 2]
        zero = {k for k, g in g64.items() if g.norm().item() < 1e-6 * med}
        err = {k: _rel(p.grad.double(), g64[k]) for k, p in mine.named_parameters() if k not in zero}
        env = {k: _rel(rm[k].grad.double(), g64[k]) for k in err}
        ratio = {k: err[k] / max(8 * env[k], 0.15) for k in err}
        wk = max(ratio, key=ratio.get)
        em_, en_ = sorted(err.values())[len(err) // 2], sorted(env.values())[len(env) // 2]
        print(f"  vs fp64: grad rel-L2 median {em_:.2e} (reference fp32 {en_:.2e}); worst {wk} {err[wk]:.2e} "
              f"(reference fp32 {env[wk]:.2e}); zero in exact arithmetic: {sorted(zero)}")
    ref.eval()
    mine.eval()
    with torch.no_grad():
        er = ref([t.clone() for t in x])
        em = mine(x)
        if fast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                ref.train()
                lr_bf = ref([t.clone() for t in x]).float()
                ref.eval()
                er_bf = ref([t.clone() for t in x]).float()
    tag = f"{yaml.split('/')[-1]} {crop}^2 {extra[:2]} {'fast' if fast else 'parity'}"
    print(f"{tag}: logits max-rel {rel_max:.2e} rel-L2 {_rel(lm, lr):.2e}; grad rel-L2 max {per[worst]:.2e} ({worst}); "
          f"eval rel-L2 {_rel(em, er):.2e}")
    if fast:
        env_t, env_e = _rel(lr_bf, lr.detach()), _rel(er_bf, er)
        print(f"  reference bf16-autocast error: train {env_t:.2e}, eval {env_e:.2e}")
        assert _rel(lm, lr) < max(2 * env_t, 1e-2)
        assert _rel(em, er) < max(2 * env_e, 1e-2)
        return
    assert rel_max < 1e-3 and torch.equal(lm.argmax(1), lr.argmax(1))
    assert ratio[wk] < 1.0, (wk, err[wk], env[wk])
    assert em_ < max(8 * en_, 0.15), (em_, en_)
    for k in zero:
        assert mine.get_parameter(k).grad.norm().item() < 1e-3 * med, k
    assert ((em - er).abs().max() / er.abs().max()).item() < 1e-3 and torch.equal(em.argmax(1), er.argmax(1))


# ============================================================================================ replay
def _t_model(graphs, dev):
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    cfg = get_cfg("MVITv2_T", MVIT={"DROPPATH_RATE": 0.0}, B200={"NSPLIT": 3, "CUDA_GRAPH": graphs})
    torch.manual_seed(0)
    model = B200MViT(cfg)
    model.load_state_dict(_fixture(model.state_dict(), 7))
    return cfg, model.to(dev).train()


def _steps(model, cfg, dev, n_steps, batch=2):
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.05)
    outs = []
    for s in range(n_steps):
        x = _images(batch, cfg.DATA.TRAIN_CROP_SIZE, 100 + s)
        y = torch.randint(0, cfg.MODEL.NUM_CLASSES, (batch,), generator=torch.Generator().manual_seed(105 + s))
        opt.zero_grad(set_to_none=True)
        logits = model([t.to(dev) for t in x])
        F.cross_entropy(logits, y.to(dev)).backward()
        opt.step()
        outs.append(logits.detach().cpu())
    torch.cuda.synchronize()
    return outs


def test_mvitv2_t_image_replay_matches_eager_over_adamw_steps(cuda_device):
    """MViTv2-T at 224^2 over five AdamW steps: the CUDA-graph replay agrees with eager within the test_gpu_replay.py
    bound, max(2e-4, 5x the eager-vs-eager noise).  The step is not bitwise deterministic: the split-K weight gradients
    and the pooling weight gradient add partial sums with float atomics, as on the video path."""
    steps = 5
    cfg, mg = _t_model(True, cuda_device)
    _, me = _t_model(False, cuda_device)
    _, me2 = _t_model(False, cuda_device)
    og, oe, oe2 = (_steps(m, cfg, cuda_device, steps) for m in (mg, me, me2))
    key = list(mg._graphs)
    assert len(key) == 1 and mg._graphs[key[0]].bwd_graph is not None, "the graphed model never switched to replay"
    assert torch.equal(og[0], oe[0])   # the first forward precedes every atomic-summed gradient
    for s in range(steps):
        rel = ((og[s] - oe[s]).abs().max() / oe[s].abs().max()).item()
        noise = ((oe2[s] - oe[s]).abs().max() / oe[s].abs().max()).item()
        print(f"step {s}: logits replay vs eager {rel:.2e} (eager vs eager {noise:.2e})")
        assert rel < max(2e-4, 5 * noise), (s, rel, noise)


# ============================================================================================ unmodified drivers
def _register_image_dataset():
    from slowfast.datasets.build import DATASET_REGISTRY
    if "Syntheticimage" in DATASET_REGISTRY._obj_map:
        return

    class Syntheticimage(torch.utils.data.Dataset):
        """Seeded images: item i is randn(3, crop, crop), returned as the ImageNet loader does
        (datasets/imagenet.py:265: [im], label, index, torch.Tensor(), {})."""

        def __init__(self, cfg, mode, num_retries=0):
            self.cfg, self.mode = cfg, mode
            self.views = cfg.TEST.NUM_ENSEMBLE_VIEWS * cfg.TEST.NUM_SPATIAL_CROPS if mode == "test" else 1
            self._n = 12 * self.views

        @property
        def num_videos(self):
            return self._n

        def __len__(self):
            return self._n

        def __getitem__(self, i):
            cfg = self.cfg
            crop = cfg.DATA.TEST_CROP_SIZE if self.mode == "test" else cfg.DATA.TRAIN_CROP_SIZE
            g = torch.Generator().manual_seed(10007 * i + {"train": 1, "val": 2, "test": 3}[self.mode])
            im = torch.randn(3, crop, crop, generator=g)
            return [im], (i // self.views) % cfg.MODEL.NUM_CLASSES, i, torch.Tensor(), {}

    DATASET_REGISTRY._do_register("Syntheticimage", Syntheticimage)


@pytest.fixture
def _stock_registry_back():
    yield
    import driver_harness as H
    if H.setup_reference() is not None:
        H.use_engine(False)


def test_unmodified_train_and_test_drivers_run_mvitv2_t_images(cuda_device, _stock_registry_back):
    """tools/train_net.py / test_net.py, unmodified, on a shrunk MViTv2-T (4 blocks, 64^2) with seeded images: engine and
    stock losses within 1e-3 relative on the first iteration and 1e-2 after."""
    import driver_harness as H
    if H.setup_reference() is None:
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    _register_image_dataset()
    over = ["TRAIN.DATASET", "syntheticimage", "TEST.DATASET", "syntheticimage", "MODEL.DROPOUT_RATE", 0.0,
            "MVIT.DROPPATH_RATE", 0.0, "MIXUP.ENABLE", False, "AUG.ENABLE", False, "MODEL.LOSS_FUNC", "cross_entropy",
            "SOLVER.BASE_LR", 1e-4, "MVIT.DEPTH", 4, "MVIT.DIM_MUL", [[1, 2.0], [3, 2.0]],
            "MVIT.HEAD_MUL", [[1, 2.0], [3, 2.0]], "MVIT.POOL_KV_STRIDE", [[0, 1, 4, 4], [1, 1, 2, 2]],
            "MVIT.POOL_Q_STRIDE", [[1, 1, 2, 2], [3, 1, 2, 2]], "TEST.ENABLE", True]
    runs = {}
    for engine in (False, True):
        H.use_engine(engine)
        cfg = H.driver_cfg("ImageNet/MVITv2_T.yaml", 1, over, batch=4)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        rec_train, _ = H.run_train(cfg)
        rec_test, result = H.run_test(cfg)
        runs[engine] = (rec_train, rec_test, result)
    from slowfast.models import build_model
    assert type(build_model(cfg)).__name__ == "B200MViT"
    (st_train, st_test, _), (en_train, en_test, result) = runs[False], runs[True]
    assert len(en_train["train"]) == len(st_train["train"]) == 3
    for i, (a, b) in enumerate(zip(en_train["train"], st_train["train"])):
        rel = abs(a["loss"] - b["loss"]) / abs(b["loss"])
        print(f"iter {i}: loss engine {a['loss']:.6f} stock {b['loss']:.6f} (rel {rel:.1e})")
        assert rel < (1e-3 if i == 0 else 1e-2), (i, a, b)
    assert len(en_test["test"]) == len(st_test["test"]) > 0
    for a, b in zip(en_test["test"], st_test["test"]):
        assert torch.equal(a["ids"], b["ids"])
        assert ((a["preds"] - b["preds"]).abs().max() / b["preds"].abs().max()).item() < 5e-2
