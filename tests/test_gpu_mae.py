"""GPU: MAE pre-training (k400_VIT_{B,L,H}_16x4_MAE_PT) on the engine.

  * kernels: the masking against torch.argsort(noise, stable=True) and the reference's own _mae_random_masking, the
    kept-patch embedding against F.conv3d + gather, the encoder / decoder token assembly bitwise against the same fp32
    arithmetic (backward against fp64, and bitwise reproducible), the pixel targets against fp64;
  * whole models against the unmodified reference (same GPU, same fixture weights, clips and seed, so the same mask):
    predictions, labels, the MSE loss and every parameter gradient (against the reference evaluated in fp64);
  * CUDA-graph replay against eager over AdamW steps, a fresh mask every step;
  * the unmodified train driver, and MAE pre-training followed by ViT-B fine-tuning from the checkpoint it wrote.
"""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _lib():
    from slowfast_b200 import lib as L
    return L, L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _restate_masking(noise, keep):
    """_mae_random_masking (masked.py:283-317) with a stable sort, plus the removed rows of the [B, L+1] decoder sequence."""
    B, Lt = noise.shape
    ids_shuffle = torch.argsort(noise, dim=1, stable=True)
    ids_restore = torch.argsort(ids_shuffle, dim=1, stable=True)
    mask = torch.ones(B, Lt, device=noise.device)
    mask[:, :keep] = 0
    mask = torch.gather(mask, 1, ids_restore)
    b, l = mask.bool().nonzero(as_tuple=True)   # row-major: clip 0 ascending, then clip 1 ...
    return ids_shuffle[:, :keep], ids_restore, mask, (b * (Lt + 1) + 1 + l)


def _run_masking(noise, keep):
    from slowfast_b200 import ops
    B, Lt = noise.shape
    dev = noise.device
    ids_keep = torch.full((B, keep), -1, dtype=torch.int32, device=dev)
    ids_restore = torch.full((B, Lt), -1, dtype=torch.int32, device=dev)
    mask = torch.full((B, Lt), float("nan"), device=dev)
    rows = torch.full((B * (Lt - keep),), -1, dtype=torch.int32, device=dev)
    ops.mae_random_masking(noise, keep, ids_keep, ids_restore, mask, rows)
    return ids_keep, ids_restore, mask, rows


@pytest.mark.parametrize("ties", ["rand", "ties"])
@pytest.mark.parametrize("b,l", [(3, 32), (32, 64), (32, 1568), (5, 1568)])
def test_masking_matches_stable_argsort(b, l, ties, cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(l + b)
    keep = int(l * (1 - 0.9)) if l > 64 else l // 4
    noise = torch.rand(b, l, device=cuda_device, generator=g)
    if ties == "ties":
        # coarse values everywhere (many ties), and a tie group straddling the keep boundary of every clip
        noise = (noise * 16).floor() / 16
        order = torch.argsort(noise, dim=1, stable=True)
        lo, hi = max(keep - 3, 0), min(keep + 3, l)
        noise.scatter_(1, order[:, lo:hi], noise.gather(1, order[:, keep:keep + 1]).expand(b, hi - lo).contiguous())
    got = _run_masking(noise, keep)
    want = _restate_masking(noise, keep)
    for name, a, w in zip(("ids_keep", "ids_restore", "mask", "rows"), got, want):
        assert torch.equal(a.long() if a.dtype == torch.int32 else a, w.long() if w.dtype != torch.float32 else w), name


def test_masking_matches_reference_at_1568_tokens(cuda_device):
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    cfg = refshim.load_cfg("masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml", ["MVIT.DEPTH", 1, "MASK.PRETRAIN_DEPTH", [0],
                                                                      "MASK.DECODER_DEPTH", 1])
    ref = refshim.build_reference_model(cfg).to(cuda_device)
    B, Lt = 32, 1568
    keep = int(Lt * (1 - cfg.AUG.MASK_RATIO))
    for seed in range(4):
        torch.manual_seed(seed)
        _, mask, ids_restore, ids_keep = ref._mae_random_masking(torch.zeros(B, Lt, 1, device=cuda_device),
                                                                 cfg.AUG.MASK_RATIO)
        torch.manual_seed(seed)
        noise = torch.rand(B, Lt, device=cuda_device)
        k, r, m, _ = _run_masking(noise, keep)
        assert torch.equal(k.long(), ids_keep) and torch.equal(r.long(), ids_restore) and torch.equal(m, mask), seed


def test_masking_rejects_too_many_tokens(cuda_device):
    L, lib = _lib()
    assert lib.sfb_mae_max_tokens() == 4096
    t = torch.zeros(8192, device=cuda_device)
    assert lib.sfb_mae_random_masking(t.data_ptr(), 1, 4097, 409, *([t.data_ptr()] * 4), _st()) != 0
    assert b"l <= 4096" in lib.sfb_last_error()


@pytest.mark.parametrize("nsplit", [3, 1])
def test_patchify_gather_gemm_and_wgrad_match_conv3d(nsplit, cuda_device):
    from slowfast_b200 import ops
    from slowfast_b200.engine import Ctx
    from slowfast_b200.ops import Planes
    g = torch.Generator().manual_seed(5)
    B, cin, k = 3, 3, (2, 16, 16)
    shape = (B, cin, 4, 64, 48)
    x = torch.randn(*shape, generator=g)
    E, K = 64, cin * 2 * 16 * 16
    w = torch.randn(E, cin, *k, generator=g) * K ** -0.5
    Lt = 2 * 4 * 3
    nkeep = 5
    keep = torch.stack([torch.randperm(Lt, generator=g)[:nkeep] for _ in range(B)]).int()
    ctx = Ctx(nsplit)
    ctx.device = cuda_device
    rows = B * nkeep
    s = ctx.storage(("rows",), 1, 1, 1, rows, K)
    xr = Planes(s.hi, s.lo, 1, 1, 1, rows, K, 0)
    xd, kd = x.to(cuda_device), keep.to(cuda_device)
    ops.patchify_gather(xd, k, kd, nkeep, xr)
    fm = ops.alloc_filter(E, 1, K, nsplit, cuda_device)
    ops.filter_pack(w.to(cuda_device).view(E, K), fm)
    y = torch.empty(rows, E, device=cuda_device)
    geom = ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, rows))
    ops.conv_igemm(xr, fm, geom, y, (rows * E, rows * E, rows * E, E), nsplit=nsplit)
    full = F.conv3d(x.double(), w.double(), stride=k).flatten(2).transpose(1, 2)   # [B, Lt, E]
    want = torch.gather(full, 1, keep.long().unsqueeze(-1).expand(B, nkeep, E)).reshape(rows, E)
    tol = 1e-5 if nsplit == 3 else 1e-2
    assert _rel(y.cpu().double(), want) < tol
    dy = torch.randn(rows, E, generator=g)
    ds = ctx.storage(("dy",), 1, 1, 1, rows, E)
    dyp = Planes(ds.hi, ds.lo, 1, 1, 1, rows, E, 0)
    ops.split_planes(dy.to(cuda_device).contiguous(), dyp)
    gw = torch.zeros(E, K, device=cuda_device)
    ops.conv_wgrad(xr, dyp, geom, gw, nsplit=nsplit)
    xv = x.double().unfold(2, 2, 2).unfold(3, 16, 16).unfold(4, 16, 16).permute(0, 2, 3, 4, 1, 5, 6, 7).reshape(B, Lt, K)
    xm = torch.gather(xv, 1, keep.long().unsqueeze(-1).expand(B, nkeep, K)).reshape(rows, K)
    assert _rel(gw.cpu().double(), dy.double().t() @ xm) < tol
    # a null table is sfb_patchify, bitwise
    s2 = ctx.storage(("rows2",), 1, 1, 1, B * Lt, K)
    s3 = ctx.storage(("rows3",), 1, 1, 1, B * Lt, K)
    ops.patchify_gather(xd, k, None, 0, Planes(s2.hi, s2.lo, 1, 1, 1, B * Lt, K, 0))
    ops.patchify(xd, k, Planes(s3.hi, s3.lo, 1, 1, 1, B * Lt, K, 0))
    assert torch.equal(s2.hi, s3.hi) and (s2.lo is None or torch.equal(s2.lo, s3.lo))


def _mask_setup(b, lt, keep, dev, seed):
    noise = torch.rand(b, lt, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)
    return _run_masking(noise, keep)


@pytest.mark.parametrize("b,t,hw,e,keep", [(4, 8, 196, 768, 156), (3, 2, 16, 40, 3)])
def test_encoder_assembly_forward_bitwise_and_backward(b, t, hw, e, keep, cuda_device):
    from slowfast_b200 import ops
    lt = t * hw
    ids_keep, ids_restore, _, _ = _mask_setup(b, lt, keep, cuda_device, 11)
    g = torch.Generator().manual_seed(hw)
    y, bias, cls = torch.randn(b, keep, e, generator=g), torch.randn(e, generator=g), torch.randn(e, generator=g)
    ps, pt, pc = torch.randn(hw, e, generator=g), torch.randn(t, e, generator=g), torch.randn(e, generator=g)
    d = [v.to(cuda_device) for v in (y, bias, cls, ps, pt, pc)]
    out = torch.empty(b, keep + 1, e, device=cuda_device)
    ops.tokens_assemble_keep(*d, ids_keep, b, keep, lt, hw, e, out)
    # masked.py:340-371 in fp32: cat(cls, x_masked) + cat(pc, gather(ps.repeat(t) + pt.repeat_interleave(hw), ids_keep))
    pos = (d[3].repeat(t, 1) + d[4].repeat_interleave(hw, dim=0)).unsqueeze(0).expand(b, lt, e)
    pos = torch.gather(pos, 1, ids_keep.long().unsqueeze(-1).expand(b, keep, e))
    want = torch.cat([d[2].view(1, 1, e).expand(b, 1, e), d[0] + d[1]], 1) + \
        torch.cat([d[5].view(1, 1, e).expand(b, 1, e), pos], 1)
    assert torch.equal(out, want)
    # backward: scatter onto the dense grid, then the separable table gradients
    dx = torch.randn(b, keep + 1, e, generator=g).to(cuda_device)
    outs = []
    for _ in range(2):
        dense = torch.full((b, lt + 1, e), float("nan"), device=cuda_device)
        ops.tokens_scatter_keep(dx, ids_restore, b, keep, lt, e, dense)
        outs.append(dense)
    want = torch.zeros(b, lt + 1, e, device=cuda_device)
    want[:, 0] = dx[:, 0]
    want[:, 1:].scatter_(1, ids_keep.long().unsqueeze(-1).expand(b, keep, e), dx[:, 1:])
    assert torch.equal(outs[0], want) and torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("b,lt,c,keep", [(4, 1568, 512, 156), (3, 32, 40, 3)])
def test_decoder_assembly_forward_bitwise_backward_fp64_deterministic(b, lt, c, keep, cuda_device):
    from slowfast_b200 import ops
    ids_keep, ids_restore, mask, rows = _mask_setup(b, lt, keep, cuda_device, 13)
    g = torch.Generator().manual_seed(lt)
    z, bias = torch.randn(b, keep + 1, c, generator=g), torch.randn(c, generator=g)
    mtok, pos = torch.randn(c, generator=g), torch.randn(lt + 1, c, generator=g)
    zd, bd, md, pd = (v.to(cuda_device) for v in (z, bias, mtok, pos))
    out = torch.empty(b, lt + 1, c, device=cuda_device)
    ops.decoder_assemble(zd, bd, md, pd, ids_restore, b, keep, lt, c, out)
    # masked.py:396-436 in fp32
    x = zd + bd
    x_ = torch.cat([x[:, 1:], md.view(1, 1, c).expand(b, lt - keep, c)], 1)
    x_ = torch.gather(x_, 1, ids_restore.long().unsqueeze(-1).expand(b, lt, c))
    want = torch.cat([x[:, :1], x_], 1) + pd
    assert torch.equal(out, want)
    dx = torch.randn(b, lt + 1, c, generator=g)
    dxd = dx.to(cuda_device)
    part = torch.empty(ops.segment_slabs(1, b * (lt - keep)) * c, device=cuda_device)
    res = []
    for _ in range(2):
        dz = torch.full((b, keep + 1, c), float("nan"), device=cuda_device)
        dpos = torch.full((lt + 1, c), float("nan"), device=cuda_device)
        dm = torch.full((c,), float("nan"), device=cuda_device)
        ops.decoder_assemble_bwd(dxd, ids_keep, rows, b, keep, lt, c, dz, dpos, dm, part)
        res.append((dz.cpu(), dpos.cpu(), dm.cpu()))
    zr, mr, pr = z.double().requires_grad_(True), mtok.double().requires_grad_(True), pos.double().requires_grad_(True)
    ir = ids_restore.long().cpu()
    xr_ = torch.cat([zr[:, 1:], mr.view(1, 1, c).expand(b, lt - keep, c)], 1)
    xr = torch.cat([zr[:, :1], torch.gather(xr_, 1, ir.unsqueeze(-1).expand(b, lt, c))], 1) + pr
    xr.backward(dx.double())
    assert _rel(res[0][0].double(), zr.grad) < 1e-6
    assert _rel(res[0][1].double(), pr.grad) < 1e-6
    assert _rel(res[0][2].double(), mr.grad) < 1e-6
    assert all(torch.equal(a, w) for a, w in zip(res[0], res[1]))


@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("time_stride_loss", [True, False])
def test_pixel_targets_match_fp64(norm, time_stride_loss, cuda_device):
    from slowfast_b200 import ops
    B, C, T, H, W, ts, p = 3, 3, 8, 64, 48, 2, 16
    x = torch.randn(B, C, T, H, W, generator=torch.Generator().manual_seed(3))
    x[1, :, 4:6, 16:32, 32:48] = 0.25      # a constant patch (zero variance) in both target layouts
    lt = (T // ts) * (H // p) * (W // p)
    keep = lt // 4
    _, _, mask, rows = _mask_setup(B, lt, keep, cuda_device, 17)
    mask[1] = 1.0   # (force the constant patch's token, clip 1 entirely, into the selection)
    b, l = mask.bool().nonzero(as_tuple=True)
    rows = (b * (lt + 1) + 1 + l).int()
    u = 1 if time_stride_loss else ts
    out = torch.empty(rows.numel(), u * p * p * C, device=cuda_device)
    ops.pixel_targets(x.to(cuda_device), ts, u, p, rows, norm, out)
    # _get_pixel_label_3d (masked.py:212-230) in fp64
    xf = x.double()[:, :, ::ts] if time_stride_loss else x.double()
    t = xf.shape[2] // u
    lab = xf.reshape(B, C, t, u, H // p, p, W // p, p)
    lab = torch.einsum("nctuhpwq->nthwupqc", lab).reshape(B, t * (H // p) * (W // p), u * p * p * C)
    lab = lab[mask.cpu().bool()]
    if norm:
        lab = (lab - lab.mean(-1, keepdim=True)) / (lab.var(-1, keepdim=True) + 1e-6) ** 0.5
    assert (out.cpu().double() - lab).abs().max().item() < 1e-5 * max(1.0, lab.abs().max().item())


# ============================================================================================ whole models vs reference
def _fixture(template, seed=3):
    from oracle import torch_oracle as TO
    state = TO.fixture_state(template, seed)
    for i, k in enumerate(template):   # position tables and the mask token at the scale of the tokens
        if k.startswith("pos_embed") or k in ("decoder_pos_embed", "mask_token"):
            state[k] = torch.randn(template[k].shape, generator=torch.Generator().manual_seed(seed * 7919 + i)) * 0.2
    return state


def _engine_mask(model, B):
    return model.ctx.buf(("mae.mask",), (B, model.n_tokens)).clone()


MODEL_CASES = [  # (yaml, frames, crop, extra overrides)
    ("masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml", 4, 64, []),
    ("masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml", 16, 224, []),
    # ViT-L / ViT-H encoders shortened to two blocks at the recipe's clip, the full 4-block decoder
    ("masked_ssl/k400_VIT_L_16x4_MAE_PT.yaml", 16, 224, ["MVIT.DEPTH", 2, "MASK.PRETRAIN_DEPTH", [1]]),
    ("masked_ssl/k400_VIT_H_16x4_MAE_PT.yaml", 16, 224, ["MVIT.DEPTH", 2, "MASK.PRETRAIN_DEPTH", [1]]),
]


@pytest.mark.parametrize("fast", [False, True], ids=["parity", "fast"])
@pytest.mark.parametrize("yaml,frames,crop,extra", MODEL_CASES)
def test_model_step_matches_reference(yaml, frames, crop, extra, fast, cuda_device):
    """One training step (MSE loss of MultipleMSELoss) of the engine and of the unmodified reference (fp32, same GPU,
    same fixture weights, clip and seed), then a second forward.  The two masks are compared first.  Parity: predictions
    and loss 1e-3 max-abs relative, labels 1e-5; gradients against the reference in fp64 within max(8x the reference's
    own fp32 error, 0.15), the median within max(8x the median envelope, 0.15).  Fast mode: predictions within 2x the
    reference's bf16-autocast error (floor 1e-2)."""
    from oracle import refshim
    from oracle import torch_oracle as TO
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    cfg = refshim.load_cfg(yaml, ["DATA.NUM_FRAMES", frames, "DATA.TRAIN_CROP_SIZE", crop, "DATA.TEST_CROP_SIZE", crop]
                           + list(extra))
    if fast:
        cfg["B200"] = {"NSPLIT": 1}
    batch = 2
    ref = refshim.build_reference_model(cfg)
    state = _fixture(ref.state_dict())
    ref.load_state_dict(state)
    ref = ref.to(cuda_device).train()
    mine = B200MaskMViT(cfg)
    mine.load_state_dict(state)
    mine = mine.to(cuda_device).train()
    x = TO.synthetic_inputs(cfg, batch, 4)[0].to(cuda_device)

    def run(model, inp, seed):
        torch.manual_seed(seed)
        preds, labels = model([inp])
        return preds[0], labels[0][0], F.mse_loss(preds[0], labels[0][0])

    torch.manual_seed(21)
    _, ref_mask, _, _ = ref._mae_random_masking(torch.zeros(batch, mine.n_tokens, 1, device=cuda_device),
                                                cfg.AUG.MASK_RATIO)
    pm, lm, lossm = run(mine, x, 21)
    assert torch.equal(_engine_mask(mine, batch), ref_mask), "engine and reference drew different masks"
    pr, lr, lossr = run(ref, x.clone(), 21)
    lossr.backward()
    lossm.backward()
    torch.cuda.synchronize()
    assert pm.shape == pr.shape
    rel_max = ((pm - pr).abs().max() / pr.abs().max()).item()
    rel_lab = ((lm - lr).abs().max() / lr.abs().max()).item()
    rel_loss = abs(lossm.item() - lossr.item()) / abs(lossr.item())
    rm = dict(ref.named_parameters())
    per = {k: _rel(p.grad.double(), rm[k].grad.double()) for k, p in mine.named_parameters()}
    rels = sorted(per.values())
    worst = max(per, key=per.get)
    tag = f"{yaml.split('/')[-1]} {frames}x{crop}^2 {extra} {'fast' if fast else 'parity'}"
    print(f"{tag}: pred max-rel {rel_max:.2e} rel-L2 {_rel(pm, pr):.2e}; labels {rel_lab:.2e}; loss {rel_loss:.2e}; "
          f"grad rel-L2 median {rels[len(rels) // 2]:.2e} max {per[worst]:.2e} ({worst})")
    # a second forward: a new mask, the same agreement
    with torch.no_grad():
        pm2, _, _ = run(mine, x, 22)
        pr2, _, _ = run(ref, x.clone(), 22)
    if fast:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            pb, _, _ = run(ref, x.clone(), 21)
        env = _rel(pb.float(), pr.detach())
        print(f"  reference bf16-autocast error {env:.2e}; engine {_rel(pm, pr):.2e}")
        assert _rel(pm, pr) < max(2 * env, 1e-2)
        assert _rel(pm2, pr2) < max(2 * env, 1e-2)
        assert rel_lab < 1e-5
        return
    r64 = copy.deepcopy(ref).double()
    r64.zero_grad(set_to_none=True)
    torch.manual_seed(21)
    p64, labels64 = r64([x.double()])
    F.mse_loss(p64[0], labels64[0][0]).backward()
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
    assert rel_max < 1e-3 and rel_loss < 1e-3 and rel_lab < 1e-5
    assert ((pm2 - pr2).abs().max() / pr2.abs().max()).item() < 1e-3
    assert ratio[wk] < 1.0, (wk, err[wk], env[wk])
    assert em_ < max(8 * en_, 0.15), (em_, en_)
    for k in zero:
        assert mine.get_parameter(k).grad.norm().item() < 1e-3 * med, k


# ============================================================================================ replay
def _mae_model(graphs, dev):
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    cfg = get_cfg("VIT_B_16x4_MAE_PT", DATA={"NUM_FRAMES": 4, "TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64},
                  MVIT={"DEPTH": 3}, MASK={"PRETRAIN_DEPTH": [2]}, B200={"NSPLIT": 3, "CUDA_GRAPH": graphs})
    torch.manual_seed(0)
    model = B200MaskMViT(cfg)
    model.load_state_dict(_fixture(model.state_dict(), 7))
    return cfg, model.to(dev).train()


def _steps(model, cfg, dev, n_steps, batch=4):
    from oracle import torch_oracle as TO
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    outs, masks = [], []
    for s in range(n_steps):
        x = TO.synthetic_inputs(cfg, batch, 100 + s)[0].to(dev)
        opt.zero_grad(set_to_none=True)
        torch.manual_seed(300 + s)
        preds, labels = model([x])
        F.mse_loss(preds[0], labels[0][0]).backward()
        opt.step()
        outs.append(preds[0].detach().cpu())
        masks.append(_engine_mask(model, batch).cpu())
    torch.cuda.synchronize()
    return outs, masks


def test_mae_replay_matches_eager_over_steps(cuda_device):
    """Eager and CUDA-graph replay give bitwise identical predictions at every one of five AdamW steps; the mask changes
    every step and is the one torch.rand draws eagerly from the step's seed."""
    steps, batch = 5, 4
    cfg, mg = _mae_model(True, cuda_device)
    _, me = _mae_model(False, cuda_device)
    og, mgm = _steps(mg, cfg, cuda_device, steps)
    oe, mem = _steps(me, cfg, cuda_device, steps)
    key = list(mg._graphs)
    assert len(key) == 1 and mg._graphs[key[0]].bwd_graph is not None, "the graphed model never switched to replay"
    keep = mg.len_keep
    for s in range(steps):
        torch.manual_seed(300 + s)
        want = _restate_masking(torch.rand(batch, mg.n_tokens, device=cuda_device), keep)[2].cpu()
        assert torch.equal(mgm[s], want) and torch.equal(mem[s], want), s
        if s:
            assert not torch.equal(mgm[s], mgm[s - 1]), s
        assert torch.equal(og[s], oe[s]), s


# ============================================================================================ unmodified drivers
@pytest.fixture
def _stock_registry_back():
    yield
    import driver_harness as H
    if H.setup_reference() is not None:
        H.use_engine(False)


MAE_OVER = ["DATA.TRAIN_CROP_NUM_TEMPORAL", 1, "MVIT.DEPTH", 2, "MASK.PRETRAIN_DEPTH", [1], "SOLVER.BASE_LR", 1e-4,
            "TRAIN.EVAL_PERIOD", 100]


def _compare_train(tag, en, st):
    assert len(en["train"]) == len(st["train"]) == 3
    for i, (a, b) in enumerate(zip(en["train"], st["train"])):
        rel = abs(a["loss"] - b["loss"]) / abs(b["loss"])
        gn = abs(a["grad_norm"] - b["grad_norm"]) / abs(b["grad_norm"])
        print(f"{tag}: iter {i} loss engine {a['loss']:.6f} stock {b['loss']:.6f} (rel {rel:.1e}); grad-norm rel {gn:.1e}")
        assert rel < (1e-3 if i == 0 else 1e-2), (i, a, b)
        assert gn < 0.1, (i, a["grad_norm"], b["grad_norm"])
        assert a["lr"] == b["lr"] and a["mb"] == b["mb"]


def test_mae_pretrain_then_fine_tune_through_the_unmodified_driver(cuda_device, _stock_registry_back):
    """TASK ssl on a shrunk k400_VIT_B_16x4_MAE_PT.yaml writes ssl_checkpoint_*; TASK ssl_eval in the same OUTPUT_DIR loads
    it into ViT-B and fine-tunes.  Engine and stock run the whole chain; the MAE losses and the fine-tuning losses agree
    within the driver bounds."""
    import os
    import tempfile
    import driver_harness as H
    if H.setup_reference() is None:
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    ft_over = ["MODEL.DROPOUT_RATE", 0.0, "MVIT.DROPPATH_RATE", 0.0, "MIXUP.ENABLE", False, "AUG.ENABLE", False,
               "AUG.NUM_SAMPLE", 1, "MODEL.LOSS_FUNC", "cross_entropy", "SOLVER.BASE_LR", 1e-4, "MVIT.DEPTH", 2,
               "TRAIN.AUTO_RESUME", True]
    runs = {}
    for engine in (False, True):
        H.use_engine(engine)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        out = tempfile.mkdtemp(prefix="sfb_mae_chain_")
        pt = H.driver_cfg("masked_ssl/k400_VIT_B_16x4_MAE_PT.yaml", 1, MAE_OVER, out_dir=out, frames=4, batch=4)
        rec_pt, _ = H.run_train(pt)
        assert any(f.startswith("ssl_checkpoint") for f in os.listdir(os.path.join(out, "checkpoints")))
        ft = H.driver_cfg("masked_ssl/k400_VIT_B_16x4_FT.yaml", 1, ft_over, out_dir=out, frames=4, batch=4)
        assert ft.TASK == "ssl_eval"
        rec_ft, _ = H.run_train(ft)
        runs[engine] = (rec_pt, rec_ft)
    from slowfast.models import build_model
    assert type(build_model(pt)).__name__ == "B200MAE"
    _compare_train("mae pre-train", runs[True][0], runs[False][0])
    _compare_train("mae -> vit-b fine-tune", runs[True][1], runs[False][1])
