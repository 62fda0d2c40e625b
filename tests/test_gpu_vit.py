"""GPU: separable absolute positions, the mean-token readout, the non-overlapping patch embedding and LayerNorm rows
wider than 768 on the engine (MViTv1-B, ViT-B / L / H and the MaskFeat fine-tuning recipes).

  * kernels: token assembly with positions, the position-gradient reduction, the mean readout and patchify + GEMM
    against fp64 (or bitwise against the same fp32 arithmetic where the kernel does exactly that arithmetic);
  * one ViT-B block at the recipe's 1569 tokens / head_dim 64 against the reference evaluated in fp64;
  * whole models against the unmodified reference (fp32, same GPU, same fixture weights and clips);
  * CUDA-graph replay against eager, and the unmodified train / test drivers, including MaskFeat pre-training followed
    by fine-tuning from the checkpoint it wrote.
"""
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


# ============================================================================================ kernels
POS_SHAPES = [  # (B, T, HW, E): ViT-B 16x224, MViTv1-B 16x224, odd extents
    (2, 8, 196, 768), (2, 8, 3136, 96), (3, 3, 35, 40), (1, 1, 1, 8)]


@pytest.mark.parametrize("b,t,hw,e", POS_SHAPES)
def test_tokens_assemble_with_positions(b, t, hw, e, cuda_device):
    from slowfast_b200 import ops
    g = torch.Generator().manual_seed(b * 1000 + hw)
    Lt = t * hw
    y, bias, cls = torch.randn(b, Lt, e, generator=g), torch.randn(e, generator=g), torch.randn(e, generator=g)
    ps, pt, pc = torch.randn(hw, e, generator=g), torch.randn(t, e, generator=g), torch.randn(e, generator=g)
    d = [v.to(cuda_device) for v in (y, bias, cls, ps, pt, pc)]
    out = torch.empty(b, Lt + 1, e, device=cuda_device)
    ops.tokens_assemble(*d, b, Lt, hw, e, out)
    # the reference's arithmetic in fp32: x = cat(cls, y + bias) + cat(pc, ps.repeat(t) + pt.repeat_interleave(hw))
    pos = torch.cat([pc.view(1, e), ps.repeat(t, 1) + pt.repeat_interleave(hw, dim=0)])
    want = torch.cat([cls.view(1, 1, e).expand(b, 1, e), y + bias], 1) + pos
    assert torch.equal(out.cpu(), want)
    # null tables: the plain assembly, bitwise
    ops.tokens_assemble(d[0], d[1], d[2], None, None, None, b, Lt, hw, e, out)
    assert torch.equal(out.cpu(), torch.cat([cls.view(1, 1, e).expand(b, 1, e), y + bias], 1))


def test_tokens_assemble_rejects_partial_tables(cuda_device):
    L, lib = _lib()
    t = torch.zeros(64, device=cuda_device)
    rc = lib.sfb_tokens_assemble(t.data_ptr(), t.data_ptr(), t.data_ptr(), t.data_ptr(), None, t.data_ptr(), 1, 4, 2, 8,
                                 t.data_ptr(), _st())
    assert rc != 0 and b"positions need all three tables" in lib.sfb_last_error()


@pytest.mark.parametrize("b,t,hw,e", POS_SHAPES)
def test_pos_embed_sep_bwd_matches_fp64_and_is_deterministic(b, t, hw, e, cuda_device):
    from slowfast_b200 import ops
    dx = torch.randn(b, 1 + t * hw, e, generator=torch.Generator().manual_seed(7))
    d = dx.to(cuda_device)
    part = torch.empty(t * ops.segment_slabs(t, hw) * e, device=cuda_device)
    outs = []
    for _ in range(2):
        dps, dpt, dpc = (torch.full(s, float("nan"), device=cuda_device) for s in ((hw, e), (t, e), (e,)))
        ops.pos_embed_sep_bwd(d, b, t, hw, e, dps, dpt, dpc, part)
        outs.append((dps.cpu(), dpt.cpu(), dpc.cpu()))
    x = dx.double()[:, 1:].view(b, t, hw, e)
    want = (x.sum((0, 1)), x.sum((0, 2)), dx.double()[:, 0].sum(0))
    for got, w in zip(outs[0], want):
        assert _rel(got.double(), w) < 1e-6
    assert all(torch.equal(a, c) for a, c in zip(outs[0], outs[1]))


@pytest.mark.parametrize("b,n,c", [(8, 1569, 768), (2, 393, 768), (3, 50, 40), (1, 2, 8)])
def test_token_mean_fwd_bwd(b, n, c, cuda_device):
    from slowfast_b200 import ops
    g = torch.Generator().manual_seed(n)
    x, dm = torch.randn(b, n, c, generator=g), torch.randn(b, c, generator=g)
    xd, dmd = x.to(cuda_device), dm.to(cuda_device)
    out = torch.empty(b, c, device=cuda_device)
    part = torch.empty(b * ops.segment_slabs(b, n - 1) * c, device=cuda_device)
    ops.token_mean_fwd(xd, b, n, c, out, part)
    assert _rel(out.cpu().double(), x.double()[:, 1:].mean(1)) < 1e-6
    out2 = torch.empty_like(out)
    ops.token_mean_fwd(xd, b, n, c, out2, part)
    assert torch.equal(out, out2)
    dx = torch.full((b, n, c), float("nan"), device=cuda_device)
    ops.token_mean_bwd(dmd, b, n, c, dx)
    want = torch.cat([torch.zeros(b, 1, c), (dm / (n - 1)).view(b, 1, c).expand(b, n - 1, c)], 1)
    torch.testing.assert_close(dx.cpu(), want, rtol=1e-6, atol=0)


@pytest.mark.parametrize("nsplit", [3, 1])
@pytest.mark.parametrize("shape,k", [((2, 3, 4, 32, 32), (2, 16, 16)),      # ViT's 2x16x16 patches
                                     ((2, 3, 6, 24, 40), (3, 8, 4))])      # non-square, odd patch grid (2 x 3 x 10)
def test_patchify_gemm_and_wgrad_match_conv3d(shape, k, nsplit, cuda_device):
    from slowfast_b200 import ops
    from slowfast_b200.engine import Ctx
    from slowfast_b200.ops import Planes
    g = torch.Generator().manual_seed(3)
    x = torch.randn(*shape, generator=g)
    B, cin = shape[:2]
    E, K = 64, cin * k[0] * k[1] * k[2]
    w = torch.randn(E, cin, *k, generator=g) * K ** -0.5
    ctx = Ctx(nsplit)
    ctx.device = cuda_device
    ot, oh, ow = shape[2] // k[0], shape[3] // k[1], shape[4] // k[2]
    rows = B * ot * oh * ow
    s = ctx.storage(("rows",), 1, 1, 1, rows, K)
    xr = Planes(s.hi, s.lo, 1, 1, 1, rows, K, 0)
    ops.patchify(x.to(cuda_device), k, xr)
    wd = w.to(cuda_device).view(E, K)
    fm = ops.alloc_filter(E, 1, K, nsplit, cuda_device)
    ops.filter_pack(wd, fm)
    y = torch.empty(rows, E, device=cuda_device)
    geom = ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, rows))
    ops.conv_igemm(xr, fm, geom, y, (rows * E, rows * E, rows * E, E), nsplit=nsplit)
    want = F.conv3d(x.double(), w.double(), stride=k).permute(0, 2, 3, 4, 1).reshape(rows, E)
    tol = 1e-5 if nsplit == 3 else 1e-2
    assert _rel(y.cpu().double(), want) < tol
    # weight gradient through the same rows: dW = dY^T . X  (Conv3d's weight layout after the view)
    dy = torch.randn(rows, E, generator=g)
    ds = ctx.storage(("dy",), 1, 1, 1, rows, E)
    dyp = Planes(ds.hi, ds.lo, 1, 1, 1, rows, E, 0)
    ops.split_planes(dy.to(cuda_device).contiguous(), dyp)
    gw = torch.zeros(E, K, device=cuda_device)
    ops.conv_wgrad(xr, dyp, geom, gw, nsplit=nsplit)
    xv = x.double().unfold(2, k[0], k[0]).unfold(3, k[1], k[1]).unfold(4, k[2], k[2])   # [B, cin, ot, oh, ow, kt, kh, kw]
    xm = xv.permute(0, 2, 3, 4, 1, 5, 6, 7).reshape(rows, K)
    assert _rel(gw.cpu().double(), dy.double().t() @ xm) < tol


@pytest.mark.parametrize("c", [1024, 1152, 1280, 1000, 768])
def test_layernorm_wide_rows_match_fp64(c, cuda_device):
    """LayerNorm at ViT-L (1024), MViTv2-L's last stage (1152) and ViT-H (1280) widths, an odd width, and 768 (the widest
    row of the register-resident kernel), forward and backward (dx accumulated, dgamma / dbeta) against fp64."""
    from slowfast_b200 import ops
    rows = 3 * 1569
    g = torch.Generator().manual_seed(c)
    x, dy = torch.randn(rows, c, generator=g) * 2 + 0.5, torch.randn(rows, c, generator=g)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    dx0 = torch.randn(rows, c, generator=g)
    xd, dyd, gd, bd = (v.to(cuda_device) for v in (x, dy, gamma, beta))
    y = torch.empty(rows, c, device=cuda_device)
    mean, rstd = torch.empty(rows, device=cuda_device), torch.empty(rows, device=cuda_device)
    ops.layernorm_fwd(xd, c, rows, c, gd, bd, 1e-6, mean, rstd, out_f32=y)
    dx, dg, db = dx0.to(cuda_device), torch.empty(c, device=cuda_device), torch.empty(c, device=cuda_device)
    part = torch.empty(ops.colsum_blocks(rows) * 2 * c, device=cuda_device)
    ops.layernorm_bwd(dyd, c, xd, c, rows, c, gd, mean, rstd, dx, c, dg, db, part, dx_accumulate=True)
    xr = x.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    yr = F.layer_norm(xr, (c,), gr, br, 1e-6)
    yr.backward(dy.double())
    assert _rel(y.cpu().double(), yr.detach()) < 1e-6
    assert _rel(dx.cpu().double() - dx0.double(), xr.grad) < 1e-5
    assert _rel(dg.cpu().double(), gr.grad) < 1e-5 and _rel(db.cpu().double(), br.grad) < 1e-5


# ============================================================================================ one ViT block, 1569 tokens
def test_vit_b_block_at_1569_tokens_matches_reference_fp64(cuda_device):
    """ViT-B with one block at the recipe's clip (16 x 224^2 -> 8 x 14 x 14 + cls = 1569 tokens, 12 heads of 64,
    unpooled attention with Nkp = 1576) through the engine in parity mode, against the unmodified reference run in fp64
    on the same fixture: logits, and every parameter gradient."""
    from oracle import refshim
    from oracle import torch_oracle as TO
    from slowfast_b200.nets.mvit import B200MViT
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    cfg = refshim.load_cfg("masked_ssl/k400_VIT_B_16x4_FT.yaml", ["MVIT.DEPTH", 1, "MODEL.DROPOUT_RATE", 0.0,
                                                                  "MVIT.DROPPATH_RATE", 0.0])
    ref = refshim.build_reference_model(cfg)
    state = _fixture(ref.state_dict())
    ref.load_state_dict(state)
    ref = ref.to(cuda_device).double().train()
    mine = B200MViT(cfg)
    mine.load_state_dict(state)
    mine = mine.to(cuda_device).train()
    x = TO.synthetic_inputs(cfg, 1, 4)[0].to(cuda_device)
    dl = torch.randn(1, cfg.MODEL.NUM_CLASSES, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    lr = ref([x.double()])
    lr.backward(dl.double())
    lm = mine([x])
    lm.backward(dl)
    torch.cuda.synchronize()
    rel = _rel(lm.double(), lr)
    rm = dict(ref.named_parameters())
    per = {k: _rel(p.grad.double(), rm[k].grad) for k, p in mine.named_parameters()}
    worst = max(per, key=per.get)
    print(f"vit-b block @1569: logits rel-L2 {rel:.2e}; grad rel-L2 median {sorted(per.values())[len(per) // 2]:.2e} "
          f"max {per[worst]:.2e} ({worst})")
    assert rel < 1e-4
    assert per[worst] < 1e-3, (worst, per[worst])


# ============================================================================================ whole models vs reference
def _fixture(template, seed=3):
    from oracle import torch_oracle as TO
    state = TO.fixture_state(template, seed)
    for i, k in enumerate(template):   # position tables at the scale of the cls token, so they matter to the output
        if k.startswith("pos_embed"):
            state[k] = torch.randn(template[k].shape, generator=torch.Generator().manual_seed(seed * 7919 + i)) * 0.2
    return state


MODEL_CASES = [  # (yaml, frames, crop, extra overrides)
    ("Kinetics/MVIT_B_16x4_CONV.yaml", 8, 64, []),
    ("Kinetics/MVIT_B_16x4_CONV.yaml", 16, 224, []),     # 3137 tokens in stage 1, adaptive 1x8x8 K/V pools
    ("masked_ssl/k400_VIT_B_16x4_FT.yaml", 4, 64, []),
    ("masked_ssl/k400_VIT_B_16x4_FT.yaml", 16, 224, []),
    ("masked_ssl/k400_MVITv2_S_16x4_FT.yaml", 8, 64, []),
    ("masked_ssl/k400_MVITv2_L_16x4_FT.yaml", 8, 64, []),  # widths 144 .. 1152
    # ViT-L (1024 wide, 16 heads of 64) and ViT-H (1280 wide, 16 heads of 80) at the recipe's 1569 tokens, two blocks
    ("masked_ssl/k400_VIT_L_16x4_FT.yaml", 16, 224, ["MVIT.DEPTH", 2]),
    ("masked_ssl/k400_VIT_H_16x4_FT.yaml", 16, 224, ["MVIT.DEPTH", 2]),
]


@pytest.mark.parametrize("fast", [False, True], ids=["parity", "fast"])
@pytest.mark.parametrize("yaml,frames,crop,extra", MODEL_CASES)
def test_model_step_and_eval_match_reference(yaml, frames, crop, extra, fast, cuda_device):
    """One training step of the engine and of the unmodified reference (fp32 on the same GPU) from the same fixture
    weights and clip; then an eval forward.  Parity mode: logits 1e-3 max-abs relative with argmax exact; gradients
    against the reference evaluated in fp64, per parameter within max(8x the reference's own fp32-vs-fp64 error, 0.15)
    and with the median error within max(8x the median envelope, 1e-3) (the position, cls and patch-embedding gradients
    included).  Gradients that are zero in exact arithmetic - the key LayerNorm bias under pooling and the key third of
    the qkv bias (softmax is invariant to a per-query constant) - are rounding noise in every implementation: there the
    engine's gradient norm is held below 1e-3 of the median gradient norm.  Fast mode (bf16 operands): logits and eval
    output within 2x the reference's own bf16-autocast error on the same step (floor 1e-2)."""
    import copy
    from oracle import refshim
    from oracle import torch_oracle as TO
    from slowfast_b200.nets.mvit import B200MViT
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    cfg = refshim.load_cfg(yaml, ["DATA.NUM_FRAMES", frames, "DATA.TRAIN_CROP_SIZE", crop, "DATA.TEST_CROP_SIZE", crop,
                                  "MODEL.DROPOUT_RATE", 0.0, "MVIT.DROPPATH_RATE", 0.0] + list(extra))
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
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, batch, 4)]
    dl = torch.randn(batch, cfg.MODEL.NUM_CLASSES, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    lr = ref([t.clone() for t in x])
    lr.backward(dl)
    lm = mine(x)
    lm.backward(dl)
    torch.cuda.synchronize()
    rel_max = ((lm - lr).abs().max() / lr.abs().max()).item()
    rm = dict(ref.named_parameters())
    per = {k: _rel(p.grad.double(), rm[k].grad.double()) for k, p in mine.named_parameters()}
    rels = sorted(per.values())
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
    tag = f"{yaml.split('/')[-1]} {frames}x{crop}^2 {extra} {'fast' if fast else 'parity'}"
    print(f"{tag}: logits max-rel {rel_max:.2e} rel-L2 {_rel(lm, lr):.2e}; grad rel-L2 median {rels[len(rels) // 2]:.2e} "
          f"max {per[worst]:.2e} ({worst}); eval rel-L2 {_rel(em, er):.2e}")
    if fast:
        env, env_eval = _rel(lr_bf, lr.detach()), _rel(er_bf, er)
        print(f"  reference bf16-autocast error: train {env:.2e}, eval {env_eval:.2e}")
        assert _rel(lm, lr) < max(2 * env, 1e-2)
        assert _rel(em, er) < max(2 * env_eval, 1e-2)
        return
    assert rel_max < 1e-3 and torch.equal(lm.argmax(1), lr.argmax(1))
    # test_gpu_models.py's sampled-gradient bounds.  Measured on an H100: median 2.0e-5 (ViT-B 64^2), 1.2e-5 (ViT-B 224^2),
    # 1.2e-5 / 1.4e-5 (ViT-L / ViT-H, two blocks at 224^2), 5.7e-4 / 5.2e-5 (MViTv1-B 64^2 / 224^2), 4.0e-3 (MViTv2-S FT;
    # worst rel_pos_w 1.3e-2), 2.5e-3 (MViTv2-L FT).  The MViT excess comes from the skip max-pool, not the block math: where
    # a window's top two values are closer than the forward error, the engine and fp64 pick different inputs, and the
    # gradient upstream of that block moves by far more than rounding.  One such window in 98 304 takes a 3-block
    # MViTv2-S FT stack from 4.6e-5 to 6.9e-4 worst; with the routing pinned, every MViT block kind is within 5e-5 of fp64
    # (test_gpu_mvit_blocks.py holds them to 1e-3).  Hence the wide per-parameter bound here
    assert ratio[wk] < 1.0, (wk, err[wk], env[wk])
    assert em_ < max(8 * en_, 0.15), (em_, en_)
    for k in zero:
        assert mine.get_parameter(k).grad.norm().item() < 1e-3 * med, k
    assert ((em - er).abs().max() / er.abs().max()).item() < 1e-3 and torch.equal(em.argmax(1), er.argmax(1))


# ============================================================================================ replay
def _vit_model(graphs, dev):
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.mvit import B200MViT
    cfg = get_cfg("VIT_B_16x4_FT", DATA={"NUM_FRAMES": 4, "TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64},
                  MVIT={"DEPTH": 3, "DROPPATH_RATE": 0.0}, MODEL={"DROPOUT_RATE": 0.0},
                  B200={"NSPLIT": 3, "CUDA_GRAPH": graphs})
    torch.manual_seed(0)
    model = B200MViT(cfg)
    model.load_state_dict(_fixture(model.state_dict(), 7))
    return cfg, model.to(dev).train()


def _steps(model, cfg, dev, n_steps, batch=2):
    from oracle import torch_oracle as TO
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    outs = []
    for s in range(n_steps):
        x = TO.synthetic_inputs(cfg, batch, 100 + s)
        y = torch.randint(0, cfg.MODEL.NUM_CLASSES, (batch,), generator=torch.Generator().manual_seed(105 + s))
        opt.zero_grad(set_to_none=True)
        logits = model([t.to(dev) for t in x])
        F.cross_entropy(logits, y.to(dev)).backward()
        opt.step()
        outs.append(logits.detach().cpu())
    torch.cuda.synchronize()
    return outs


def test_vit_replay_matches_eager_over_steps(cuda_device):
    """The ViT step is deterministic: two eager runs and the CUDA-graph replay give bitwise identical logits at every one
    of five SGD steps (the position-gradient and mean-readout reductions are atomic-free, and at this shape no other
    reduction of the step depends on scheduling order)."""
    steps = 5
    cfg, mg = _vit_model(True, cuda_device)
    _, me = _vit_model(False, cuda_device)
    _, me2 = _vit_model(False, cuda_device)
    og, oe, oe2 = _steps(mg, cfg, cuda_device, steps), _steps(me, cfg, cuda_device, steps), \
        _steps(me2, cfg, cuda_device, steps)
    key = list(mg._graphs)
    assert len(key) == 1 and mg._graphs[key[0]].bwd_graph is not None, "the graphed model never switched to replay"
    for s in range(steps):
        rel = ((og[s] - oe[s]).abs().max() / oe[s].abs().max()).item()
        noise = ((oe2[s] - oe[s]).abs().max() / oe[s].abs().max()).item()
        print(f"step {s}: logits replay vs eager {rel:.2e} (eager vs eager {noise:.2e})")
        assert torch.equal(oe2[s], oe[s]), s
        assert torch.equal(og[s], oe[s]), s


# ============================================================================================ unmodified drivers
@pytest.fixture
def _stock_registry_back():
    yield
    import driver_harness as H
    if H.setup_reference() is not None:
        H.use_engine(False)


FT_OVER = ["MODEL.DROPOUT_RATE", 0.0, "MVIT.DROPPATH_RATE", 0.0, "MIXUP.ENABLE", False, "AUG.ENABLE", False,
           "AUG.NUM_SAMPLE", 1, "MODEL.LOSS_FUNC", "cross_entropy", "SOLVER.BASE_LR", 1e-4]


def _compare_train(tag, en, st):
    assert len(en["train"]) == len(st["train"]) == 3
    for i, (a, b) in enumerate(zip(en["train"], st["train"])):
        rel = abs(a["loss"] - b["loss"]) / abs(b["loss"])
        gn = abs(a["grad_norm"] - b["grad_norm"]) / abs(b["grad_norm"])
        print(f"{tag}: iter {i} loss engine {a['loss']:.6f} stock {b['loss']:.6f} (rel {rel:.1e}); grad-norm rel {gn:.1e}")
        assert rel < (1e-3 if i == 0 else 1e-2), (i, a, b)
        assert gn < 0.1, (i, a["grad_norm"], b["grad_norm"])
        assert a["lr"] == b["lr"] and a["mb"] == b["mb"]


@pytest.mark.parametrize("yaml,frames", [("masked_ssl/k400_VIT_B_16x4_FT.yaml", 4), ("Kinetics/MVIT_B_16x4_CONV.yaml", 8)])
def test_unmodified_train_and_test_drivers_match_stock_model(yaml, frames, cuda_device, _stock_registry_back):
    import driver_harness as H
    if H.setup_reference() is None:
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    runs = {}
    for engine in (False, True):
        H.use_engine(engine)
        cfg = H.driver_cfg(yaml, 1, FT_OVER, frames=frames, batch=4)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        rec_train, _ = H.run_train(cfg)
        rec_test, result = H.run_test(cfg)
        runs[engine] = (rec_train, rec_test, result)
    from slowfast.models import build_model
    assert type(build_model(cfg)).__name__ == "B200MViT"
    (st_train, st_test, _), (en_train, en_test, result) = runs[False], runs[True]
    _compare_train(yaml, en_train, st_train)
    assert len(en_train["val"]) == len(st_train["val"]) > 0
    assert len(en_test["test"]) == len(st_test["test"]) > 0
    for a, b in zip(en_test["test"], st_test["test"]):
        assert torch.equal(a["ids"], b["ids"])
        assert ((a["preds"] - b["preds"]).abs().max() / b["preds"].abs().max()).item() < 5e-2
    assert "Top5 Acc" in result


def test_maskfeat_pretrain_then_fine_tune_through_the_unmodified_driver(cuda_device, _stock_registry_back):
    """TASK ssl (MaskMViT pre-training) writes ssl_checkpoint_epoch_00001.pyth; TASK ssl_eval in the same OUTPUT_DIR loads
    it into the mean-readout MViT (train_net.py: the ssl_eval branch of the resume logic) and fine-tunes.  Engine and
    stock run the whole chain each; the fine-tuning losses agree within the driver bounds."""
    import os
    import tempfile
    import driver_harness as H
    if H.setup_reference() is None:
        pytest.skip("no reference tree: build() copies it into oracle/_ref from a reference checkout")
    runs = {}
    for engine in (False, True):
        H.use_engine(engine)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        out = tempfile.mkdtemp(prefix="sfb_maskfeat_chain_")
        pt = H.driver_cfg("masked_ssl/k400_MVITv2_S_16x4_MaskFeat_PT.yaml", 1, ["SOLVER.BASE_LR", 1e-4, "TASK", "ssl"],
                          out_dir=out, frames=8, batch=4)
        H.run_train(pt)
        assert any(f.startswith("ssl_checkpoint") for f in os.listdir(os.path.join(out, "checkpoints")))
        ft = H.driver_cfg("masked_ssl/k400_MVITv2_S_16x4_FT.yaml", 1, FT_OVER + ["TRAIN.AUTO_RESUME", True],
                          out_dir=out, frames=8, batch=4)
        assert ft.TASK == "ssl_eval"
        rec, _ = H.run_train(ft)
        runs[engine] = rec
    _compare_train("maskfeat fine-tune", runs[True], runs[False])
