"""GPU: the MViT token-path kernels (csrc/mvit_ops.cu) and the MaskFeat HOG kernel (csrc/maskfeat.cu), each on its own
through the C ABI against a PyTorch fp64 restatement of the reference operator it replaces:

  sfb_layernorm_fwd/bwd        nn.LayerNorm(eps=1e-6)                        attention.py:40-44, :500, :509
  sfb_dwpool_fwd/bwd           attention_pool's depthwise Conv3d on tokens   attention.py:13-45 (all four MViTv2-S
                               (kernel 3x3x3, stride, cls passes through)     stride / size pairs)
  sfb_softmax_relpos_fwd/bwd   rel-pos bias + softmax                        attention.py:64-147, :355-379
  sfb_bias_gelu / _bwd         fc1 bias + GELU(erf)                          common.py:26-44
  sfb_token_maxpool_fwd/bwd    MaxPool3d skip path on tokens                 attention.py:485-489
  sfb_hog_targets              HOGLayerC + per-token regrouping              operators.py:79-122, masked.py:254-281
Whole-model tests only run these at B <= 3 with one geometry each; here shapes are ragged on purpose.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def planes_to_float(hi, lo):
    return hi.float() + (lo.float() if lo is not None else 0)


@pytest.mark.parametrize("rows,c", [(1000, 96), (777, 192), (130, 768), (515, 384)])
def test_layernorm_forward_backward(rows, c, cuda_device):
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    g = torch.Generator().manual_seed(rows + c)
    x = torch.randn(rows, c, generator=g).to(dev) * 2 + 0.5
    gamma = (torch.rand(c, generator=g) + 0.5).to(dev)
    beta = torch.randn(c, generator=g).to(dev)
    hi = torch.empty(rows, c, dtype=torch.bfloat16, device=dev)
    lo = torch.empty_like(hi)
    of = torch.empty(rows, c, device=dev)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    L.check(lib.sfb_layernorm_fwd(x.data_ptr(), c, rows, c, gamma.data_ptr(), beta.data_ptr(), 1e-6, hi.data_ptr(),
                                  lo.data_ptr(), of.data_ptr(), c, mean.data_ptr(), rstd.data_ptr(), _st()))
    xd = x.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    ref = F.layer_norm(xd, (c,), gd, bd, 1e-6)
    assert relerr(of, ref) < 2e-6
    assert relerr(planes_to_float(hi, lo), ref) < 2e-5          # split planes carry ~16 mantissa bits
    dy = torch.randn(rows, c, generator=g).to(dev)
    ref.backward(dy.double())
    nb = lib.sfb_rowslab_blocks(rows)
    part = torch.empty(nb * 2 * c, device=dev)
    dx = torch.full((rows, c), float("nan"), device=dev)
    dg, db = torch.empty(c, device=dev), torch.empty(c, device=dev)
    L.check(lib.sfb_layernorm_bwd(dy.data_ptr(), c, x.data_ptr(), c, rows, c, gamma.data_ptr(), mean.data_ptr(),
                                  rstd.data_ptr(), dx.data_ptr(), c, 0, dg.data_ptr(), db.data_ptr(), 0, part.data_ptr(),
                                  _st()))
    assert relerr(dx, xd.grad) < 1e-5 and relerr(dg, gd.grad) < 1e-5 and relerr(db, bd.grad) < 1e-5
    base = torch.randn(rows, c, generator=g).to(dev)   # accumulate forms (dx +=, parameter gradients +=)
    acc = base.clone()
    L.check(lib.sfb_layernorm_bwd(dy.data_ptr(), c, x.data_ptr(), c, rows, c, gamma.data_ptr(), mean.data_ptr(),
                                  rstd.data_ptr(), acc.data_ptr(), c, 1, dg.data_ptr(), db.data_ptr(), 1, part.data_ptr(),
                                  _st()))
    assert relerr(acc - base, xd.grad) < 1e-4 and relerr(dg, 2 * gd.grad) < 1e-5


# (B, heads, hd, T, H, W, kernel, stride): the four (size, stride) pairs of MViTv2-S at reduced extents + a no-pool copy
DWPOOL_CASES = [
    (2, 1, 96, 4, 16, 16, (3, 3, 3), (1, 8, 8)),     # block 0 K/V pool
    (2, 2, 96, 4, 12, 12, (3, 3, 3), (1, 4, 4)),     # blocks 1-2 K/V
    (3, 4, 96, 2, 14, 14, (3, 3, 3), (1, 2, 2)),     # blocks 3-13 K/V, and the strided Q pools
    (2, 4, 96, 3, 7, 9, (3, 3, 3), (1, 1, 1)),       # stride-1 Q pool, ragged grid (gather kernels)
    (2, 2, 96, 3, 14, 14, (3, 3, 3), (1, 1, 1)),     # stride-1 Q pool on the shared-memory ring kernels (14x14 tiles)
    (1, 4, 96, 2, 7, 21, (3, 3, 3), (1, 1, 1)),      # ring kernels, 7x7 tiles, 3 tiles per frame
    (2, 1, 96, 4, 28, 14, (3, 3, 3), (1, 1, 1)),     # ring kernels, one head
    (2, 8, 96, 2, 7, 7, None, None),                 # has_pool = 0 (POOL_KVQ_KERNEL absent): copy + bias
]


@pytest.mark.parametrize("case", DWPOOL_CASES)
def test_dwpool_forward_backward(case, cuda_device):
    """attention_pool (attention.py:13-45): tokens [B, 1+THW, 3A] (fused qkv output, + qkv bias) -> per head NCTHW ->
    depthwise Conv3d(kernel, stride, pad k//2, weight shared by the heads) -> tokens, cls passes through."""
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    B, Hn, hd, T, Hh, W, kern, strd = case
    A = Hn * hd
    Lin = T * Hh * W
    g = torch.Generator().manual_seed(B * 100 + Hn)
    src = torch.randn(B, Lin + 1, 3 * A, generator=g).to(dev)
    bias = torch.randn(3 * A, generator=g).to(dev) * 0.3
    j = 1  # the k third of the fused projection
    has = kern is not None
    if has:
        w = (torch.randn(hd, 1, *kern, generator=g) / 3).to(dev)
        othw = [(i + 2 * (k // 2) - k) // s + 1 for i, k, s in zip((T, Hh, W), kern, strd)]
    else:
        w, othw = None, [T, Hh, W]
    Lo = math.prod(othw)
    out = torch.full((B, Hn, Lo + 1, hd), float("nan"), device=dev)
    d = L.DwPoolDesc()
    d.src, d.src_pitch, d.src_c0, d.bias = src.data_ptr(), 3 * A, j * A, bias.data_ptr()
    d.out = out.data_ptr()
    d.b, d.heads, d.hd, d.t, d.h, d.w_ = B, Hn, hd, T, Hh, W
    d.ot, d.oh, d.ow = othw
    d.has_pool = 1 if has else 0
    if has:
        d.w = w.data_ptr()
        d.kt, d.kh, d.kw = kern
        d.st, d.sh, d.sw = strd
    else:
        d.kt = d.kh = d.kw = d.st = d.sh = d.sw = 1
    L.check(lib.sfb_dwpool_fwd(C.byref(d), _st()))
    # reference in fp64
    sd = src.double().requires_grad_(True)
    wd = w.double().requires_grad_(True) if has else None
    t = (sd[:, :, j * A:(j + 1) * A] + bias.double()[j * A:(j + 1) * A]).view(B, Lin + 1, Hn, hd).permute(0, 2, 1, 3)
    cls, tok = t[:, :, :1], t[:, :, 1:]
    if has:
        x5 = tok.reshape(B * Hn, T, Hh, W, hd).permute(0, 4, 1, 2, 3)
        y5 = F.conv3d(x5, wd, None, strd, [k // 2 for k in kern], 1, hd)
        tok = y5.reshape(B, Hn, hd, Lo).transpose(2, 3)
    ref = torch.cat([cls, tok], 2)
    assert relerr(out, ref) < 1e-5
    dout = torch.randn(B, Hn, Lo + 1, hd, generator=g).to(dev)
    ref.backward(dout.double())
    dsrc = torch.zeros(B, Lin + 1, 3 * A, device=dev)
    d.dout, d.dsrc = dout.data_ptr(), dsrc.data_ptr()
    dw = None
    if has:
        nb = lib.sfb_dwpool_wgrad_blocks(C.byref(d))
        wp = torch.empty(max(nb, 1) * hd * math.prod(kern), device=dev)
        d.wpartials = wp.data_ptr()
        dw = torch.full_like(w, float("nan"))
    L.check(lib.sfb_dwpool_bwd(C.byref(d), dw.data_ptr() if has else None, 0, _st()))
    assert relerr(dsrc, sd.grad) < 1e-5
    assert (dsrc[:, :, :j * A] == 0).all() and (dsrc[:, :, (j + 1) * A:] == 0).all()   # only this third is touched
    if has:
        assert relerr(dw, wd.grad) < 2e-5


def _rel_index(nq, nk):
    """get_rel_pos distances (attention.py:75-92 / :118-127): q_idx*max(nk/nq,1) - k_idx*max(nq/nk,1) + (nk-1)*max(nq/nk,1)."""
    qr, kr = max(nk / nq, 1.0), max(nq / nk, 1.0)
    d = torch.arange(nq)[:, None] * qr - torch.arange(nk)[None, :] * kr + (nk - 1) * kr
    return d.long()


@pytest.mark.parametrize("q_thw,k_thw,bh", [((2, 8, 8), (2, 4, 4), 3), ((4, 14, 14), (4, 7, 7), 2), ((2, 7, 7), (2, 7, 7), 5),
                                            ((2, 7, 7), (2, 14, 14), 2), ((3, 6, 10), (3, 3, 5), 2)])
def test_softmax_relpos_forward_backward(q_thw, k_thw, bh, cuda_device):
    """P = softmax(S + bias), bias[q,k] = RQ[q, ih(q,k)] + RQ[q, Lh + iw] + RQ[q, Lh+Lw + it] for non-cls (q, k)
    (cal_rel_pos_spatial / cal_rel_pos_temporal, attention.py:64-147; the cls row and column get no bias); backward
    dS = P * (dP - sum(dP*P)) and dRQ = the scatter of dS onto the table columns."""
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    qt, qh, qw = q_thw
    kt, kh, kw = k_thw
    Lq, Lk = qt * qh * qw, kt * kh * kw
    Nq, Nk = Lq + 1, Lk + 1
    Nkp = (Nk + 7) // 8 * 8
    Lh, Lw, Lt = 2 * max(qh, kh) - 1, 2 * max(qw, kw) - 1, 2 * max(qt, kt) - 1
    Ltp = (Lh + Lw + Lt + 7) // 8 * 8
    g = torch.Generator().manual_seed(Lq + Lk)
    S = torch.zeros(bh, Nq, Nkp)
    S[..., :Nk] = torch.randn(bh, Nq, Nk, generator=g) * 2
    rq = torch.zeros(bh * Lq, Ltp)
    rq[:, :Lh + Lw + Lt] = torch.randn(bh * Lq, Lh + Lw + Lt, generator=g)
    S, rq = S.to(dev), rq.to(dev)
    p_hi = torch.full((bh, Nq, Nkp), float("nan"), dtype=torch.bfloat16, device=dev)
    p_lo = torch.full_like(p_hi, float("nan"))
    sd = L.SoftmaxDesc()
    sd.s, sd.s_pitch, sd.rq, sd.rq_pitch = S.data_ptr(), Nkp, rq.data_ptr(), Ltp
    sd.p_hi, sd.p_lo, sd.p_pitch = p_hi.data_ptr(), p_lo.data_ptr(), Nkp
    sd.bh, sd.nq, sd.nk = bh, Nq, Nk
    sd.qt, sd.qh, sd.qw = q_thw
    sd.kt, sd.kh, sd.kw = k_thw
    L.check(lib.sfb_softmax_relpos_fwd(C.byref(sd), _st()))
    # fp64 reference with explicit index tables
    Sd = S[..., :Nk].double().cpu().requires_grad_(True)
    rqd = rq.double().cpu().requires_grad_(True)
    ih, iw, it = _rel_index(qh, kh), _rel_index(qw, kw), _rel_index(qt, kt)
    r = rqd.view(bh, qt, qh, qw, Ltp)
    # gather per axis: bias[b,qt,qh,qw,kt,kh,kw]
    bh_idx = ih[None, None, :, None, :].expand(bh, qt, qh, qw, kh)
    bw_idx = iw[None, None, None, :, :].expand(bh, qt, qh, qw, kw) + Lh
    bt_idx = it[None, :, None, None, :].expand(bh, qt, qh, qw, kt) + Lh + Lw
    rel_h = torch.gather(r, 4, bh_idx)   # [bh,qt,qh,qw,kh]
    rel_w = torch.gather(r, 4, bw_idx)
    rel_t = torch.gather(r, 4, bt_idx)
    bias = (rel_t[..., :, None, None] + rel_h[..., None, :, None] + rel_w[..., None, None, :]).reshape(bh, Lq, Lk)
    full = Sd + F.pad(bias, (1, 0, 1, 0))
    P = torch.softmax(full, dim=-1)
    got = planes_to_float(p_hi, p_lo).cpu()
    assert relerr(got[..., :Nk], P) < 2e-5
    assert (got[..., Nk:] == 0).all()
    dP = torch.zeros(bh, Nq, Nkp)
    dP[..., :Nk] = torch.randn(bh, Nq, Nk, generator=g)
    P.backward(dP[..., :Nk].double())
    dPd = dP.to(dev)
    ds_hi = torch.full((bh, Nq, Nkp), float("nan"), dtype=torch.bfloat16, device=dev)
    ds_lo = torch.full_like(ds_hi, float("nan"))
    drq = torch.full((bh * Lq, Ltp), float("nan"), device=dev)
    sd.dp, sd.dp_pitch = dPd.data_ptr(), Nkp
    sd.ds_hi, sd.ds_lo, sd.ds_pitch = ds_hi.data_ptr(), ds_lo.data_ptr(), Nkp
    sd.drq = drq.data_ptr()
    L.check(lib.sfb_softmax_relpos_bwd(C.byref(sd), _st()))
    dS = planes_to_float(ds_hi, ds_lo).cpu()
    assert relerr(dS[..., :Nk], Sd.grad) < 5e-5
    assert relerr(drq.cpu()[:, :Lh + Lw + Lt], rqd.grad[:, :Lh + Lw + Lt]) < 1e-4


@pytest.mark.parametrize("rows,c", [(1000, 384), (333, 1536), (64, 3072)])
def test_bias_gelu_forward_backward(rows, c, cuda_device):
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    g = torch.Generator().manual_seed(c)
    y = (torch.randn(rows, c, generator=g) * 2).to(dev)
    b = torch.randn(c, generator=g).to(dev)
    hi = torch.empty(rows, c, dtype=torch.bfloat16, device=dev)
    lo = torch.empty_like(hi)
    L.check(lib.sfb_bias_gelu(y.data_ptr(), b.data_ptr(), rows, c, hi.data_ptr(), lo.data_ptr(), _st()))
    pre = (y.double() + b.double()).requires_grad_(True)
    ref = F.gelu(pre)  # exact erf form (nn.GELU default, common.py:33)
    assert relerr(planes_to_float(hi, lo), ref) < 2e-5
    dh = torch.randn(rows, c, generator=g).to(dev)
    ref.backward(dh.double())
    ghi = torch.empty_like(hi)
    glo = torch.empty_like(hi)
    dpre = torch.empty(rows, c, device=dev)
    L.check(lib.sfb_bias_gelu_bwd(dh.data_ptr(), y.data_ptr(), b.data_ptr(), rows, c, ghi.data_ptr(), glo.data_ptr(),
                                  dpre.data_ptr(), _st()))
    assert relerr(dpre, pre.grad) < 1e-5
    assert relerr(planes_to_float(ghi, glo), pre.grad) < 2e-5


@pytest.mark.parametrize("B,c,thw,stride", [(2, 192, (4, 8, 8), (1, 2, 2)), (3, 96, (2, 14, 10), (1, 2, 2)),
                                            (1, 384, (3, 7, 7), (1, 2, 2))])
def test_token_maxpool_forward_backward(B, c, thw, stride, cuda_device):
    """MaxPool3d(kernel s+1, stride s, padding k//2) on tokens, cls passes through (attention.py:485-489, :13-45)."""
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    T, Hh, W = thw
    ks = [s + 1 if s > 1 else s for s in stride]
    pad = [k // 2 for k in ks]
    othw = [(i + 2 * p - k) // s + 1 for i, k, s, p in zip(thw, ks, stride, pad)]
    Lin, Lo = math.prod(thw), math.prod(othw)
    g = torch.Generator().manual_seed(c)
    x = torch.randn(B, Lin + 1, c, generator=g).to(dev)
    out = torch.full((B, Lo + 1, c), float("nan"), device=dev)
    amax = torch.empty(B, Lo + 1, c, dtype=torch.uint8, device=dev)
    td = L.TokPoolDesc()
    td.x, td.out, td.argmax = x.data_ptr(), out.data_ptr(), amax.data_ptr()
    td.b, td.c, td.t, td.h, td.w = B, c, T, Hh, W
    td.ot, td.oh, td.ow = othw
    td.kt, td.kh, td.kw = ks
    td.st, td.sh, td.sw = stride
    L.check(lib.sfb_token_maxpool_fwd(C.byref(td), _st()))
    xd = x.double().requires_grad_(True)
    tok = xd[:, 1:].reshape(B, T, Hh, W, c).permute(0, 4, 1, 2, 3)
    pooled = F.max_pool3d(tok, ks, stride, pad).reshape(B, c, Lo).transpose(1, 2)
    ref = torch.cat([xd[:, :1], pooled], 1)
    assert torch.equal(out.double(), ref.detach())   # a selection: bit-exact
    dout = torch.randn(B, Lo + 1, c, generator=g).to(dev)
    ref.backward(dout.double())
    dx = torch.full((B, Lin + 1, c), float("nan"), device=dev)
    td.dout, td.dx, td.dx_accumulate = dout.data_ptr(), dx.data_ptr(), 0
    L.check(lib.sfb_token_maxpool_bwd(C.byref(td), _st()))
    assert relerr(dx, xd.grad) < 1e-6


@pytest.mark.parametrize("B,T,H,fs", [(2, 4, 64, 4), (1, 8, 112, 7), (3, 2, 32, 2)])
def test_hog_targets_kernel(B, T, H, fs, cuda_device):
    """HOG regression targets for every output token against the oracle's CPU restatement of HOGLayerC +
    _get_hog_label_3d (bit-identical to the reference on the CPU, tests/test_oracle.py).  Orientation bins are decided by
    atan2 in fp32: a pixel within an ulp of a bin edge may land in the neighbouring bin on the GPU."""
    from oracle import torch_oracle as TO
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    g = torch.Generator().manual_seed(H)
    frames = torch.randn(B, 3, T, H, H, generator=g)
    ts, nbins, cell = 2, 9, 8
    u = (H // cell) // fs
    out = torch.full((B, (T // ts) * fs * fs, 3 * nbins * u * u), float("nan"), device=dev)
    fd = frames.to(dev)
    L.check(lib.sfb_hog_targets(fd.data_ptr(), B, 3, T, H, H, ts, nbins, cell, fs, out.data_ptr(), _st()))
    torch.cuda.synchronize()
    x = frames[:, :, ::ts].transpose(1, 2)
    hog = TO.hog_layer(x.flatten(0, 1)).flatten(1, 2)
    hog = hog.permute(0, 2, 3, 1).unfold(1, u, u).unfold(2, u, u).flatten(3).view(B, T // ts, fs, fs, -1).flatten(1, 3)
    got = out.cpu()
    assert got.shape == hog.shape
    bad = ((got - hog).abs() > 1e-4).sum().item()
    assert bad <= max(4, got.numel() // 5000), f"{bad} of {got.numel()} HOG values differ by > 1e-4"


@pytest.mark.parametrize("arch,reverse", [("slowfast", False), ("mvit", True)])
def test_device_input_pipeline_matches_reference_host_functions(arch, reverse, cuda_device):
    """sfb_clip_normalize_pack / slowfast_b200.data.pack_pathways_u8 (SURVEY.md 8f-3) against the reference's own host
    functions when the reference tree is on the box (slowfast.datasets.utils.tensor_normalize + pack_pathway_output),
    else against their restatement: (x / 255 - mean) / std, THWC -> CTHW, slow pathway = frames linspace(0, T-1, T // ALPHA)."""
    from slowfast_b200.config import get_cfg
    from slowfast_b200.data import pack_pathways_u8
    preset = "SLOWFAST_8x8_R50" if arch == "slowfast" else "MVITv2_S_16x4"
    cfg = get_cfg(preset, DATA={"REVERSE_INPUT_CHANNEL": reverse, "MEAN": [0.45, 0.40, 0.5], "STD": [0.225, 0.2, 0.25]})
    B, T, H, W = 2, cfg.DATA.NUM_FRAMES, 36, 52
    g = torch.Generator().manual_seed(3)
    u8 = torch.randint(0, 256, (B, T, H, W, 3), generator=g, dtype=torch.uint8)
    got = pack_pathways_u8(u8.to(cuda_device), cfg)
    want = []
    ref_fns = None
    try:
        from oracle import refshim
        if refshim.reference_available():
            refshim.install()
            from slowfast.datasets import utils as dsu
            rcfg = refshim.load_cfg("Kinetics/SLOWFAST_8x8_R50.yaml" if arch == "slowfast" else "Kinetics/MVITv2_S_16x4.yaml",
                                    ["DATA.REVERSE_INPUT_CHANNEL", reverse])
            ref_fns = (dsu, rcfg)
    except Exception:  # noqa: BLE001
        ref_fns = None
    for b in range(B):
        if ref_fns is not None:
            dsu, rcfg = ref_fns
            fr = dsu.tensor_normalize(u8[b], list(cfg.DATA.MEAN), list(cfg.DATA.STD)).permute(3, 0, 1, 2)
            want.append(dsu.pack_pathway_output(rcfg, fr))
        else:
            fr = ((u8[b].float() / 255.0 - torch.tensor(cfg.DATA.MEAN)) / torch.tensor(cfg.DATA.STD)).permute(3, 0, 1, 2)
            if reverse:
                fr = fr[[2, 1, 0]]
            if arch == "slowfast":
                want.append([fr.index_select(1, torch.linspace(0, T - 1, T // cfg.SLOWFAST.ALPHA).long()), fr])
            else:
                want.append([fr])
    assert len(got) == len(want[0])
    for p in range(len(got)):
        ref = torch.stack([w[p] for w in want])
        assert got[p].shape == ref.shape
        assert torch.allclose(got[p].cpu(), ref, rtol=1e-6, atol=1e-6), (got[p].cpu() - ref).abs().max()


@pytest.mark.parametrize("q_thw,bh,rel,nsplit", [((8, 7, 7), 2, True, 3), ((8, 14, 14), 3, True, 3), ((8, 28, 28), 1, True, 3),
                                                  ((8, 14, 14), 2, False, 3), ((8, 14, 14), 2, True, 1)])
def test_fused_attention_forward(q_thw, bh, rel, nsplit, cuda_device):
    """sfb_attn_fwd (csrc/attn_fused.cu): O = softmax(scale q k^T + rel-pos bias) v with the scores kept in shared memory, for the
    8x7x7 key grid (Nk = 393), against fp64 on the operand values the kernel saw (split planes); also the normalised P planes
    it leaves for the backward and the log-sum-exp.  Tile tails (Nq = 393, 1569, 6273 are not multiples of 64), cls row /
    column without bias, and the no-rel-pos variant are covered."""
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    k_thw = (8, 7, 7)
    hd = 96
    qt, qh, qw = q_thw
    kt, kh, kw = k_thw
    Lq, Lk = qt * qh * qw, kt * kh * kw
    Nq, Nk = Lq + 1, Lk + 1
    assert lib.sfb_attn_fwd_supported(Nk, hd, kt, kh, kw)
    Nkp = (Nk + 7) // 8 * 8
    Lh, Lw, Lt = 2 * max(qh, kh) - 1, 2 * max(qw, kw) - 1, 2 * max(qt, kt) - 1
    Ltp = (Lh + Lw + Lt + 7) // 8 * 8
    g = torch.Generator().manual_seed(Lq + bh)

    def planes(x):
        hi = x.bfloat16()
        lo = (x - hi.float()).bfloat16()
        return hi.contiguous(), lo.contiguous()

    q = torch.randn(bh, Nq, hd, generator=g).to(dev)
    k = torch.randn(bh, Nk, hd, generator=g).to(dev)
    v = torch.randn(bh, Nk, hd, generator=g).to(dev)
    qh_, ql_ = planes(q)
    kh_, kl_ = planes(k)
    vh_, vl_ = planes(v)

    def val(hi, lo):
        return hi.double() + (lo.double() if nsplit == 3 else 0)

    rq = None
    if rel:
        rq = torch.zeros(bh * Lq, Ltp)
        rq[:, :Lh + Lw + Lt] = torch.randn(bh * Lq, Lh + Lw + Lt, generator=g)
        rq = rq.to(dev)
    out = torch.full((bh, Nq, hd), float("nan"), device=dev)
    p_hi = torch.full((bh * Nq, Nkp), float("nan"), dtype=torch.bfloat16, device=dev)
    p_lo = torch.full_like(p_hi, float("nan"))
    lse = torch.full((bh * Nq,), float("nan"), device=dev)
    d = L.AttnFwdDesc()
    d.q_hi, d.q_lo, d.k_hi, d.k_lo, d.v_hi, d.v_lo = (qh_.data_ptr(), ql_.data_ptr(), kh_.data_ptr(), kl_.data_ptr(),
                                                      vh_.data_ptr(), vl_.data_ptr())
    d.rq, d.rq_pitch = (rq.data_ptr() if rel else None), Ltp
    d.bh, d.nq, d.nk, d.hd = bh, Nq, Nk, hd
    d.qt, d.qh, d.qw = q_thw
    d.kt, d.kh, d.kw = k_thw
    d.scale = hd ** -0.5
    d.out, d.p_hi, d.p_lo, d.p_pitch, d.lse = out.data_ptr(), p_hi.data_ptr(), (p_lo.data_ptr() if nsplit == 3 else None), Nkp, lse.data_ptr()
    d.nsplit = nsplit
    L.check(lib.sfb_attn_fwd(C.byref(d), _st()), "sfb_attn_fwd")
    torch.cuda.synchronize()
    # fp64 reference on the plane values
    Q, K, V = val(qh_, ql_).cpu(), val(kh_, kl_).cpu(), val(vh_, vl_).cpu()
    S = (Q @ K.transpose(1, 2)) * hd ** -0.5
    if rel:
        r = rq.double().cpu().view(bh, qt, qh, qw, Ltp)
        ih, iw, it = _rel_index(qh, kh), _rel_index(qw, kw), _rel_index(qt, kt)
        rel_h = torch.gather(r, 4, ih[None, None, :, None, :].expand(bh, qt, qh, qw, kh))
        rel_w = torch.gather(r, 4, iw[None, None, None, :, :].expand(bh, qt, qh, qw, kw) + Lh)
        rel_t = torch.gather(r, 4, it[None, :, None, None, :].expand(bh, qt, qh, qw, kt) + Lh + Lw)
        bias = (rel_t[..., :, None, None] + rel_h[..., None, :, None] + rel_w[..., None, None, :]).reshape(bh, Lq, Lk)
        S = S + F.pad(bias, (1, 0, 1, 0))
    Pr = torch.softmax(S, dim=-1)
    Or = Pr @ V
    tol = 3e-5 if nsplit == 3 else 2e-2
    got_p = (p_hi.float() + (p_lo.float() if nsplit == 3 else 0)).cpu().view(bh, Nq, Nkp)
    assert not torch.isnan(out).any() and not torch.isnan(got_p).any()
    assert relerr(got_p[..., :Nk], Pr) < tol, relerr(got_p[..., :Nk], Pr)
    assert (got_p[..., Nk:] == 0).all()
    assert relerr(out.cpu(), Or) < tol, relerr(out.cpu(), Or)
    assert relerr(lse.cpu().view(bh, Nq), torch.logsumexp(S, dim=-1)) < (1e-5 if nsplit == 3 else 2e-2)


@pytest.mark.parametrize("q_thw,bh,rel,nsplit", [((8, 7, 7), 2, True, 3), ((8, 14, 14), 3, True, 3), ((8, 28, 28), 1, True, 3),
                                                  ((8, 14, 14), 2, False, 3), ((8, 14, 14), 2, True, 1)])
def test_fused_attention_backward_ds(q_thw, bh, rel, nsplit, cuda_device):
    """sfb_attn_bwd_ds (csrc/attn_fused.cu): dP = dO v^T in shared memory, dS = P (dP - sum_k P dP) as planes, and the gradient of the
    decomposed rel-pos bias dRQ, against fp64 on the
    operand values the kernel saw."""
    from slowfast_b200 import lib as L
    lib, dev = L.load(), cuda_device
    k_thw = (8, 7, 7)
    hd = 96
    qt, qh, qw = q_thw
    kt, kh, kw = k_thw
    Lq, Lk = qt * qh * qw, kt * kh * kw
    Nq, Nk = Lq + 1, Lk + 1
    Nkp = (Nk + 7) // 8 * 8
    assert Nkp == 400
    Lh, Lw, Lt = 2 * max(qh, kh) - 1, 2 * max(qw, kw) - 1, 2 * max(qt, kt) - 1
    Ltp = (Lh + Lw + Lt + 7) // 8 * 8
    g = torch.Generator().manual_seed(Lq + 3 * bh)

    def planes(x):
        hi = x.bfloat16()
        lo = (x - hi.float()).bfloat16()
        return hi.contiguous(), lo.contiguous()

    def val(hi, lo):
        return hi.double() + (lo.double() if nsplit == 3 else 0)

    dO = torch.randn(bh, Nq, hd, generator=g).to(dev)
    v = torch.randn(bh, Nk, hd, generator=g).to(dev)
    P = torch.zeros(bh, Nq, Nkp)
    P[..., :Nk] = torch.softmax(torch.randn(bh, Nq, Nk, generator=g) * 2.0, dim=-1)
    P = P.to(dev)
    doh, dol = planes(dO)
    vh, vl = planes(v)
    ph, plo = planes(P.view(bh * Nq, Nkp))
    ds_hi = torch.full((bh * Nq, Nkp), float("nan"), dtype=torch.bfloat16, device=dev)
    ds_lo = torch.full_like(ds_hi, float("nan"))
    drq = torch.full((bh * Lq, Ltp), float("nan"), device=dev) if rel else None
    d = L.AttnBwdDesc()
    d.do_hi, d.do_lo, d.v_hi, d.v_lo = doh.data_ptr(), dol.data_ptr(), vh.data_ptr(), vl.data_ptr()
    d.p_hi, d.p_lo, d.p_pitch = ph.data_ptr(), plo.data_ptr(), Nkp
    d.ds_hi, d.ds_lo, d.ds_pitch = ds_hi.data_ptr(), (ds_lo.data_ptr() if nsplit == 3 else None), Nkp
    d.drq, d.rq_pitch = (drq.data_ptr() if rel else None), Ltp
    d.bh, d.nq, d.nk, d.hd = bh, Nq, Nk, hd
    d.qt, d.qh, d.qw = q_thw
    d.kt, d.kh, d.kw = k_thw
    d.nsplit = nsplit
    L.check(lib.sfb_attn_bwd_ds(C.byref(d), _st()), "sfb_attn_bwd_ds")
    torch.cuda.synchronize()
    DO, V, Pv = val(doh, dol).cpu(), val(vh, vl).cpu(), val(ph, plo).cpu().view(bh, Nq, Nkp)[..., :Nk]
    dP = DO @ V.transpose(1, 2)
    dS = Pv * (dP - (Pv * dP).sum(-1, keepdim=True))
    got = (ds_hi.float() + (ds_lo.float() if nsplit == 3 else 0)).cpu().view(bh, Nq, Nkp)
    tol = 3e-5 if nsplit == 3 else 2e-2
    assert not torch.isnan(got).any()
    assert relerr(got[..., :Nk], dS) < tol, relerr(got[..., :Nk], dS)
    assert (got[..., Nk:] == 0).all()
    if rel:
        # dRQ[q, bin] = sum of dS over the keys whose (kh | kw | kt) coordinate looks that bin up, for non-cls (q, k)
        gS = dS[:, 1:, 1:].reshape(bh, qt, qh, qw, kt, kh, kw)
        ih, iw, it = _rel_index(qh, kh), _rel_index(qw, kw), _rel_index(qt, kt)
        ref = torch.zeros(bh, qt, qh, qw, Ltp, dtype=torch.float64)
        ref.scatter_add_(4, ih[None, None, :, None, :].expand(bh, qt, qh, qw, kh), gS.sum((4, 6)))
        ref.scatter_add_(4, iw[None, None, None, :, :].expand(bh, qt, qh, qw, kw) + Lh, gS.sum((4, 5)))
        ref.scatter_add_(4, it[None, :, None, None, :].expand(bh, qt, qh, qw, kt) + Lh + Lw, gS.sum((5, 6)))
        assert not torch.isnan(drq).any()
        assert relerr(drq.cpu().view(bh, qt, qh, qw, Ltp), ref) < (5e-5 if nsplit == 3 else 2e-2)
