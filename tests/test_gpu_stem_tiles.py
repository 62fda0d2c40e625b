"""GPU: every compile-time instantiation of the stem kernels against fp64 conv3d / autograd on the operands the kernels
saw, with the BatchNorm partials against fp64 column sums and the weight gradient accumulated into a non-zero matrix.

W-shift stem (csrc/conv_stem.cu): forward tile widths 16 / 32 / 48 / 64 (cout rounded up to 16), weight gradient with
2 or 4 folded W taps and 3 or 4 (kt, kh) pairs per CTA, including groups padded past the last pair.  Toeplitz stem
(csrc/conv_stem8.cu): 1, 3, 4 and 5 T taps, one and several bands, fewer steps than CTAs.  The extents leave partial
128-pixel tiles, odd T / H tails and partial last waves.  The engine's fast-pathway stem unit, forward and backward, at
the 158-wide short-cycle crop of multigrid training."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernels import TOL, make_planes, planes_value, relerr

pytestmark = pytest.mark.gpu

STEM_CASES = [
    # n, t, h, w, cin, cout, k, stride, pad          forward BN; weight-gradient folded taps x pairs per CTA
    (1, 3, 17, 46, 3, 8, (1, 7, 7), (1, 2, 2), (0, 3, 3)),     # BN 16; 4 x 4 (7 pairs: second group padded)
    (2, 2, 9, 38, 3, 16, (3, 7, 7), (1, 2, 2), (1, 3, 3)),     # BN 16; 4 x 3 (21 pairs)
    (1, 4, 11, 30, 3, 24, (1, 3, 3), (1, 2, 2), (0, 1, 1)),    # BN 32; 2 x 3 (X3D conv_xy)
    (1, 2, 13, 270, 3, 32, (1, 7, 7), (1, 2, 2), (0, 3, 3)),   # BN 32; output row of 135 pixels = two W tiles
    (1, 3, 10, 42, 3, 40, (3, 3, 3), (1, 2, 2), (1, 1, 1)),    # BN 48; 2 x 3 (9 pairs)
    (2, 2, 15, 34, 3, 48, (5, 7, 7), (1, 2, 2), (2, 3, 3)),    # BN 48; 4 x 4 (35 pairs)
    (1, 2, 12, 26, 3, 56, (1, 7, 7), (1, 2, 2), (0, 3, 3)),    # BN 64
    (2, 2, 6, 22, 3, 8, (1, 2, 3), (1, 2, 2), (0, 0, 1)),      # 2 x 3 (two pairs, one padded)
    (2, 8, 32, 64, 3, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3)),    # SlowFast slow pathway / C2D / Slow stem
    (1, 4, 32, 64, 3, 64, (5, 7, 7), (1, 2, 2), (2, 3, 3)),    # I3D stem
    (1, 5, 20, 48, 3, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3)),     # SlowFast fast-pathway stem in the W-shift layout
]


def _rnd(v, nsplit):
    hi = v.bfloat16()
    return hi.double() + ((v - hi.float()).bfloat16().double() if nsplit == 3 else 0)


def _check_stats(stats, ref, cout):
    rs = ref.reshape(-1, cout)
    assert relerr(stats[0].double().sum(1), rs.sum(0)) < 1e-4
    assert relerr(stats[1].double().sum(1), (rs * rs).sum(0)) < 1e-4


def _check_wgrad(dwm, pre, x_r, dyp, geo, k, stride, pad, nsplit, dev):
    from slowfast_b200 import ops
    cout, cin = geo.cout, geo.cin
    dw = torch.zeros(cout, cin, *k, device=dev)
    ops.stem_filter_unfold_grad(dwm - pre, dw, geo)
    wref = torch.zeros(cout, cin, *k, dtype=torch.float64, device=dev, requires_grad=True)
    (gref,) = torch.autograd.grad(F.conv3d(x_r, wref, stride=stride, padding=pad), wref,
                                  planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert relerr(dw, gref) < TOL[nsplit] * 2


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", STEM_CASES)
def test_stem_wshift_tiles(case, nsplit, cuda_device):
    from slowfast_b200 import ops
    dev = cuda_device
    n, t, h, w, cin, cout, k, stride, pad = case
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randn(n, cin, t, h, w, generator=g).to(dev)
    wt = (torch.randn(cout, cin, *k, generator=g) / (cin * k[0] * k[1] * k[2]) ** 0.5).to(dev)
    geo = ops.StemGeom(cin, cout, k, stride, pad)
    assert ops.stem_supported(cin, k, stride, pad, w)
    xp = ops.alloc_planes(n, t, h, w // 2, 8, nsplit, dev)
    ops.stem_input_fold(x, xp)
    f = ops.FilterMat(torch.empty(cout, geo.kfold, dtype=torch.bfloat16, device=dev),
                      torch.empty(cout, geo.kfold, dtype=torch.bfloat16, device=dev) if nsplit == 3 else None,
                      cout, geo.kfold // 8, 8)
    ops.stem_filter_fold(wt, geo, f)
    ot, oh, ow = geo.out_dims(t, h, w)
    y = torch.full((n, ot, oh, ow, cout), float("nan"), device=dev)
    stats = torch.zeros(2, cout, ops.stem_m_tiles(xp, geo), device=dev)
    ops.stem_fprop(xp, f, geo, y, stats, nsplit=nsplit)
    xr = _rnd(x, nsplit)
    ref = F.conv3d(xr, _rnd(wt, nsplit), stride=stride, padding=pad).permute(0, 2, 3, 4, 1)
    assert not torch.isnan(y).any()
    assert relerr(y, ref) < TOL[nsplit]
    _check_stats(stats, ref, cout)

    dyp = make_planes(torch.randn(n, ot, oh, ow, cout, generator=g).to(dev), nsplit)
    pre = torch.randn(cout, geo.kfold, generator=g).to(dev)
    dwm = pre.clone()
    ops.stem_wgrad(xp, dyp, geo, dwm, nsplit=nsplit)
    _check_wgrad(dwm, pre, xr, dyp, geo, k, stride, pad, nsplit, dev)


STEM8_CASES = [
    # n, t, h, w, kt   (3 -> 8 channels, [kt,7,7], stride (1,2,2), pad (kt//2,3,3))
    (1, 3, 16, 32, 5),       # fewer frames than T taps, one band
    (2, 5, 32, 48, 3),       # odd T, two bands
    (1, 5, 16, 64, 4),       # even T taps: one more output frame than input frames
    (3, 2, 16, 16, 5),       # 8 output pixels per row: one group per row
    (2, 3, 48, 224, 1),      # kt = 1, the full 112-pixel output row
    (2, 8, 224, 224, 5),     # the fast pathway's extent at batch 2
]


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", STEM8_CASES)
def test_stem8_tiles(case, nsplit, cuda_device):
    from slowfast_b200 import ops
    dev = cuda_device
    n, t, h, w, kt = case
    cin, cout, k, stride, pad = 3, 8, (kt, 7, 7), (1, 2, 2), (kt // 2, 3, 3)
    g = torch.Generator(device="cpu").manual_seed(13)
    x = torch.randn(n, cin, t, h, w, generator=g).to(dev)
    wt = (torch.randn(cout, cin, *k, generator=g) / (cin * k[0] * k[1] * k[2]) ** 0.5).to(dev)
    geo = ops.StemGeom(cin, cout, k, stride, pad)
    assert ops.stem8_supported(cin, cout, k, stride, pad, t, h, w)
    xp = ops.alloc_planes(*ops.stem8_plane_dims(n, t, h, w), nsplit, dev)
    ops.stem8_input_fold(x, xp)
    zh = torch.empty(kt * ops.STEM8_ZG * 64, dtype=torch.bfloat16, device=dev)
    zl = torch.empty_like(zh) if nsplit == 3 else None
    ops.stem8_filter_fold(wt, zh, zl)
    ot, oh, ow = geo.out_dims(t, h, w)
    y = torch.full((n, ot, oh, ow, cout), float("nan"), device=dev)
    stats = torch.zeros(2, cout, ops.stem8_m_tiles(xp, geo), device=dev)
    ops.stem8_fprop(xp, zh, zl, geo, y, stats, nsplit=nsplit)
    xr = _rnd(x, nsplit)
    ref = F.conv3d(xr, _rnd(wt, nsplit), stride=stride, padding=pad).permute(0, 2, 3, 4, 1)
    assert not torch.isnan(y).any()
    assert relerr(y, ref) < TOL[nsplit]
    _check_stats(stats, ref, cout)

    dyp = make_planes(torch.randn(n, ot, oh, ow, cout, generator=g).to(dev), nsplit)
    pre = torch.randn(cout, geo.kfold, generator=g).to(dev)
    dwm = pre.clone()
    ops.stem8_wgrad(xp, dyp, geo, dwm, nsplit=nsplit)
    _check_wgrad(dwm, pre, xr, dyp, geo, k, stride, pad, nsplit, dev)


@pytest.mark.parametrize("nsplit", [1, 3])
def test_fast_stem_unit_at_crop_158(nsplit, cuda_device):
    """The engine's fast-pathway stem unit (StemConvBN: Conv3d 3 -> 8, 5x7x7, stride (1,2,2), + train-mode BatchNorm)
    forward and backward on a 158 x 158 clip, multigrid's short-cycle crop: 158 is not a multiple of 16, so the W-shift
    kernels take it instead of the Toeplitz ones.  Conv output and the conv / BN parameter gradients against fp64
    conv3d + batch_norm autograd on the fp32 clip and weights."""
    import torch.nn as nn
    from slowfast_b200 import ops
    from slowfast_b200.engine import Ctx, StemConvBN
    dev = cuda_device
    n, t, h, w = 2, 4, 158, 158
    k, stride, pad = (5, 7, 7), (1, 2, 2), (2, 3, 3)
    g = torch.Generator().manual_seed(17)
    conv = nn.Conv3d(3, 8, k, stride, pad, bias=False)
    bn = nn.BatchNorm3d(8)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / conv.weight[0].numel() ** 0.5)
        bn.weight.copy_(torch.rand(8, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(8, generator=g) * 0.2)
    conv, bn = conv.to(dev), bn.to(dev)
    ctx = Ctx(nsplit)
    ctx.device = dev
    assert StemConvBN.supported(conv, w)
    unit = StemConvBN("s1.pathway1_stem", conv, bn, ctx)
    x = torch.randn(n, 3, t, h, w, generator=g).to(dev)
    xin = unit.pack_input(x, ("in", 1))
    assert not unit.t8
    y = unit.fprop(xin.planes)
    ctx.begin_backward([conv.weight, bn.weight, bn.bias])
    dz = torch.randn(y.shape, generator=g).to(dev)
    unit.bwd(ops.f32view(dz), None, None)
    torch.cuda.synchronize()

    wr, gr, br = (p.detach().double().requires_grad_(True) for p in (conv.weight, bn.weight, bn.bias))
    yr = F.conv3d(x.double(), wr, stride=stride, padding=pad)
    F.batch_norm(yr, None, None, gr, br, training=True, eps=bn.eps).backward(dz.double().permute(0, 4, 1, 2, 3))
    # parity: split-bf16 operands; fast: bf16 operands (clip, weights and the conv-output gradient)
    tol = 1e-4 if nsplit == 3 else 2e-2
    assert relerr(y, yr.detach().permute(0, 2, 3, 4, 1)) < tol
    assert relerr(ctx.grad_of(conv.weight), wr.grad) < tol
    assert relerr(ctx.grad_of(bn.weight), gr.grad) < tol
    assert relerr(ctx.grad_of(bn.bias), br.grad) < tol
