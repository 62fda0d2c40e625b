"""GPU parity of the implicit-GEMM convolution's register epilogue where the tile schedule matters: CTAs that run
several tiles (so both consumer warpgroups of a CTA take turns), an M tail that is not a multiple of 128 with BatchNorm
partials, a channel-slice output, and the strided data-gradient scatter at the widest tile.  Against PyTorch fp64 on
the operands the kernel saw (tolerances as in test_gpu_kernels.py)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {1: 1e-5, 3: 2e-5}


def _ops():
    from slowfast_b200 import ops
    return ops


def relerr(got, ref):
    return ((got.double() - ref.double()).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _planes(x, nsplit):
    ops = _ops()
    n, t, h, w, c = x.shape
    p = ops.alloc_planes(n, t, h, w, c, nsplit, x.device)
    ops.split_planes(x.contiguous(), p)
    return p


def _value(p, nsplit):
    return p.to_float().double() if nsplit == 3 else p.hi[..., p.c0:p.c0 + p.c].double()


# 4 x 8 x 37 x 37 = 43 808 rows: 343 tiles, the last one 32 rows; three k-blocks (no split-K).  On a 132-SM H100 every
# CTA runs two or three tiles (343 = 2 x 132 + 79), so both consumers work and consumer 0 takes a second turn in 79 of
# them.  116 output channels: a 128-wide tile whose last 12 columns are past cout.
MANY = dict(n=4, t=8, h=37, w=37, cin=192, cout=116)


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("pitch", [116, 160])
def test_conv_many_tiles_per_cta(pitch, mode, nsplit, cuda_device):
    """Overwrite (with BatchNorm partials), read-add-write and red.add into a dense output and into channels
    [24, 140) of a 160-channel tensor: every row of the M tail is stored, nothing outside the view is touched, and a
    consumer's second tile reuses its row table and scratch."""
    ops = _ops()
    dev = cuda_device
    s = MANY
    g = torch.Generator().manual_seed(21)
    x = torch.randn(s["n"], s["t"], s["h"], s["w"], s["cin"], generator=g).to(dev)
    wt = (torch.randn(s["cout"], s["cin"], 1, 1, 1, generator=g) / s["cin"] ** 0.5).to(dev)
    xp = _planes(x, nsplit)
    f = ops.alloc_filter(s["cout"], 1, s["cin"], nsplit, dev)
    ops.filter_pack(wt, f)
    geom = ops.fprop_geom(xp, (1, 1, 1), (1, 1, 1), (0, 0, 0))
    wr = (f.hi.double() + (f.lo.double() if nsplit == 3 else 0)).reshape(s["cout"], -1, f.cols_pad)[:, :, :s["cin"]]
    ref = torch.einsum("nthwc,oc->nthwo", _value(xp, nsplit), wr[:, 0])

    ot, oh, ow = geom.out
    off = 0 if pitch == s["cout"] else 24
    pre = torch.randn(s["n"], ot, oh, ow, pitch, generator=torch.Generator().manual_seed(22)).to(dev)
    buf = pre.clone()
    strides = (ot * oh * ow * pitch, oh * ow * pitch, ow * pitch, pitch)
    assert ops.conv_ksplit(xp, f, geom, buf, strides, out_offset=off, accumulate=mode, nsplit=nsplit) == 1
    stats = None
    if mode == 0:
        tiles = ops.conv_stats_tiles(xp, f, geom, buf, strides, out_offset=off, nsplit=nsplit)
        assert tiles == 343
        stats = torch.full((2, s["cout"], tiles), float("nan"), device=dev)
    ops.conv_igemm(xp, f, geom, buf, strides, out_offset=off, accumulate=mode, stats=stats, nsplit=nsplit)
    got = buf[..., off:off + s["cout"]] - (pre[..., off:off + s["cout"]] if mode else 0)
    assert relerr(got, ref) < TOL[nsplit]
    if pitch != s["cout"]:
        assert torch.equal(buf[..., :off], pre[..., :off]) and torch.equal(buf[..., off + s["cout"]:],
                                                                              pre[..., off + s["cout"]:])
    if stats is not None:
        rs = ref.reshape(-1, s["cout"])
        assert relerr(stats[0].double().sum(1), rs.sum(0)) < 1e-4
        assert relerr(stats[1].double().sum(1), (rs * rs).sum(0)) < 1e-4


@pytest.mark.parametrize("nsplit", [1, 3])
def test_conv_dgrad_strided_scatter_bn128(nsplit, cuda_device):
    """Data gradient of a 1x3x3 / stride-2 convolution with 128 input channels: every strided sub-problem runs at tile
    width 128 and scatters its rows through the strided output view."""
    ops = _ops()
    from slowfast_b200.conv_plan import dgrad_out_view, dgrad_plan
    dev = cuda_device
    n, t, h, w, cin, cout, k, stride, pad = 2, 4, 28, 28, 128, 96, (1, 3, 3), (1, 2, 2), (0, 1, 1)
    g = torch.Generator().manual_seed(31)
    wt = (torch.randn(cout, cin, *k, generator=g) / (cin * 9) ** 0.5).to(dev)
    xp = ops.alloc_planes(n, t, h, w, cin, nsplit, dev)
    geom = ops.fprop_geom(xp, k, stride, pad)
    ot, oh, ow = geom.out
    dyp = _planes(torch.randn(n, ot, oh, ow, cout, generator=g).to(dev), nsplit)
    plan = dgrad_plan((t, h, w), k, stride, pad)
    dx = torch.full((n, t, h, w, cin), float("nan"), device=dev)
    if plan.needs_zero_fill:
        dx.zero_()
    for sub in plan.subs:
        f = ops.alloc_filter(cin, len(sub.tapmap), cout, nsplit, dev)
        ops.filter_pack(wt, f, tapmap=sub.tapmap, transpose=True)
        off, strides = dgrad_out_view((t, h, w), stride, sub, cin)
        ops.conv_igemm(dyp, f, ops.ConvGeom(sub.k, (1, 1, 1), sub.low, sub.out), dx, strides, out_offset=off,
                       nsplit=nsplit)
    wr = wt.bfloat16()
    wr = wr.double() + ((wt - wr.float()).bfloat16().double() if nsplit == 3 else 0)
    xin = torch.zeros(n, cin, t, h, w, dtype=torch.float64, device=dev, requires_grad=True)
    yy = F.conv3d(xin, wr, stride=stride, padding=pad)
    (ref,) = torch.autograd.grad(yy, xin, _value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert not torch.isnan(dx).any()
    assert relerr(dx, ref.permute(0, 2, 3, 4, 1)) < TOL[nsplit]
