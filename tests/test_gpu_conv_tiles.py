"""GPU parity of the implicit-GEMM convolution at every compiled tile width and on the split-K path, against PyTorch fp64
on the operands the kernel saw (tolerances as in test_gpu_kernels.py)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {1: 1e-5, 3: 2e-5}


def _ops():
    from slowfast_b200 import ops
    return ops


def _setup(n, t, h, w, cin, cout, k, pad, nsplit, dev, seed=0):
    ops = _ops()
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(n, t, h, w, cin, generator=g).to(dev)
    wt = (torch.randn(cout, cin, *k, generator=g) / (cin * k[0] * k[1] * k[2]) ** 0.5).to(dev)
    xp = ops.alloc_planes(n, t, h, w, cin, nsplit, dev)
    ops.split_planes(x, xp)
    f = ops.alloc_filter(cout, k[0] * k[1] * k[2], cin, nsplit, dev)
    ops.filter_pack(wt, f)
    geom = ops.fprop_geom(xp, k, (1, 1, 1), pad)
    xr = xp.to_float().double() if nsplit == 3 else xp.hi[..., :cin].double()
    wr = (f.hi.double() + (f.lo.double() if nsplit == 3 else 0)).reshape(cout, -1, f.cols_pad)[:, :, :cin]
    wr = wr.reshape(cout, *k, cin).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(xr.permute(0, 4, 1, 2, 3), wr, padding=pad).permute(0, 2, 3, 4, 1)
    return xp, f, geom, ref


def relerr(got, ref):
    return ((got.double() - ref.double()).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _check_stats(stats, ref):
    rs = ref.reshape(-1, ref.shape[-1])
    assert relerr(stats[0].double().sum(1), rs.sum(0)) < 1e-4
    assert relerr(stats[1].double().sum(1), (rs * rs).sum(0)) < 1e-4


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("cout", [16, 32, 48, 64, 80, 96, 112, 128])
def test_conv_tile_width(cout, nsplit, cuda_device):
    """One output tile column per launch at each width 16..128 (cout <= 128 picks BN = cout), K = 576 + a 3-tap
    16-channel layer whose single k-block is mostly zero chunks."""
    ops = _ops()
    for cin, k, pad in ((64, (1, 3, 3), (0, 1, 1)), (16, (3, 1, 1), (1, 0, 0))):
        xp, f, geom, ref = _setup(2, 4, 14, 14, cin, cout, k, pad, nsplit, cuda_device)
        ot, oh, ow = geom.out
        y = torch.full((2, ot, oh, ow, cout), float("nan"), device=cuda_device)
        strides = (ot * oh * ow * cout, oh * ow * cout, ow * cout, cout)
        stats = torch.zeros(2, cout, ops.conv_stats_tiles(xp, f, geom, y, strides, nsplit=nsplit), device=cuda_device)
        ops.conv_igemm(xp, f, geom, y, strides, stats=stats, nsplit=nsplit)
        assert relerr(y, ref) < TOL[nsplit]
        _check_stats(stats, ref)


# 2 x 4 x 40 x 40 = 12 800 rows, 128 output channels: 100 tiles (3/4 of a wave on 132 SMs), K = 1728 (27 k-blocks)
SPLIT = dict(n=2, t=4, h=40, w=40, cin=64, cout=128, k=(3, 3, 3), pad=(1, 1, 1))


def _split_problem(nsplit, dev):
    s = SPLIT
    return _setup(s["n"], s["t"], s["h"], s["w"], s["cin"], s["cout"], s["k"], s["pad"], nsplit, dev, seed=3)


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("pitch", [128, 192])
def test_conv_split_k_overwrite_stats(pitch, nsplit, cuda_device):
    """Overwrite launch split over K, into a dense output and into channels [32, 160) of a 192-channel tensor: the
    zero fill and the red.add slices touch only the view, and the BatchNorm partials sum to the fp64 column sums."""
    ops = _ops()
    xp, f, geom, ref = _split_problem(nsplit, cuda_device)
    cout = SPLIT["cout"]
    ot, oh, ow = geom.out
    off = 0 if pitch == cout else 32
    buf = torch.full((SPLIT["n"], ot, oh, ow, pitch), 7.0, device=cuda_device)
    strides = (ot * oh * ow * pitch, oh * ow * pitch, ow * pitch, pitch)
    tiles = ops.conv_stats_tiles(xp, f, geom, buf, strides, out_offset=off, nsplit=nsplit)
    stats = torch.full((2, cout, tiles), float("nan"), device=cuda_device)
    assert ops.conv_ksplit(xp, f, geom, buf, strides, out_offset=off, stats=stats, nsplit=nsplit) > 1
    ops.conv_igemm(xp, f, geom, buf, strides, out_offset=off, stats=stats, nsplit=nsplit)
    assert relerr(buf[..., off:off + cout], ref) < TOL[nsplit]
    if pitch != cout:
        assert torch.all(buf[..., :off] == 7.0) and torch.all(buf[..., off + cout:] == 7.0)
    _check_stats(stats, ref)


@pytest.mark.parametrize("mode", [1, 2])
def test_conv_split_k_accumulate(mode, cuda_device):
    """accumulate = 1 / 2 on the split-K path: every slice adds its partial sum to what the destination holds."""
    ops = _ops()
    xp, f, geom, ref = _split_problem(3, cuda_device)
    cout = SPLIT["cout"]
    ot, oh, ow = geom.out
    strides = (ot * oh * ow * cout, oh * ow * cout, ow * cout, cout)
    pre = torch.randn(SPLIT["n"], ot, oh, ow, cout, generator=torch.Generator().manual_seed(9)).to(cuda_device)
    y = pre.clone()
    assert ops.conv_ksplit(xp, f, geom, y, strides, accumulate=mode, nsplit=3) > 1
    ops.conv_igemm(xp, f, geom, y, strides, accumulate=mode, nsplit=3)
    assert relerr(y - pre, ref) < TOL[3]


def test_conv_split_k_rule(cuda_device):
    """Split-K is chosen from the problem shape: 3.03 waves are split; a tiny grid and a single k-block are not."""
    ops = _ops()
    dev = cuda_device
    for (n, h, w, cin, cout, k, pad) in ((2, 80, 80, 64, 128, (3, 3, 3), (1, 1, 1)),    # 400 tiles: 3.03 waves
                                         (1, 8, 8, 64, 128, (3, 3, 3), (1, 1, 1)),      # 2 tiles
                                         (2, 40, 40, 64, 128, (1, 1, 1), (0, 0, 0))):   # K = 64: one k-block
        xp, f, geom, _ = _setup(n, 4, h, w, cin, cout, k, pad, 1, dev)
        ot, oh, ow = geom.out
        y = torch.empty(n, ot, oh, ow, cout, device=dev)
        strides = (ot * oh * ow * cout, oh * ow * cout, ow * cout, cout)
        want = 1 if (h == 8 or k == (1, 1, 1)) else None
        s = ops.conv_ksplit(xp, f, geom, y, strides, nsplit=1)
        if want is not None:
            assert s == want, (h, k, s)
        else:
            assert s > 1, (h, k, s)
