"""GPU parity of every kernel behind the C ABI against plain PyTorch (fp64 on the operands the kernel saw).

Tolerances: nsplit=1 results must match the fp64 product of the bf16-rounded operands to fp32 accumulation error
(<= 1e-5 relative to the output scale for reductions up to K = 4608); nsplit=3 must match the fp64 product of the
(hi+lo) operands to the dropped lo*lo term (<= 2e-5).  Index outputs (pool argmax routing) are compared exactly.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {1: 1e-5, 3: 2e-5}


def _ops():
    from slowfast_b200 import ops
    return ops


def make_planes(x, nsplit):
    """x: fp32 NDHWC cuda tensor -> Planes (split done by the library kernel)."""
    ops = _ops()
    n, t, h, w, c = x.shape
    p = ops.alloc_planes(n, t, h, w, c, nsplit, x.device)
    ops.split_planes(x.contiguous(), p)
    return p


def planes_value(p, nsplit):
    return p.to_float().double() if nsplit == 3 else p.hi[..., p.c0:p.c0 + p.c].double()


def relerr(got, ref):
    return ((got.double() - ref.double()).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


CONV_CASES = [
    # n, t, h, w, cin, cout, k, stride, pad
    (2, 4, 14, 14, 64, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    (2, 4, 14, 14, 128, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    (2, 4, 28, 28, 64, 64, (1, 3, 3), (1, 2, 2), (0, 1, 1)),
    (2, 8, 14, 14, 32, 8, (3, 1, 1), (1, 1, 1), (1, 0, 0)),
    (2, 8, 14, 14, 8, 8, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    (1, 32, 7, 7, 16, 32, (7, 1, 1), (4, 1, 1), (3, 0, 0)),
    (2, 4, 14, 14, 80, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    (2, 4, 14, 14, 64, 128, (1, 1, 1), (1, 2, 2), (0, 0, 0)),
    (1, 2, 32, 32, 8, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3)),
    (2, 4, 7, 7, 512, 512, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
]


def _conv_setup(case, nsplit, dev, seed=0):
    ops = _ops()
    n, t, h, w, cin, cout, k, stride, pad = case
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(n, t, h, w, cin, generator=g).to(dev)
    wt = (torch.randn(cout, cin, *k, generator=g) / (cin * k[0] * k[1] * k[2]) ** 0.5).to(dev)
    xp = make_planes(x, nsplit)
    geom = ops.fprop_geom(xp, k, stride, pad)
    return x, wt, xp, geom


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fprop(case, nsplit, cuda_device):
    ops = _ops()
    n, t, h, w, cin, cout, k, stride, pad = case
    x, wt, xp, geom = _conv_setup(case, nsplit, cuda_device)
    f = ops.alloc_filter(cout, k[0] * k[1] * k[2], cin, nsplit, cuda_device)
    ops.filter_pack(wt, f)
    ot, oh, ow = geom.out
    y = torch.empty(n, ot, oh, ow, cout, device=cuda_device)
    stats = torch.zeros(2, cout, ops.conv_m_tiles(n, geom), device=cuda_device)
    ops.conv_igemm(xp, f, geom, y, (ot * oh * ow * cout, oh * ow * cout, ow * cout, cout), stats=stats, nsplit=nsplit)
    xr = planes_value(xp, nsplit)
    wr = (f.hi.double() + (f.lo.double() if nsplit == 3 else 0)).reshape(cout, -1, f.cols_pad)[:, :, :cin]
    wr = wr.reshape(cout, *k, cin).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(xr.permute(0, 4, 1, 2, 3), wr, stride=stride, padding=pad).permute(0, 2, 3, 4, 1)
    assert relerr(y, ref) < TOL[nsplit]
    rs = ref.reshape(-1, cout)
    assert relerr(stats[0].double().sum(1), rs.sum(0)) < 1e-4
    assert relerr(stats[1].double().sum(1), (rs * rs).sum(0)) < 1e-4
    # the filter packer itself: hi+lo reproduces the fp32 weights to 2^-16
    if nsplit == 3:
        assert relerr(wr, wt.double()) < 3e-5


ACC_CASES = [
    # n, t, h, w, cin, cout, k, stride, pad   (both epilogue variants of the wgmma kernel, and the SIMT body)
    (2, 4, 14, 14, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0)),     # short K: line-coalesced epilogue
    (1, 2, 14, 14, 256, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1)),     # K = 2304: direct per-row stores
    (2, 4, 28, 28, 8, 32, (1, 1, 1), (1, 1, 1), (0, 0, 0)),       # C_in = 8: fp32 SIMT body
    (1, 4, 10, 12, 64, 24, (3, 1, 1), (1, 1, 1), (1, 0, 0)),      # ragged tile, N not a multiple of 32
]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("case", ACC_CASES)
def test_conv_accumulate_modes(case, mode, cuda_device):
    """accumulate = 1 (read-modify-write) and 2 (red.global.add: the second-consumer data gradients of the engine) add the
    convolution to what the destination holds; both equal prefill + the plain-store result bit for bit (one add per element)."""
    ops = _ops()
    n, t, h, w, cin, cout, k, stride, pad = case
    x, wt, xp, geom = _conv_setup(case, 3, cuda_device)
    f = ops.alloc_filter(cout, k[0] * k[1] * k[2], cin, 3, cuda_device)
    ops.filter_pack(wt, f)
    ot, oh, ow = geom.out
    strides = (ot * oh * ow * cout, oh * ow * cout, ow * cout, cout)
    plain = torch.empty(n, ot, oh, ow, cout, device=cuda_device)
    ops.conv_igemm(xp, f, geom, plain, strides, nsplit=3)
    pre = torch.randn(n, ot, oh, ow, cout, device=cuda_device)
    y = pre.clone()
    ops.conv_igemm(xp, f, geom, y, strides, accumulate=mode, nsplit=3)
    assert torch.equal(y, pre + plain)


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_dgrad(case, nsplit, cuda_device):
    """dgrad through the fprop kernel + strided sub-problem plan == autograd's input gradient."""
    ops = _ops()
    from slowfast_b200.conv_plan import dgrad_out_view, dgrad_plan
    n, t, h, w, cin, cout, k, stride, pad = case
    x, wt, xp, geom = _conv_setup(case, nsplit, cuda_device)
    ot, oh, ow = geom.out
    g = torch.Generator(device="cpu").manual_seed(7)
    dy = torch.randn(n, ot, oh, ow, cout, generator=g).to(cuda_device)
    dyp = make_planes(dy, nsplit)
    plan = dgrad_plan((t, h, w), k, stride, pad)
    dx = torch.full((n, t, h, w, cin), float("nan"), device=cuda_device)
    if plan.needs_zero_fill:
        dx.zero_()
    wsum = None
    for sub in plan.subs:
        f = ops.alloc_filter(cin, len(sub.tapmap), cout, nsplit, cuda_device)
        ops.filter_pack(wt, f, tapmap=sub.tapmap, transpose=True)
        off, strides = dgrad_out_view((t, h, w), stride, sub, cin)
        ops.conv_igemm(dyp, f, ops.ConvGeom(sub.k, (1, 1, 1), sub.low, sub.out), dx, strides, out_offset=off,
                       nsplit=nsplit)
    # reference on the operands the kernel saw
    wr = wt.bfloat16()
    wr = wr.double() + ((wt - wr.float()).bfloat16().double() if nsplit == 3 else 0)
    xin = torch.zeros(n, cin, t, h, w, dtype=torch.float64, device=cuda_device, requires_grad=True)
    yy = F.conv3d(xin, wr, stride=stride, padding=pad)
    (ref,) = torch.autograd.grad(yy, xin, planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert not torch.isnan(dx).any()
    assert relerr(dx, ref.permute(0, 2, 3, 4, 1)) < TOL[nsplit]


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_wgrad(case, nsplit, cuda_device):
    ops = _ops()
    n, t, h, w, cin, cout, k, stride, pad = case
    x, wt, xp, geom = _conv_setup(case, nsplit, cuda_device)
    ot, oh, ow = geom.out
    g = torch.Generator(device="cpu").manual_seed(11)
    dy = torch.randn(n, ot, oh, ow, cout, generator=g).to(cuda_device)
    dyp = make_planes(dy, nsplit)
    taps = k[0] * k[1] * k[2]
    dwm = torch.zeros(cout, taps * cin, device=cuda_device)
    ops.conv_wgrad(xp, dyp, geom, dwm, nsplit=nsplit)
    dw = torch.empty(cout, cin, *k, device=cuda_device)
    ops.filter_unpack_grad(dwm, dw, cin, accumulate=False)
    wref = torch.zeros(cout, cin, *k, dtype=torch.float64, device=cuda_device, requires_grad=True)
    yy = F.conv3d(planes_value(xp, nsplit).permute(0, 4, 1, 2, 3), wref, stride=stride, padding=pad)
    (ref,) = torch.autograd.grad(yy, wref, planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert relerr(dw, ref) < TOL[nsplit] * 2


WGRAD_DIRECT_CASES = [
    # n, t, h, w, cin, cout, k, stride, pad   (>= 32768 output positions, cin*cout <= 512: the fast pathway's narrow layers)
    (2, 8, 56, 56, 8, 8, (1, 3, 3), (1, 1, 1), (0, 1, 1)),      # res2 conv b
    (2, 8, 56, 56, 8, 32, (1, 1, 1), (1, 1, 1), (0, 0, 0)),     # res2 conv c / shortcut
    (2, 8, 56, 56, 32, 8, (3, 1, 1), (1, 1, 1), (1, 0, 0)),     # res2 conv a (temporal)
    (6, 8, 56, 56, 16, 16, (1, 3, 3), (1, 2, 2), (0, 1, 1)),    # res3 conv b of the first block: tensor-core path (both modes)
    (3, 8, 58, 54, 16, 16, (1, 3, 3), (1, 1, 1), (0, 1, 1)),    # ragged rows / partial chunks
    (6, 32, 28, 28, 8, 16, (7, 1, 1), (4, 1, 1), (3, 0, 0)),    # FuseFastToSlow conv_f2s (temporal stride 4, 14 jobs)
    (6, 8, 56, 56, 8, 8, (1, 3, 3), (1, 2, 2), (0, 1, 1)),      # spatial stride 2 on the direct path
]


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", WGRAD_DIRECT_CASES)
def test_conv_wgrad_direct_narrow_layers(case, nsplit, cuda_device):
    """fp32 SIMT weight gradient of the narrow layers (csrc/conv_wgrad_direct.cu, taken inside sfb_conv_wgrad) vs torch
    autograd in fp64, and against the tensor-core kernel on the same operands."""
    from slowfast_b200 import lib as L
    ops = _ops()
    n, t, h, w, cin, cout, k, stride, pad = case
    x, wt, xp, geom = _conv_setup(case, nsplit, cuda_device)
    ot, oh, ow = geom.out
    g = torch.Generator(device="cpu").manual_seed(13)
    dy = torch.randn(n, ot, oh, ow, cout, generator=g).to(cuda_device)
    dyp = make_planes(dy, nsplit)
    taps = k[0] * k[1] * k[2]
    res = {}
    try:
        for mode in (1, 0):
            L.load().sfb_set_wgrad_direct(mode)
            dwm = torch.zeros(cout, taps * cin, device=cuda_device)
            ops.conv_wgrad(xp, dyp, geom, dwm, nsplit=nsplit)
            dw = torch.empty(cout, cin, *k, device=cuda_device)
            ops.filter_unpack_grad(dwm, dw, cin, accumulate=False)
            res[mode] = dw
    finally:
        L.load().sfb_set_wgrad_direct(1)
    wref = torch.zeros(cout, cin, *k, dtype=torch.float64, device=cuda_device, requires_grad=True)
    yy = F.conv3d(planes_value(xp, nsplit).permute(0, 4, 1, 2, 3), wref, stride=stride, padding=pad)
    (ref,) = torch.autograd.grad(yy, wref, planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert relerr(res[1], ref) < 5e-5      # exact fp32 products of the operands as stored, fp32 accumulation
    assert relerr(res[0], ref) < TOL[nsplit] * 2
    assert relerr(res[1], res[0]) < TOL[nsplit] * 2


def test_input_pack(cuda_device):
    ops = _ops()
    x = torch.randn(2, 3, 4, 10, 12, device=cuda_device)
    p = ops.alloc_planes(2, 4, 10, 12, 8, 3, cuda_device)
    ops.input_pack(x, p)
    v = p.to_float()
    assert relerr(v[..., :3], x.permute(0, 2, 3, 4, 1)) < 2e-5
    assert (v[..., 3:] == 0).all()


@pytest.mark.parametrize("c,rows_shape", [(64, (2, 4, 14, 14)), (8, (2, 8, 9, 9)), (256, (1, 2, 7, 7))])
def test_bn_forward_backward(c, rows_shape, cuda_device):
    """conv-epilogue partials -> finalize -> apply(+residual, ReLU) and the full backward, vs torch batch_norm."""
    ops = _ops()
    dev = cuda_device
    n, t, h, w = rows_shape
    rows = n * t * h * w
    g = torch.Generator(device="cpu").manual_seed(3)
    y = (torch.randn(n, t, h, w, c, generator=g) * 1.7 + 0.3).to(dev)
    res = torch.randn(n, t, h, w, c, generator=g).to(dev)
    gamma = (torch.rand(c, generator=g) + 0.5).to(dev)
    beta = torch.randn(c, generator=g).to(dev)
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    # partials exactly as the conv epilogue lays them out: per 128-row tile (sum, sumsq)
    m_tiles = (rows + 127) // 128
    yr = F.pad(y.reshape(rows, c), (0, 0, 0, m_tiles * 128 - rows)).reshape(m_tiles, 128, c)
    partials = torch.stack([yr.sum(1).t(), (yr * yr).sum(1).t()], 0).contiguous()  # [2][c][m_tiles]
    scale, shift, mean, invstd = (torch.empty(c, device=dev) for _ in range(4))
    ops.bn_finalize(partials, m_tiles, c, rows, gamma, beta, rm, rv, 0.1, 1e-5, True, scale, shift, mean, invstd)
    resp = make_planes(res, 3)
    out = ops.alloc_planes(n, t, h, w, c, 3, dev)
    ops.bn_apply(ops.f32view(y), scale, shift, out, relu=True, res=resp)

    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm_ref, rv_ref = torch.zeros(c, device=dev, dtype=torch.float64), torch.ones(c, device=dev, dtype=torch.float64)
    bn = F.batch_norm(y64.permute(0, 4, 1, 2, 3), rm_ref, rv_ref, g64, b64, True, 0.1, 1e-5).permute(0, 2, 3, 4, 1)
    ref = torch.relu(bn + resp.to_float().double())
    assert relerr(out.to_float(), ref) < 2e-5
    assert relerr(rm, rm_ref) < 1e-5 and relerr(rv, rv_ref) < 1e-5

    dout = torch.randn(n, t, h, w, c, generator=g).to(dev)
    dgamma, dbeta = torch.empty(c, device=dev), torch.empty(c, device=dev)
    dy = ops.alloc_planes(n, t, h, w, c, 3, dev)
    dres = torch.empty(n, t, h, w, c, device=dev)
    partials_b, coef = ops.bn_bwd_scratch(rows, c, dev)
    ops.bn_bwd(ops.f32view(dout), out, ops.f32view(y), mean, invstd, gamma, dgamma, dbeta, dy, partials_b, coef,
               dres=ops.f32view(dres))
    # torch reference: mask defined by OUR forward output (identical up to rounding at exact zeros)
    mask = (out.hi.float() > 0).double()
    dz = dout.double() * mask
    gy, gg, gb = torch.autograd.grad(bn, (y64, g64, b64), dz)
    assert relerr(dy.to_float(), gy) < 3e-5
    assert relerr(dgamma, gg) < 1e-5 and relerr(dbeta, gb) < 1e-5
    assert relerr(dres, dz) < 1e-6


def test_bn_two_branch_and_eval(cuda_device):
    ops = _ops()
    dev = cuda_device
    c, shp = 32, (2, 2, 6, 6)
    rows = shp[0] * shp[1] * shp[2] * shp[3]
    y1, y2 = torch.randn(*shp, c, device=dev), torch.randn(*shp, c, device=dev)
    s1, b1, s2, b2 = (torch.randn(c, device=dev) for _ in range(4))
    out = ops.alloc_planes(*shp, c, 3, dev, pitch=c + 16).slice(0, c)
    out = ops.Planes(out.hi, out.lo, *shp, c, 16)  # write at channel offset 16 of a 48-wide tensor
    out.hi.zero_(); out.lo.zero_()
    ops.bn_apply(ops.f32view(y1), s1, b1, out, relu=True, y2=ops.f32view(y2), scale2=s2, shift2=b2)
    ref = torch.relu(y1.double() * s1.double() + b1.double() + y2.double() * s2.double() + b2.double())
    assert relerr(out.to_float(), ref) < 2e-5
    assert (out.hi[..., :16] == 0).all()
    # eval-mode finalize uses the running statistics
    rm, rv = torch.randn(c, device=dev), torch.rand(c, device=dev) + 0.5
    gamma, beta = torch.randn(c, device=dev), torch.randn(c, device=dev)
    scale, shift = torch.empty(c, device=dev), torch.empty(c, device=dev)
    ops.bn_finalize(None, 0, c, rows, gamma, beta, rm, rv, 0.1, 1e-5, False, scale, shift, None, None)
    inv = 1.0 / torch.sqrt(rv.double() + 1e-5)
    assert relerr(scale, gamma.double() * inv) < 1e-6
    assert relerr(shift, beta.double() - rm.double() * gamma.double() * inv) < 1e-6


@pytest.mark.parametrize("c", [8, 64])
def test_bn_relu_maxpool(c, cuda_device):
    ops = _ops()
    dev = cuda_device
    n, t, h, w = 2, 3, 14, 14
    y = torch.randn(n, t, h, w, c, device=dev)
    scale, shift = torch.randn(c, device=dev), torch.randn(c, device=dev) * 0.3
    k, s, p = (3, 3), (2, 2), (1, 1)
    oh, ow = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
    out = ops.alloc_planes(n, t, oh, ow, c, 3, dev)
    argmax = torch.empty(n, t, oh, ow, c, dtype=torch.uint8, device=dev)
    ops.bn_relu_maxpool_fwd(y, scale, shift, out, argmax, k, s, p)
    z = torch.relu(y * scale + shift).requires_grad_(True)  # fp32, same arithmetic as the kernel (fma vs mul+add)
    ref = F.max_pool3d(z.permute(0, 4, 1, 2, 3), (1, 3, 3), (1, 2, 2), (0, 1, 1)).permute(0, 2, 3, 4, 1)
    assert relerr(out.to_float(), ref.detach()) < 2e-5
    dout = torch.randn(n, t, oh, ow, c, device=dev)
    dz = torch.empty(n, t, h, w, c, device=dev)
    ops.bn_relu_maxpool_bwd(ops.f32view(dout), argmax, dz, oh, ow, k, s, p)
    (gz,) = torch.autograd.grad(ref, z, dout)
    gz = gz * (z > 0)  # our dz is the gradient w.r.t. the ReLU output restricted to where it survives the ReLU
    assert relerr(dz, gz) < 1e-6


STEM_CASES = [
    # n, t, h, w, cin, cout, k, stride, pad
    (2, 4, 16, 32, 3, 64, (1, 7, 7), (1, 2, 2), (0, 3, 3)),     # slow-pathway / C2D stem
    (1, 6, 20, 48, 3, 8, (5, 7, 7), (1, 2, 2), (2, 3, 3)),      # fast-pathway stem
    (1, 2, 12, 300, 3, 24, (1, 3, 3), (1, 2, 2), (0, 1, 1)),    # X3D conv_xy, output row (150) > one 128-pixel tile
]


STEM8_CASES = [
    # n, t, h, w, kt   (3 -> 8 channels, [kt,7,7], stride (1,2,2), pad (kt//2,3,3))
    (1, 6, 32, 64, 5),       # 5 granule rows per array, 2 bands
    (2, 3, 16, 48, 5),       # one band, output frames fewer than T taps at the clip ends
    (1, 4, 48, 32, 1),       # kt = 1
    (1, 8, 224, 224, 5),     # the fast pathway's extent: 15 granule rows, 14 bands
]


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", STEM8_CASES)
def test_stem8_toeplitz_fprop_wgrad(case, nsplit, cuda_device):
    """Toeplitz stem kernels (8 output pixels per GEMM row, csrc/conv_stem8.cu) vs torch conv3d / autograd in fp64."""
    ops = _ops()
    dev = cuda_device
    n, t, h, w, kt = case
    cin, cout, k, stride, pad = 3, 8, (kt, 7, 7), (1, 2, 2), (kt // 2, 3, 3)
    g = torch.Generator(device="cpu").manual_seed(11)
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
    m_tiles = ops.stem8_m_tiles(xp, geo)
    assert m_tiles == n * ot * (oh // 8)
    stats = torch.zeros(2, cout, m_tiles, device=dev)
    ops.stem8_fprop(xp, zh, zl, geo, y, stats, nsplit=nsplit)

    def rnd(v):
        hi = v.bfloat16()
        return hi.double() + ((v - hi.float()).bfloat16().double() if nsplit == 3 else 0)
    xr, wr = rnd(x), rnd(wt)
    ref = F.conv3d(xr, wr, stride=stride, padding=pad).permute(0, 2, 3, 4, 1)
    assert not torch.isnan(y).any()
    assert relerr(y, ref) < TOL[nsplit]
    rs = ref.reshape(-1, cout)
    assert relerr(stats[0].double().sum(1), rs.sum(0)) < 1e-4
    assert relerr(stats[1].double().sum(1), (rs * rs).sum(0)) < 1e-4
    # wgrad
    dy = torch.randn(n, ot, oh, ow, cout, generator=g).to(dev)
    dyp = make_planes(dy, nsplit)
    dwm = torch.zeros(cout, geo.kfold, device=dev)
    ops.stem8_wgrad(xp, dyp, geo, dwm, nsplit=nsplit)
    dw = torch.zeros(cout, cin, *k, device=dev)
    ops.stem_filter_unfold_grad(dwm, dw, geo)
    wref = torch.zeros(cout, cin, *k, dtype=torch.float64, device=dev, requires_grad=True)
    (gref,) = torch.autograd.grad(F.conv3d(xr, wref, stride=stride, padding=pad), wref,
                                  planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert relerr(dw, gref) < TOL[nsplit] * 2


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case", STEM_CASES)
def test_stem_wshift_fprop_wgrad(case, nsplit, cuda_device):
    """W-shift stem kernels (folded clip, shifted UMMA descriptors) vs torch conv3d / autograd wgrad in fp64."""
    ops = _ops()
    dev = cuda_device
    n, t, h, w, cin, cout, k, stride, pad = case
    g = torch.Generator(device="cpu").manual_seed(5)
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
    m_tiles = ops.stem_m_tiles(xp, geo)
    stats = torch.zeros(2, cout, m_tiles, device=dev)
    ops.stem_fprop(xp, f, geo, y, stats, nsplit=nsplit)
    # operands as the kernel saw them
    def rnd(v):
        hi = v.bfloat16()
        return hi.double() + ((v - hi.float()).bfloat16().double() if nsplit == 3 else 0)
    xr, wr = rnd(x), rnd(wt)
    ref = F.conv3d(xr, wr, stride=stride, padding=pad).permute(0, 2, 3, 4, 1)
    assert not torch.isnan(y).any()
    assert relerr(y, ref) < TOL[nsplit]
    rs = ref.reshape(-1, cout)
    assert relerr(stats[0].double().sum(1), rs.sum(0)) < 1e-4
    assert relerr(stats[1].double().sum(1), (rs * rs).sum(0)) < 1e-4
    # wgrad
    dy = torch.randn(n, ot, oh, ow, cout, generator=g).to(dev)
    dyp = make_planes(dy, nsplit)
    dwm = torch.zeros(cout, geo.kfold, device=dev)
    ops.stem_wgrad(xp, dyp, geo, dwm, nsplit=nsplit)
    dw = torch.zeros(cout, cin, *k, device=dev)
    ops.stem_filter_unfold_grad(dwm, dw, geo)
    wref = torch.zeros(cout, cin, *k, dtype=torch.float64, device=dev, requires_grad=True)
    (gref,) = torch.autograd.grad(F.conv3d(xr, wref, stride=stride, padding=pad), wref,
                                  planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert relerr(dw, gref) < TOL[nsplit] * 2


def test_gemm_batched_all_layouts(cuda_device):
    """Batched wgmma GEMM in the four operand-major combinations the attention products need."""
    ops = _ops()
    from slowfast_b200 import lib as L
    import ctypes as C
    dev = cuda_device
    lib = L.load()
    g = torch.Generator(device="cpu").manual_seed(2)
    for nsplit in (1, 3):
        for (bt, m, n, k, a_mn, b_mn) in [(3, 200, 96, 96, 0, 0), (2, 300, 96, 393, 0, 1), (2, 393, 96, 300, 1, 1),
                                          (3, 130, 200, 96, 0, 0), (2, 96, 40, 520, 1, 1),
                                          # long reductions over few tiles: the split-K path (float atomics into the zeroed output)
                                          (2, 393, 96, 4100, 1, 1), (1, 100, 96, 2500, 0, 0), (2, 200, 96, 3000, 0, 1)]:
            kp, mp, np_ = (k + 7) // 8 * 8, (m + 7) // 8 * 8, (n + 7) // 8 * 8
            A = torch.randn(bt, m, k, generator=g).to(dev)
            Bm = torch.randn(bt, n, k, generator=g).to(dev)
            # storage in the requested major-ness, pitches padded to 8
            a_st = torch.zeros(bt, k, mp, device=dev) if a_mn else torch.zeros(bt, m, kp, device=dev)
            b_st = torch.zeros(bt, k, np_, device=dev) if b_mn else torch.zeros(bt, n, kp, device=dev)
            if a_mn:
                a_st[:, :, :m] = A.transpose(1, 2)
            else:
                a_st[:, :, :k] = A
            if b_mn:
                b_st[:, :, :n] = Bm.transpose(1, 2)
            else:
                b_st[:, :, :k] = Bm
            def split(v):
                hi = v.bfloat16()
                return hi, (v - hi.float()).bfloat16()
            a_hi, a_lo = split(a_st)
            b_hi, b_lo = split(b_st)
            out = torch.full((bt, m, n), float("nan"), device=dev)
            d = L.BgemmDesc()
            d.a_hi, d.a_lo, d.lda, d.batch_stride_a, d.a_mn_major = a_hi.data_ptr(), a_lo.data_ptr(), a_st.shape[2], a_st[0].numel(), a_mn
            d.b_hi, d.b_lo, d.ldb, d.batch_stride_b, d.b_mn_major = b_hi.data_ptr(), b_lo.data_ptr(), b_st.shape[2], b_st[0].numel(), b_mn
            d.m, d.n, d.k, d.batch = m, n, k, bt
            d.out, d.ldd, d.batch_stride_d = out.data_ptr(), n, m * n
            d.alpha, d.accumulate, d.nsplit = 0.5, 0, nsplit
            L.check(lib.sfb_gemm_batched(C.byref(d), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "bgemm")
            def val(hi, lo):
                return hi.double() + (lo.double() if nsplit == 3 else 0)
            Ar = val(a_hi, a_lo)
            Br = val(b_hi, b_lo)
            Ar = Ar[:, :, :m].transpose(1, 2) if a_mn else Ar[:, :, :k]
            Br = Br[:, :, :n].transpose(1, 2) if b_mn else Br[:, :, :k]
            ref = 0.5 * Ar @ Br.transpose(1, 2)
            assert not torch.isnan(out).any(), (nsplit, bt, m, n, k, a_mn, b_mn)
            assert relerr(out, ref) < TOL[nsplit], (nsplit, bt, m, n, k, a_mn, b_mn, relerr(out, ref))


@pytest.mark.parametrize("k,s,p", [((2, 1, 1), (2, 1, 1), (0, 0, 0)), ((1, 3, 3), (1, 2, 2), (0, 1, 1)),
                                   ((3, 3, 3), (2, 2, 2), (1, 1, 1))])
def test_maxpool3d_planes(k, s, p, cuda_device):
    ops = _ops()
    dev = cuda_device
    n, t, h, w, c = 2, 6, 10, 12, 16
    x = torch.randn(n, t, h, w, c, device=dev)
    xp = make_planes(x, 3)
    xv = xp.to_float().clone().requires_grad_(True)
    ref = F.max_pool3d(xv.permute(0, 4, 1, 2, 3), k, s, p).permute(0, 2, 3, 4, 1)
    ot, oh, ow = ref.shape[1:4]
    out = ops.alloc_planes(n, ot, oh, ow, c, 3, dev)
    argmax = torch.empty(n, ot, oh, ow, c, dtype=torch.uint8, device=dev)
    ops.maxpool3d_fwd(xp, out, argmax, k, s, p)
    assert torch.equal(out.to_float(), ref.detach())  # values are exactly representable: bit-exact
    dout = torch.randn(n, ot, oh, ow, c, device=dev)
    din = torch.full((n, t, h, w, c), float("nan"), device=dev)
    ops.maxpool3d_bwd(ops.f32view(dout), argmax, xp, (ot, oh, ow), ops.f32view(din), k, s, p)
    (g,) = torch.autograd.grad(ref, xv, dout)
    assert relerr(din, g) < 1e-6


# ------------------------------------------------------------------------------------------------ X3D kernels
DW_CASES = [
    # n, t, h, w, c_valid, k, stride, pad, input format
    (2, 4, 14, 14, 54, (3, 3, 3), (1, 1, 1), (1, 1, 1), "planes"),
    (2, 4, 14, 14, 54, (3, 3, 3), (1, 2, 2), (1, 1, 1), "planes"),
    (3, 4, 9, 9, 216, (3, 3, 3), (1, 2, 2), (1, 1, 1), "planes"),
    (1, 3, 7, 7, 432, (3, 3, 3), (1, 1, 1), (1, 1, 1), "planes"),
    (2, 6, 12, 12, 24, (5, 1, 1), (1, 1, 1), (2, 0, 0), "f32"),
    (2, 5, 13, 15, 54, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32"),
    (2, 4, 14, 18, 108, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f32"),
    (1, 3, 7, 7, 432, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32+affine"),
    (2, 3, 10, 10, 216, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f32+affine"),
    # shared-memory ring kernels (x3d_ops.cu "v3": stride 1, pad 1, H and W multiples of 7): 14x14 and 7x7 tiles, partial
    # last channel slab (56 = 32 + 24 lanes), several tiles per sample, the minimum of two frames
    (2, 4, 14, 14, 54, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32"),
    (2, 3, 28, 14, 108, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32+affine"),
    (1, 2, 7, 21, 24, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32"),
    (2, 5, 14, 28, 216, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32+affine"),
    (1, 2, 14, 14, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), "f32"),
    # ring kernels at spatial stride 2 (7x7 output tiles over 15x15 input tiles): forward + weight gradient
    (2, 4, 14, 14, 54, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f32"),
    (1, 3, 28, 14, 108, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f32+affine"),
    (2, 2, 56, 28, 24, (3, 3, 3), (1, 2, 2), (1, 1, 1), "f32"),
]


@pytest.mark.parametrize("case", DW_CASES)
def test_dwconv_forward_backward(case, cuda_device):
    """Channelwise Conv3d (X3DTransform.b / X3DStem.conv): y, BN partial sums, dx (fp32 and planes) and dw against
    torch's grouped conv in fp64 on the operands the kernel saw; pad channels (54 -> 56) stay exactly zero."""
    ops = _ops()
    n, t, h, w, c, k, stride, pad, fmt = case
    dev = cuda_device
    cp = ops.pad8(c)
    g = torch.Generator().manual_seed(5)
    x = torch.zeros(n, t, h, w, cp)
    x[..., :c] = torch.randn(n, t, h, w, c, generator=g)
    x = x.to(dev)
    wt = (torch.randn(c, 1, *k, generator=g) / (k[0] * k[1] * k[2]) ** 0.5).to(dev)
    geom = ops.DwGeom(n, t, h, w, k, stride, pad)
    ot, oh, ow = geom.out
    if fmt == "planes":
        xp = make_planes(x, 3)
        xin = dict(x_planes=xp)
        xv = planes_value(xp, 3)
    elif fmt == "f32":
        xin = dict(x_f32=ops.f32view(x))
        xv = x.double()
    else:  # producer BatchNorm + ReLU applied on the fly (pad channels: scale = shift = 0)
        sc = torch.zeros(cp, device=dev)
        sh = torch.zeros(cp, device=dev)
        sc[:c] = torch.rand(c, generator=g).to(dev) + 0.5
        sh[:c] = torch.randn(c, generator=g).to(dev) * 0.5
        xin = dict(x_f32=ops.f32view(x), in_affine=(sc, sh, True))
        xv = torch.relu(torch.addcmul(sh, x, sc)).double()
    y = torch.full((n, ot, oh, ow, cp), float("nan"), device=dev)
    m_tiles, tps = ops.dwconv_tiles(geom, cp, fmt != "planes")
    stats = torch.zeros(2, c, m_tiles, device=dev)
    ops.dwconv_fwd(geom, cp, c, wt, ops.f32view(y), stats, **xin)
    ref = F.conv3d(xv[..., :c].permute(0, 4, 1, 2, 3), wt.double(), None, stride, pad, 1, c).permute(0, 2, 3, 4, 1)
    assert relerr(y[..., :c], ref) < 1e-5
    assert (y[..., c:] == 0).all()
    assert relerr(stats[0].sum(1), ref.sum((0, 1, 2, 3))) < 1e-4 or ref.sum((0, 1, 2, 3)).abs().max() < 1e-3
    assert relerr(stats[1].sum(1), (ref * ref).sum((0, 1, 2, 3))) < 1e-5
    # per-sample tiles: sample s owns tiles [s*tps, (s+1)*tps)
    per_sample = stats[0].view(c, n, tps).sum(2).t()
    assert relerr(per_sample, ref.sum((1, 2, 3))) < 1e-4
    # backward
    dy = torch.zeros(n, ot, oh, ow, cp)
    dy[..., :c] = torch.randn(n, ot, oh, ow, c, generator=g)
    dy = dy.to(dev)
    xr = xv[..., :c].permute(0, 4, 1, 2, 3).clone().requires_grad_(True)
    wr = wt.double().clone().requires_grad_(True)
    F.conv3d(xr, wr, None, stride, pad, 1, c).backward(dy[..., :c].double().permute(0, 4, 1, 2, 3))
    dx = torch.full((n, t, h, w, cp), float("nan"), device=dev)
    dw = torch.empty_like(wt)
    wp = torch.empty(ops.dwconv_wgrad_blocks(geom) * cp * wt[0].numel(), device=dev)
    ops.dwconv_bwd(geom, cp, c, wt, ops.f32view(dy), dw, wp, dx=ops.f32view(dx), **xin)
    assert relerr(dx[..., :c], xr.grad.permute(0, 2, 3, 4, 1)) < 1e-5
    assert (dx[..., c:] == 0).all()
    assert relerr(dw, wr.grad) < 2e-5
    if stride == (1, 1, 1) or fmt == "planes":  # (the stride-2 register-tiled data gradient is fp32-output only)
        dxp = ops.alloc_planes(n, t, h, w, cp, 3, dev)
        ops.dwconv_bwd(geom, cp, c, wt, ops.f32view(dy), None, None, dx_planes=dxp, **xin)
        assert relerr(dxp.to_float()[..., :c], xr.grad.permute(0, 2, 3, 4, 1)) < 2e-5
    # accumulate form
    base = torch.randn(n, t, h, w, cp, generator=g).to(dev)
    acc = base.clone()
    ops.dwconv_bwd(geom, cp, c, wt, ops.f32view(dy), None, None, dx=ops.f32view(acc), dx_accumulate=True, **xin)
    assert relerr((acc - base)[..., :c], xr.grad.permute(0, 2, 3, 4, 1)) < 1e-4


@pytest.mark.parametrize("c,f,use_se,act,training", [(54, 8, True, "swish", True), (432, 32, True, "swish", True),
                                                     (216, 16, False, "swish", True), (24, 0, False, "relu", True),
                                                     (108, 8, True, "swish", False)])
def test_bn_se_act_forward_backward(c, f, use_se, act, training, cuda_device):
    """out = act(BN(y) * SE(BN(y))): forward planes and the full backward (dy, dgamma, dbeta, SE parameter gradients)
    against torch autograd in fp64; BN in train (batch statistics) and eval (running statistics) mode."""
    import ctypes as C
    from slowfast_b200 import lib as L
    ops = _ops()
    dev = cuda_device
    n, t, h, w = 3, 2, 5, 6
    rps = t * h * w
    cp = ops.pad8(c)
    g = torch.Generator().manual_seed(c + f)
    y = torch.zeros(n, t, h, w, cp)
    y[..., :c] = torch.randn(n, t, h, w, c, generator=g) * 1.5 + 0.3
    gamma = torch.rand(c, generator=g) + 0.5
    beta = torch.randn(c, generator=g) * 0.3
    rm, rv = torch.randn(c, generator=g) * 0.1 + 0.3, torch.rand(c, generator=g) + 1.5
    w1 = torch.randn(max(f, 1), c, generator=g) / c ** 0.5
    b1 = torch.randn(max(f, 1), generator=g) * 0.1
    w2 = torch.randn(c, max(f, 1), generator=g) / max(f, 1) ** 0.5
    b2 = torch.randn(c, generator=g) * 0.1
    dout = torch.zeros(n, t, h, w, cp)
    dout[..., :c] = torch.randn(n, t, h, w, c, generator=g)

    # ---- fp64 reference through autograd
    leaves = [v.double().clone().requires_grad_(True) for v in (y[..., :c], gamma, beta, w1, b1, w2, b2)]
    yr, gr, br, w1r, b1r, w2r, b2r = leaves
    if training:
        mu, var = yr.mean((0, 1, 2, 3)), yr.var((0, 1, 2, 3), unbiased=False)
    else:
        mu, var = rm.double(), rv.double()
    z = (yr - mu) / torch.sqrt(var + 1e-5) * gr + br
    if use_se:
        avg = z.mean((1, 2, 3))
        gate = torch.sigmoid(F.relu(avg @ w1r.t() + b1r) @ w2r.t() + b2r)
        u = z * gate[:, None, None, None, :]
    else:
        u = z
    o = u * torch.sigmoid(u) if act == "swish" else F.relu(u)
    o.backward(dout[..., :c].double())

    # ---- kernels
    y_d, dout_d = y.to(dev), dout.to(dev)
    to = lambda v: v.to(dev).contiguous()
    gamma_d, beta_d, rm_d, rv_d, w1_d, b1_d, w2_d, b2_d = map(to, (gamma, beta, rm, rv, w1, b1, w2, b2))
    # per-sample-tile partial sums exactly as the channelwise conv's epilogue would emit them
    tps = 2
    m_tiles = n * tps
    ys = y_d.view(n, rps, cp)[..., :c]
    half = rps // 2
    stats = torch.zeros(2, c, m_tiles, device=dev)
    for s in range(n):
        for j, sl in enumerate((slice(0, half), slice(half, rps))):
            stats[0, :, s * tps + j] = ys[s, sl].sum(0)
            stats[1, :, s * tps + j] = (ys[s, sl] ** 2).sum(0)
    bb = {k: torch.zeros(cp, device=dev) for k in ("scale", "shift", "mean", "invstd")}
    ops.bn_finalize(stats, m_tiles, c, n * rps, gamma_d, beta_d, rm_d, rv_d, 0.1, 1e-5, training, bb["scale"],
                    bb["shift"], bb["mean"], bb["invstd"])
    act_id = ops.ACT_SWISH if act == "swish" else ops.ACT_RELU
    d = L.SeDesc()
    gate_d = None
    sv = {}
    if use_se:
        d.n, d.c, d.c_pad, d.f, d.rows_per_sample, d.tiles_per_sample, d.m_tiles = n, c, cp, f, rps, tps, m_tiles
        d.stats, d.scale, d.shift = stats.data_ptr(), bb["scale"].data_ptr(), bb["shift"].data_ptr()
        d.mean, d.invstd = bb["mean"].data_ptr(), bb["invstd"].data_ptr()
        d.w1, d.b1, d.w2, d.b2 = w1_d.data_ptr(), b1_d.data_ptr(), w2_d.data_ptr(), b2_d.data_ptr()
        sv = {k: torch.empty(n, cp, device=dev) for k in ("ymean", "avg", "gate")}
        sv["hid"] = torch.empty(n, f, device=dev)
        d.ymean, d.avg, d.hid, d.gate = (sv[k].data_ptr() for k in ("ymean", "avg", "hid", "gate"))
        ops.se_fwd(d)
        gate_d = sv["gate"]
        assert relerr(gate_d[:, :c].cpu(), gate.detach()) < 1e-5
        assert (gate_d[:, c:] == 0).all()
    out = ops.alloc_planes(n, t, h, w, cp, 3, dev)
    yv = ops.f32view(y_d)
    ops.bnact_fwd(yv, bb["scale"], bb["shift"], gate_d, act_id, rps, out)
    assert relerr(out.to_float()[..., :c].cpu(), o.detach()) < 2e-5
    assert (out.to_float()[..., c:] == 0).all()
    # backward
    tps2 = ops.bnact_tiles_per_sample(n * rps, rps)
    partials = torch.empty(n * tps2 * 2 * cp, device=dev)
    ops.bnact_bwd_reduce(yv, bb["scale"], bb["shift"], bb["mean"], bb["invstd"], gate_d, act_id, rps,
                         ops.f32view(dout_d), partials)
    d.n, d.c, d.c_pad, d.rows_per_sample = n, c, cp, rps
    d.mean, d.invstd = bb["mean"].data_ptr(), bb["invstd"].data_ptr()
    d.partials, d.tiles2_per_sample = partials.data_ptr(), tps2
    scratch = {k: torch.empty(n * 2 * cp, device=dev) for k in ("a12", "do2", "davg")}
    scratch["dhid"] = torch.empty(n * max(f, 1), device=dev)
    coef = torch.empty(3, cp, device=dev)
    d.a12, d.coef = scratch["a12"].data_ptr(), coef.data_ptr()
    d.gamma, d.beta = gamma_d.data_ptr(), beta_d.data_ptr()
    dgamma, dbeta = torch.empty(c, device=dev), torch.empty(c, device=dev)
    d.dgamma, d.dbeta = dgamma.data_ptr(), dbeta.data_ptr()
    d.training = 1 if training else 0
    gw = {k: torch.empty_like(v) for k, v in (("w1", w1_d), ("b1", b1_d), ("w2", w2_d), ("b2", b2_d))}
    davg = None
    if use_se:
        d.has_se = 1
        d.do2, d.dhid, d.davg = scratch["do2"].data_ptr(), scratch["dhid"].data_ptr(), scratch["davg"].data_ptr()
        d.dw1, d.db1, d.dw2, d.db2 = (gw[k].data_ptr() for k in ("w1", "b1", "w2", "b2"))
        davg = scratch["davg"]
    else:
        d.has_se, d.f = 0, 0
    ops.se_bwd(d)
    dy = torch.full((n * rps, cp), float("nan"), device=dev)
    ops.bnact_bwd_apply(yv, bb["scale"], bb["shift"], bb["mean"], bb["invstd"], gate_d, act_id, rps,
                        ops.f32view(dout_d), davg, coef, ops.f32view(dy))
    assert relerr(dy.view(n, t, h, w, cp)[..., :c].cpu(), yr.grad) < 5e-5
    assert (dy[:, c:] == 0).all()
    assert relerr(dgamma.cpu(), gr.grad) < 5e-5 and relerr(dbeta.cpu(), br.grad) < 5e-5
    if use_se:
        assert relerr(gw["w1"].cpu(), w1r.grad) < 5e-5 and relerr(gw["b1"].cpu(), b1r.grad) < 5e-5
        assert relerr(gw["w2"].cpu(), w2r.grad) < 5e-5 and relerr(gw["b2"].cpu(), b2r.grad) < 5e-5


def test_conv_padded_output_channels(cuda_device):
    """1x1x1 conv with 54 output channels written into a 56-wide tensor: pad columns are exact zeros, the BN
    partials cover the 54 real channels (ConvBN's cout_pad path used by X3D)."""
    ops = _ops()
    dev = cuda_device
    n, t, h, w, cin, cout = 2, 2, 9, 9, 24, 54
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, t, h, w, cin, generator=g).to(dev)
    wt = (torch.randn(cout, cin, 1, 1, 1, generator=g) / cin ** 0.5).to(dev)
    xp = make_planes(x, 3)
    geom = ops.fprop_geom(xp, (1, 1, 1), (1, 1, 1), (0, 0, 0))
    fm = ops.alloc_filter(cout, 1, cin, 3, dev)
    ops.filter_pack(wt, fm)
    cp = ops.pad8(cout)
    y = torch.full((n, t, h, w, cp), float("nan"), device=dev)
    m_tiles = ops.conv_m_tiles(n, geom)
    stats = torch.zeros(2, cout, m_tiles, device=dev)
    ops.conv_igemm(xp, fm, geom, y, (t * h * w * cp, h * w * cp, w * cp, cp), stats=stats, nsplit=3)
    ref = torch.einsum("nthwc,oc->nthwo", planes_value(xp, 3), wt.double().view(cout, cin))
    assert relerr(y[..., :cout], ref) < TOL[3]
    assert (y[..., cout:] == 0).all()
    assert relerr(stats[1].sum(1), (ref * ref).sum((0, 1, 2, 3))) < 1e-4


@pytest.mark.parametrize("shape", [(1, 6, 20, 48), (2, 9, 14, 64), (1, 32, 28, 224)])
def test_stem_wgrad_direct(shape, cuda_device):
    """fp32 SIMT weight gradient of the fast-pathway stem (3 -> 8, 5x7x7, stride (1,2,2)) vs torch autograd in fp64:
    exact fp32 inputs on the X side, the (hi+lo) planes on the dY side."""
    ops = _ops()
    dev = cuda_device
    n, t, h, w = shape
    k, stride, pad = (5, 7, 7), (1, 2, 2), (2, 3, 3)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, 3, t, h, w, generator=g).to(dev)
    ot, oh, ow = t, (h + 6 - 7) // 2 + 1, (w + 6 - 7) // 2 + 1
    dy = torch.randn(n, ot, oh, ow, 8, generator=g).to(dev)
    dyp = make_planes(dy, 3)
    dw = torch.full((8, 3, *k), float("nan"), device=dev)
    ops.stem_wgrad_direct(x, dyp, k, stride, pad, dw)
    wref = torch.zeros(8, 3, *k, dtype=torch.float64, device=dev, requires_grad=True)
    (gref,) = torch.autograd.grad(F.conv3d(x.double(), wref, stride=stride, padding=pad), wref,
                                  planes_value(dyp, 3).permute(0, 4, 1, 2, 3))
    assert relerr(dw, gref) < 1e-5
    # bf16 fast mode: no lo plane
    dyp1 = make_planes(dy, 1)
    ops.stem_wgrad_direct(x, dyp1, k, stride, pad, dw)
    (gref1,) = torch.autograd.grad(F.conv3d(x.double(), wref, stride=stride, padding=pad), wref,
                                   planes_value(dyp1, 1).permute(0, 4, 1, 2, 3))
    assert relerr(dw, gref1) < 1e-5
