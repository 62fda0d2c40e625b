"""GPU: every tile shape of the tensor-core weight gradient (co-rows and transposed orientations, 64- and 128-row tiles,
CK = 8 / 16 / 32 / 64 chunks, tiled and im2col X loads, split and unsplit reductions) against fp64 autograd on the
operands the kernel saw, accumulating into a non-zero dW.  The plan query pins which tiling each case takes."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernels import TOL, make_planes, planes_value, relerr

pytestmark = pytest.mark.gpu

CASES = [
    # n, t, h, w, cin, cout, k, stride, pad, (transposed, tile rows, BN, CK) at 132 SMs
    ((2, 4, 14, 14, 16, 16, (1, 3, 3), (1, 1, 1), (0, 1, 1)), (1, 64, 16, 16)),
    ((2, 8, 28, 28, 32, 16, (3, 1, 1), (1, 1, 1), (1, 0, 0)), (1, 64, 16, 32)),
    ((2, 8, 28, 28, 64, 16, (3, 3, 3), (1, 1, 1), (1, 1, 1)), (1, 128, 16, 64)),
    ((2, 8, 28, 28, 64, 32, (3, 1, 1), (1, 1, 1), (1, 0, 0)), (1, 64, 32, 64)),
    ((2, 4, 28, 28, 32, 32, (1, 3, 3), (1, 2, 2), (0, 1, 1)), (1, 64, 32, 32)),
    ((2, 4, 14, 14, 8, 24, (1, 3, 3), (1, 1, 1), (0, 1, 1)), (1, 64, 32, 8)),
    ((2, 8, 28, 28, 128, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1)), (1, 128, 32, 64)),
    ((2, 8, 14, 14, 128, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0)), (1, 64, 64, 64)),
    ((2, 8, 14, 14, 8, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1)), (1, 64, 64, 8)),
    ((2, 4, 14, 14, 64, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0)), (0, 64, 64, 64)),
    ((2, 4, 28, 28, 16, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0)), (0, 64, 16, 16)),
    ((2, 4, 14, 14, 32, 128, (1, 1, 1), (1, 1, 1), (0, 0, 0)), (0, 64, 32, 32)),
    ((2, 4, 14, 14, 24, 48, (1, 1, 1), (1, 1, 1), (0, 0, 0)), (0, 64, 32, 8)),
    ((2, 4, 14, 14, 48, 128, (1, 1, 1), (1, 1, 1), (0, 0, 0)), (0, 64, 48, 16)),
    ((1, 8, 28, 28, 32, 80, (1, 3, 3), (1, 1, 1), (0, 1, 1)), (0, 64, 96, 32)),
    ((2, 4, 14, 14, 40, 96, (3, 3, 3), (1, 1, 1), (1, 1, 1)), (0, 64, 128, 8)),
    ((2, 4, 14, 14, 256, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0)), (0, 64, 128, 64)),   # unsplit, strided
    ((1, 2, 7, 7, 512, 512, (1, 3, 3), (1, 1, 1), (0, 1, 1)), (0, 64, 128, 64)),     # unsplit, padded
    ((2, 8, 28, 28, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0)), (0, 64, 64, 64)),
    ((4, 8, 28, 28, 128, 128, (3, 3, 3), (1, 1, 1), (1, 1, 1)), (0, 128, 128, 64)),
]


@pytest.mark.parametrize("nsplit", [1, 3])
@pytest.mark.parametrize("case,tiling", CASES)
def test_wgrad_tile(case, tiling, nsplit, cuda_device):
    from slowfast_b200 import ops
    n, t, h, w, cin, cout, k, stride, pad = case
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(n, t, h, w, cin, generator=g).to(cuda_device)
    xp = make_planes(x, nsplit)
    geom = ops.fprop_geom(xp, k, stride, pad)
    dy = torch.randn(n, *geom.out, cout, generator=g).to(cuda_device)
    dyp = make_planes(dy, nsplit)
    plan = ops.conv_wgrad_plan(xp, dyp, geom, nsplit=nsplit, num_sms=132)
    assert not plan.direct and (plan.transposed, plan.tile_rows, plan.bn, plan.ck) == tiling
    taps = k[0] * k[1] * k[2]
    pre = torch.randn(cout, taps * cin, generator=g).to(cuda_device)
    dwm = pre.clone()
    ops.conv_wgrad(xp, dyp, geom, dwm, nsplit=nsplit)
    dw = torch.empty(cout, cin, *k, device=cuda_device)
    ops.filter_unpack_grad(dwm - pre, dw, cin, accumulate=False)
    wref = torch.zeros(cout, cin, *k, dtype=torch.float64, device=cuda_device, requires_grad=True)
    yy = F.conv3d(planes_value(xp, nsplit).permute(0, 4, 1, 2, 3), wref, stride=stride, padding=pad)
    (ref,) = torch.autograd.grad(yy, wref, planes_value(dyp, nsplit).permute(0, 4, 1, 2, 3))
    assert relerr(dw, ref) < TOL[nsplit] * 2
