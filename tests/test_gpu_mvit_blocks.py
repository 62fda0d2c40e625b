"""GPU: short MViT stacks of every block kind through the engine in parity mode, against the unmodified reference run in
fp64 on the same GPU, with the skip max-pool routed the way the engine routed it.

The skip max-pool (MultiScaleBlock.pool_skip) is the one non-smooth operator of these blocks: where the top two values
of a window are closer than the engine's forward error, the engine and the fp64 reference pick different inputs and
the gradient below the pool differs by far more than the rounding error.  Each pooled block of the reference therefore
gets a PinnedMaxPool that takes the window maxima at the taps the engine saved (its ``amax``), which leaves the
reference a smooth function of its inputs that follows the same routing; then the bounds of the ViT-B block test apply
to every block kind: logits rel-L2 < 1e-4 with the argmax exact, every parameter gradient rel-L2 < 1e-3.
"""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_gpu_vit import _fixture, _rel


def _triple(v):
    return tuple(v) if isinstance(v, (list, tuple)) else (v, v, v)


class PinnedMaxPool(nn.Module):
    """MaxPool3d(kernel, stride, padding) over [B, C, T, H, W] with the winning tap of every window given: out[b, c, o] =
    x[b, c, input position of tap taps[b, c, o] in window o].  Taps count (kz * kh + ky) * kw + kx over the kernel, padded
    positions included (token_maxpool_fwd_kernel's encoding).  ``rerouted`` counts, after each forward, the windows where
    max_pool3d of that same input picks a different position."""

    def __init__(self, taps, kernel, stride, padding):
        super().__init__()
        self.taps = taps.long()
        self.kernel, self.stride, self.padding = _triple(kernel), _triple(stride), _triple(padding)
        self.rerouted = None

    def forward(self, x):
        B, C, T, H, W = x.shape
        (kt, kh, kw), (st, sh, sw), (pt, ph, pw) = self.kernel, self.stride, self.padding
        oT, oH, oW = self.taps.shape[2:]
        assert self.taps.shape == (B, C, oT, oH, oW), (tuple(self.taps.shape), tuple(x.shape))
        taps = self.taps.to(x.device)
        dev = x.device
        iz = torch.arange(oT, device=dev).view(oT, 1, 1) * st - pt + taps // (kh * kw)
        iy = torch.arange(oH, device=dev).view(1, oH, 1) * sh - ph + taps // kw % kh
        ix = torch.arange(oW, device=dev).view(1, 1, oW) * sw - pw + taps % kw
        assert bool(((iz >= 0) & (iz < T) & (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)).all()), "tap in the padding"
        idx = ((iz * H + iy) * W + ix).view(B, C, -1)
        with torch.no_grad():
            _, own = F.max_pool3d(x, self.kernel, self.stride, self.padding, return_indices=True)
        self.rerouted = int((own.view(B, C, -1) != idx).sum())
        return x.flatten(2).gather(2, idx).view(B, C, oT, oH, oW)


def taps_from_amax(amax, ncls, othw):
    """The engine's saved skip-pool argmax [B, ncls + L_out, C] (uint8 taps, the cls row a pass-through) -> taps
    [B, C, oT, oH, oW] in the layout of the pooled tensor that attention_pool hands to the pool (cls row stripped)."""
    B, _, C = amax.shape
    return amax[:, ncls:].permute(0, 2, 1).reshape(B, C, *othw)


def _taps_from_indices(idx, thw, kernel, stride, padding):
    """max_pool3d's flat input indices [B, C, oT, oH, oW] -> taps in the encoding above."""
    T, H, W = thw
    oT, oH, oW = idx.shape[2:]
    iz, iy, ix = idx // (H * W), idx // W % H, idx % W
    kz = iz - (torch.arange(oT).view(oT, 1, 1) * stride[0] - padding[0])
    ky = iy - (torch.arange(oH).view(1, oH, 1) * stride[1] - padding[1])
    kx = ix - (torch.arange(oW).view(1, 1, oW) * stride[2] - padding[2])
    return (kz * kernel[1] + ky) * kernel[2] + kx


@pytest.mark.parametrize("thw,kernel,stride", [((8, 16, 16), (1, 3, 3), (1, 2, 2)),   # the MViT skip pool
                                               ((3, 7, 5), (3, 3, 3), (2, 2, 2)),     # odd extents, every axis pooled
                                               ((4, 6, 6), (1, 2, 2), (1, 2, 2))])    # no padding, no overlap
def test_pinned_maxpool_equals_maxpool3d_on_its_own_routing(thw, kernel, stride):
    """Pinned at the taps max_pool3d itself picked (passed through the engine's [B, cls + L, C] argmax layout), the
    module is MaxPool3d: forward and backward bitwise in fp64.  The output gradient is on a 2^-10 grid, so the sums of
    overlapping windows are exact in any order."""
    padding = tuple(k // 2 for k in kernel)
    g = torch.Generator().manual_seed(11)
    B, C = 2, 5
    x = torch.randn(B, C, *thw, generator=g, dtype=torch.float64)
    pool = nn.MaxPool3d(kernel, stride, padding)
    ref_in = x.clone().requires_grad_(True)
    want = pool(ref_in)
    _, idx = F.max_pool3d(x, kernel, stride, padding, return_indices=True)
    taps = _taps_from_indices(idx, thw, kernel, stride, padding)
    assert int(taps.min()) >= 0 and int(taps.max()) < kernel[0] * kernel[1] * kernel[2]
    othw = idx.shape[2:]
    amax = torch.cat([torch.zeros(B, 1, C, dtype=torch.uint8),
                      taps.to(torch.uint8).reshape(B, C, -1).permute(0, 2, 1)], 1)
    pinned = PinnedMaxPool(taps_from_amax(amax, 1, othw), kernel, stride, padding)
    got_in = x.clone().requires_grad_(True)
    got = pinned(got_in)
    assert pinned.rerouted == 0
    assert torch.equal(got, want)
    dy = torch.round(torch.randn(want.shape, generator=g, dtype=torch.float64) * 1024) / 1024
    want.backward(dy)
    got.backward(dy)
    assert torch.equal(got_in.grad, ref_in.grad)
    if not any(padding):  # pinned elsewhere (every tap in range), the module follows the taps, not the maxima
        other = PinnedMaxPool(torch.where(taps == 0, 1, 0), kernel, stride, padding)
        out = other(x)
        assert other.rerouted == out.numel() and not torch.equal(out, want.detach())


# ============================================================================================ block stacks vs fp64
_V2 = ["MVIT.DEPTH", 3, "MVIT.DIM_MUL", [[1, 2.0]], "MVIT.HEAD_MUL", [[1, 2.0]],
       "MVIT.POOL_Q_STRIDE", [[0, 1, 1, 1], [1, 1, 2, 2], [2, 1, 1, 1]]]

BLOCK_CASES = [  # (id, yaml, frames, crop, batch, overrides)
    # cls, rel-pos t + h + w, residual pooling, DIM_MUL_IN_ATT True (skip = proj(norm1 x) then max-pool), adaptive K/V
    ("v2s", "Kinetics/MVITv2_S_16x4.yaml", 8, 64, 2, _V2),
    # DIM_MUL_IN_ATT False (the proj(norm2 x1) residual), mean-token readout
    ("v2s-ft", "masked_ssl/k400_MVITv2_S_16x4_FT.yaml", 8, 64, 2, _V2),
    # head dim 72: 144 -> 288 wide, 2 -> 4 heads
    ("v2l-ft", "masked_ssl/k400_MVITv2_L_16x4_FT.yaml", 8, 64, 2, _V2),
    # MViTv1-B: separable absolute positions, no relative positions, no residual pooling
    ("v1b", "Kinetics/MVIT_B_16x4_CONV.yaml", 8, 64, 2,
     ["MVIT.DEPTH", 3, "MVIT.DIM_MUL", [[1, 2.0]], "MVIT.HEAD_MUL", [[1, 2.0]], "MVIT.POOL_Q_STRIDE", [[1, 1, 2, 2]]]),
    # images: no cls token, spatial-only relative positions, 2-D patch embedding
    ("v2t-image", "ImageNet/MVITv2_T.yaml", 1, 64, 2,
     _V2 + ["MVIT.POOL_KV_STRIDE", [[0, 1, 4, 4], [1, 1, 2, 2], [2, 1, 2, 2]]]),
    # the recipe's clip: 25 089 tokens in stage 1 (dwpool ring kernels, split-K dK / dV with K = Nq, Nk = 393 padded
    # to 400) and the stage-transition block; a third block after it, because under the cls readout the last block's
    # query-side parameters (pool_q, rel_pos_*) have no gradient
    ("v2s-224", "Kinetics/MVITv2_S_16x4.yaml", 16, 224, 1, _V2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("yaml,frames,crop,batch,over", [c[1:] for c in BLOCK_CASES], ids=[c[0] for c in BLOCK_CASES])
def test_mvit_blocks_match_reference_fp64_with_pinned_skip_pool(yaml, frames, crop, batch, over, cuda_device):
    """Logits and every parameter gradient of the engine (parity mode) against the reference in fp64, same fixture
    weights, clip and output gradient, skip pools pinned to the engine's routing.  Gradients that are zero in exact
    arithmetic (the key LayerNorm bias under pooling, the key third of the qkv bias) are held below 1e-3 of the median
    gradient norm, as in the whole-model comparison."""
    from oracle import refshim
    from oracle import torch_oracle as TO
    from slowfast_b200.nets.mvit import B200MViT
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    cfg = refshim.load_cfg(yaml, ["DATA.NUM_FRAMES", frames, "DATA.TRAIN_CROP_SIZE", crop, "DATA.TEST_CROP_SIZE", crop,
                                  "MODEL.DROPOUT_RATE", 0.0, "MVIT.DROPPATH_RATE", 0.0] + list(over))
    ref = refshim.build_reference_model(cfg)
    state = _fixture(ref.state_dict())
    ref.load_state_dict(state)
    ref = ref.to(cuda_device).double().train()
    mine = B200MViT(cfg)
    mine.load_state_dict(state)
    mine = mine.to(cuda_device).train()
    x = TO.synthetic_inputs(cfg, batch, 4)[0]
    if cfg.MVIT.PATCH_2D:
        x = x[:, :, 0]
    x = x.to(cuda_device)
    dl = torch.randn(batch, cfg.MODEL.NUM_CLASSES, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    lm = mine([x])
    saved = [(sv["amax"].clone() if sv["pool_skip"] else None, sv["q_thw"]) for sv in mine._saved["blocks"]]
    lm.backward(dl)
    torch.cuda.synchronize()
    pins = {}
    for i, (blk, (amax, q_thw)) in enumerate(zip(ref.blocks, saved)):
        assert (blk.pool_skip is None) == (amax is None), i
        if amax is not None:
            p = blk.pool_skip
            pins[i] = blk.pool_skip = PinnedMaxPool(taps_from_amax(amax, mine.ncls, q_thw), p.kernel_size, p.stride,
                                                    p.padding)
    assert pins, "no pooled skip in this stack"
    lr = ref([x.double()])
    lr.backward(dl.double())
    rel = _rel(lm.double(), lr)
    g64 = {k: p.grad for k, p in ref.named_parameters()}
    med = sorted(g.norm().item() for g in g64.values())[len(g64) // 2]
    zero = {k for k, g in g64.items() if g.norm().item() < 1e-6 * med}
    per = {k: _rel(p.grad.double(), g64[k]) for k, p in mine.named_parameters() if k not in zero}
    worst = max(per, key=per.get)
    windows = {i: (pin.rerouted, pin.taps.numel()) for i, pin in pins.items()}
    print(f"{yaml.split('/')[-1]} {frames}x{crop}^2 depth {cfg.MVIT.DEPTH} batch {batch}: logits rel-L2 {rel:.2e}; "
          f"grad rel-L2 median {sorted(per.values())[len(per) // 2]:.2e} max {per[worst]:.2e} ({worst}); "
          f"skip windows re-routed by the pin (of all): {windows}; zero in exact arithmetic: {sorted(zero)}")
    assert rel < 1e-4 and torch.equal(lm.argmax(1), lr.argmax(1))
    assert per[worst] < 1e-3, (worst, per[worst])
    for k in zero:
        assert mine.get_parameter(k).grad.norm().item() < 1e-3 * med, k
