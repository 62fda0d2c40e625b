"""MaskFeat pre-training wrapper (slowfast/models/masked.py:25 MaskMViT) on the engine.

``MaskMViT`` = the MViTv2 encoder with (a) masked patch tokens replaced by a learned ``mask_token`` right after the
patch embedding (masked.py:551-565), (b) no final norm / classification head but an ``MSSeparateHead`` (LayerNorm +
Linear on every masked token of the ``PRETRAIN_DEPTH`` blocks' outputs, head_helper.py:566-672) and (c) HOG regression
targets computed from the input frames (operators.py:79 HOGLayerC, masked.py:254-281).  ``forward`` returns
``(preds, labels)`` exactly like the reference so that ``MultipleMSELoss`` (losses.py:25) consumes it unchanged.

Execution: the encoder is ``B200MViT``'s program; the wrapper adds the masked token assembly, the prediction head
(LayerNorm over all token rows -> split planes -> wgmma GEMM 768 -> 108, run for every token so the program is
static and CUDA-graph capturable; the boolean row selection ``pred[mask]`` happens on the result, row-wise identical
to selecting first) and the HOG target kernel (csrc/maskfeat.cu).

Scope (asserted): MASK.PRED_HOG, HEAD_TYPE "separate" (no decoder transformer), MAE off, one or more PRETRAIN_DEPTH
entries that all equal the last block kept (the shipped MaskFeat yamls use [15] / [23]).
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import lib as L
from .. import ops
from ..engine import Namespace
from ..ops import BF16, F32, Planes
from .mvit import B200MViT


def calc_mvit_feature_geometry(cfg):
    """slowfast/models/utils.py:185-214."""
    depth = cfg.MVIT.DEPTH
    ps = list(cfg.MVIT.PATCH_STRIDE)
    feat_size = [[cfg.DATA.NUM_FRAMES // ps[0] if len(ps) > 2 else 1, cfg.DATA.TRAIN_CROP_SIZE // ps[-2],
                  cfg.DATA.TRAIN_CROP_SIZE // ps[-1]] for _ in range(depth)]
    feat_stride = [[ps[0] if len(ps) > 2 else 1, ps[-2], ps[-1]] for _ in range(depth)]
    for x in cfg.MVIT.POOL_Q_STRIDE:
        for i in range(depth):
            if i >= x[0]:
                for j in range(3):
                    feat_size[i][j] = feat_size[i][j] // x[j + 1]
                    feat_stride[i][j] = feat_stride[i][j] * x[j + 1]
    return feat_size, feat_stride


class HOGBuffers(nn.Module):
    """operators.HOGLayerC's registered buffers (checkpoint parity); the arithmetic is sfb_hog_targets."""

    def __init__(self, nbins=9, pool=8):
        super().__init__()
        self.nbins, self.pool = nbins, pool
        wx = torch.FloatTensor([[1, 0, -1], [2, 0, -2], [1, 0, -1]]).view(1, 1, 3, 3).repeat(3, 1, 1, 1)
        self.register_buffer("weight_x", wx)
        self.register_buffer("weight_y", wx.transpose(2, 3))


class MSSeparateHeadModule(Namespace):
    """MSSeparateHead parameter container: transforms[i] = Sequential(LayerNorm), projections[i] = Linear."""

    def __init__(self, dims, num_classes):
        super().__init__()
        self.transforms = nn.ModuleList()
        self.projections = nn.ModuleList()
        for d, nc in zip(dims, num_classes):
            self.transforms.append(nn.Sequential(nn.LayerNorm(d, eps=1e-6)))
            self.projections.append(nn.Linear(d, nc, bias=True))
        self.apply(self._init_weights)

    @staticmethod
    def _init_weights(m):  # head_helper.py:644-654
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)


class B200MaskMViT(B200MViT):
    """Drop-in for the reference's registered ``MaskMViT`` (MaskFeat with HOG targets).  A config with MASK.MAE_ON
    builds the MAE pre-training model instead (nets/mae.py), as the reference's one class serves both."""

    def __new__(cls, *args, **kwargs):
        if cls is B200MaskMViT and args and args[0].MASK.MAE_ON:
            from .mae import B200MAE
            return B200MAE(*args, **kwargs)
        return super().__new__(cls)

    def __init__(self, cfg):
        if cfg.MVIT.USE_ABS_POS:
            raise NotImplementedError("MVIT.USE_ABS_POS with MaskMViT (masked tokens before the position tables) is not "
                                      "on the engine path")
        if cfg.MVIT.PATCH_2D:
            raise NotImplementedError("MVIT.PATCH_2D with MaskMViT (image MaskFeat pre-training) is not on the engine "
                                      "path")
        super().__init__(cfg)
        mk = cfg.MASK
        assert mk.PRED_HOG and not mk.MAE_ON and not mk.MAE_RND_MASK, "only the HOG-target MaskFeat path is built"
        assert mk.HEAD_TYPE == "separate", "decoder-transformer heads are not on the engine path"
        assert not mk.SCALE_INIT_BY_DEPTH
        self.pretrain_depth = list(mk.PRETRAIN_DEPTH)
        last = self.pretrain_depth[-1]
        if last + 1 < cfg.MVIT.DEPTH:
            del self.blocks[last + 1:]
            self.specs = self.specs[:last + 1]
        assert all(d == last for d in self.pretrain_depth), "multi-depth prediction heads are not on the engine path"
        del self.norm
        del self.head
        self.feat_size, self.feat_stride = calc_mvit_feature_geometry(cfg)
        self.hogs = nn.ModuleList([HOGBuffers(nbins=9, pool=8)])
        self.nbins, self.cell_sz = 9, 8
        self.ncells = [(self.feat_stride[d][-1] // self.cell_sz) ** 2 for d in self.pretrain_depth]
        classes = [self.nbins * nc * 3 for nc in self.ncells]
        self.pred_head = MSSeparateHeadModule([self.specs[d]["dim_out"] for d in self.pretrain_depth], classes)
        self.hog_loss = "mse"
        self.mask_token = nn.Parameter(torch.zeros(1, 1, cfg.MVIT.EMBED_DIM))
        nn.init.trunc_normal_(self.mask_token, std=0.02)
        self.pred_hog_wt = 1.0

    @torch.jit.ignore
    def no_weight_decay(self):
        names = []
        if self.cfg.MVIT.ZERO_DECAY_POS_CLS and self.cfg.MVIT.CLS_EMBED_ON:
            names.append("cls_token")
        return names

    # ------------------------------------------------------------------------------------------ public forward
    def forward(self, x, return_all=False):
        """x = [frames (B,3,T,H,W), meta, mask (B, T', mh, mw)] -> (preds, labels) (masked.py:614-624)."""
        assert len(x) > 1, "MaskFeat needs the loader's mask: x = [frames, meta, mask]"
        frames, _, mask = x
        float_mask = mask.type_as(frames).contiguous()
        # multiscale boolean masks (masked.py:165-176): nearest resize of the cube mask to each feature map
        output_masks = [F.interpolate(float_mask, size=self.feat_size[d][-1]).flatten(1).to(torch.bool)
                        for d in self.pretrain_depth]
        pred_all = self._run([frames, float_mask])  # [B, L, classes], every token
        labels_all = self.hog_targets(frames)
        preds, labels = [], []
        for m in output_masks:
            preds.append(pred_all if return_all else pred_all[m])
            labels.append((labels_all[m], self.pred_hog_wt, self.hog_loss))
        return preds, labels

    @torch.no_grad()
    def hog_targets(self, frames: torch.Tensor) -> torch.Tensor:
        """_get_hog_label_3d (masked.py:254-281) for every token: [B, T'*fs*fs, 3*nbins*u*u]."""
        if frames.device.type != "cuda":
            raise L.NativeLibraryError("slowfast_b200 runs on CUDA devices only (no CPU fallback)")
        B, C, T, H, W = frames.shape
        ts = self.cfg.MVIT.PATCH_STRIDE[0]
        fs = self.feat_size[self.pretrain_depth[-1]][-1]
        u = (H // self.cell_sz) // fs
        out = torch.empty((B, (T // ts) * fs * fs, C * self.nbins * u * u), dtype=F32, device=frames.device)
        ops.hog_targets(frames.contiguous().float(), ts, self.nbins, self.cell_sz, fs, out)
        return out

    # ------------------------------------------------------------------------------------------ engine hooks
    def _tokens_assemble(self, ype, x0, B, Lt, E, inputs) -> None:
        ctx = self.ctx
        fmask = inputs[1]
        mb, mt, mh, mw = fmask.shape
        assert mb == B and mt == self.T, "the cube mask must have one slice per token frame"
        tokmask = ctx.buf(("mf.tokmask",), (B, Lt))
        ops.mask_upsample(fmask, (self.T, self.H, self.W), tokmask)
        pe = self.patch_embed.proj
        ops.tokens_assemble_masked(ype, pe.bias, self.cls_token, self.mask_token, tokmask, B, Lt, E, x0)

    def _tokens_split_grad(self, dx, B, Lt, E):
        ctx = self.ctx
        dyp = self._rows_planes("pe.dy", B * Lt, E, scratch=True)
        dyf = ctx.scratch("pe.dyf", B * Lt * E, F32)
        dxm = ctx.scratch("mf.dxm", B * Lt * E, F32)
        tokmask = ctx.buf(("mf.tokmask",), (B, Lt))
        ops.tokens_split_grad_masked(dx, tokmask, B, Lt, E, dyp, dyf, dxm)
        self._colsum(dxm, B * Lt, E, ctx.grad_of(self.mask_token).view(E))
        return dyp, dyf

    def _final_forward(self, cur: torch.Tensor, thw, B) -> torch.Tensor:
        """MSSeparateHead (head_helper.py:656-672) for every token of the last kept block."""
        ctx = self.ctx
        Nf, Cf = cur.shape[1], cur.shape[2]
        ln = self.pred_head.transforms[0][0]
        proj = self.pred_head.projections[0]
        nc = proj.out_features
        rows = B * Nf
        xn = self._rows_planes(("mf.xn",), rows, Cf)
        mean, rstd = ctx.buf(("mf.mean",), (rows,)), ctx.buf(("mf.rstd",), (rows,))
        self._ln_fwd(cur, Cf, rows, Cf, ln, xn, None, mean, rstd)
        y = self._lin_fwd(("mf.y",), proj, xn)  # [rows, nc] (bias added below)
        pred = torch.empty((B, Nf - 1, nc), dtype=F32, device=ctx.device)
        ops.rows_unpad_bias(y, nc, proj.bias, B, Nf - 1, nc, pred)
        self._saved["final"] = (cur, xn, mean, rstd)
        return pred

    def _final_backward(self, dpred: torch.Tensor) -> torch.Tensor:
        ctx = self.ctx
        sv = self._saved
        B = sv["B"]
        cur, xn, mean, rstd = sv["final"]
        Nf, Cf = cur.shape[1], cur.shape[2]
        ln = self.pred_head.transforms[0][0]
        proj = self.pred_head.projections[0]
        nc = proj.out_features
        ncp = ops.pad8(nc)
        rows = B * Nf
        # gradient w.r.t. the Linear output for every row (cls rows and the pad columns are zero)
        dyp = ctx.scratch_planes("mf.dy", 1, 1, 1, rows, ncp)
        ops.rows_pad_split(dpred, B, Nf - 1, nc, dyp)
        self._colsum(dpred, B * (Nf - 1), nc, ctx.grad_of(proj.bias))
        # dW [ncp, Cf] (rows >= nc are zero) -> parameter gradient; dxn = dy . W
        dwm = ctx.scratch("mf.dwm", ncp * Cf, F32).view(ncp, Cf)
        ops.zero_f32(ops.f32view(dwm))
        geom = ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (xn.t, xn.h, xn.w))
        ops.conv_wgrad(xn, dyp, geom, dwm, nsplit=ctx.nsplit)
        ops.filter_unpack_grad(dwm, ctx.grad_of(proj.weight), Cf, accumulate=False)
        f = ctx.scratch("lin.ft.hi", Cf * ncp, BF16).view(Cf, ncp)
        flo = ctx.scratch("lin.ft.lo", Cf * ncp, BF16).view(Cf, ncp) if ctx.nsplit == 3 else None
        fm = ops.FilterMat(f, flo, Cf, 1, ncp)
        ops.filter_pack(proj.weight, fm, tapmap=[0], transpose=True)
        dxn = ctx.scratch("mf.dxn", rows * Cf, F32).view(rows, Cf)
        ops.conv_igemm(dyp, fm, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, rows)), dxn,
                       (rows * Cf, rows * Cf, rows * Cf, Cf), nsplit=ctx.nsplit)
        dx = ctx.scratch("dx.a", rows * Cf, F32).view(B, Nf, Cf)
        self._ln_bwd(dxn, Cf, cur, Cf, rows, Cf, ln, mean, rstd, dx, Cf, False)
        return dx
