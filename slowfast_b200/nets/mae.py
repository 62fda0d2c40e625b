"""MAE pre-training (slowfast/models/masked.py:25 MaskMViT with MASK.MAE_ON, the k400_VIT_{B,L,H}_16x4_MAE_PT recipes)
on the engine.

Module tree and initialisation mirror the reference: the MViT (ViT) encoder is built whole - its ``norm`` and ``head``
draw from the RNG and are then deleted - and cut after ``PRETRAIN_DEPTH[-1]``; then ``pred_head`` (MSSeparateHead:
``transforms[0]`` = DECODER_DEPTH unpooled blocks at DECODER_EMBED_DIM + LayerNorm, ``projections[0]`` = Linear to the
patch pixels, head_helper.py:565-654), a fresh ``norm`` (ones / zeros), ``decoder_embed`` (PyTorch's default init),
``decoder_pos_embed`` [1, L+1, D] and ``mask_token`` [1, 1, D], trunc-normal in that order (masked.py:78-121).

Execution (one static program per input signature; len_keep = int(L * (1 - MASK_RATIO)) is fixed by the shapes):
  * ``forward`` draws ``noise = torch.rand(B, L)`` exactly as the reference does and hands it to the program as an
    input, so eager and CUDA-graph runs mask the tokens the reference would mask under the same seed;
  * sfb_mae_random_masking: stable-argsort ranks -> ids_keep / ids_restore / mask / the removed rows;
  * only the kept patches are packed (sfb_patchify_gather) and embedded: the GEMM and its weight gradient run over
    B * len_keep rows; sfb_tokens_assemble_keep adds the cls token and the separable positions gathered by ids_keep;
  * the encoder blocks run at 1 + len_keep tokens.  They see the kept tokens as a 1 x 1 x len_keep grid, which is exact
    because the MAE encoders neither pool nor use relative positions (rejected at construction);
  * norm -> decoder_embed on all B * (1 + len_keep) rows; sfb_decoder_assemble un-shuffles with the mask token and adds
    the joint table; the decoder blocks run at L + 1 tokens;
  * the head's LayerNorm and projection run on the removed tokens only (rows are independent, so selecting first is
    row-wise identical to the reference's x[mask] after the LayerNorm); the prediction rows come out in the reference's
    order, removed tokens of clip 0 in ascending position, then clip 1 ...;
  * sfb_pixel_targets computes the normalised-pixel labels of the same rows.
"""
from __future__ import annotations

import math
from typing import List

import torch
import torch.nn as nn

from .. import lib as L
from .. import ops
from ..engine import Namespace
from ..ops import F32
from .maskfeat import MSSeparateHeadModule, calc_mvit_feature_geometry
from .mvit import B200MViT, BlockModule, _is_pool, block_specs

MAE_MAX_TOKENS = 4096  # sfb_mae_max_tokens(): one clip's noise row in the masking kernel's shared memory
I32 = torch.int32


class MAEHeadModule(Namespace):
    """MSSeparateHead with the "xformer" transform: transforms[0] = Sequential(blocks..., LayerNorm), projections[0]."""

    def __init__(self, blocks: List[nn.Module], dim: int, num_classes: int):
        super().__init__()
        self.transforms = nn.ModuleList([nn.Sequential(*blocks, nn.LayerNorm(dim, eps=1e-6))])
        self.projections = nn.ModuleList([nn.Linear(dim, num_classes, bias=True)])
        self.apply(MSSeparateHeadModule._init_weights)


class B200MAE(B200MViT):
    """Drop-in for the reference's ``MaskMViT`` with MASK.MAE_ON (served through ``B200MaskMViT``'s constructor)."""

    def __init__(self, cfg):
        self._reject_mae(cfg)
        super().__init__(cfg)
        mk = cfg.MASK
        last = list(mk.PRETRAIN_DEPTH)[-1]
        if last + 1 < cfg.MVIT.DEPTH:
            del self.blocks[last + 1:]
            self.specs = self.specs[:last + 1]
        del self.norm
        del self.head
        _, feat_stride = calc_mvit_feature_geometry(cfg)
        self.pred_t = 1 if mk.TIME_STRIDE_LOSS else self.patch_stride[0]
        self.pixel_patch = feat_stride[last][-1]
        num_classes = self.pred_t * self.pixel_patch ** 2 * 3
        dec = mk.DECODER_EMBED_DIM
        n_dec = mk.DECODER_DEPTH if "xformer" in mk.HEAD_TYPE.split("_")[1:] else 0
        self.dec_specs = [dict(dim=dec, dim_out=dec, heads=dec // 64, kq=[], kkv=[], sq=[], skv=[],
                               size=[self.T, self.H, self.W]) for _ in range(n_dec)]
        blocks = [BlockModule(s, cfg.MVIT.MLP_RATIO, cfg.MVIT.QKV_BIAS, False, False, False, False)
                  for s in self.dec_specs]
        self.pred_head = MAEHeadModule(blocks, dec, num_classes)
        dim = self.specs[-1]["dim_out"]
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.decoder_embed = nn.Linear(dim, dec, bias=True)
        self.n_tokens = self.T * self.H * self.W
        self.decoder_pos_embed = nn.Parameter(torch.zeros(1, self.n_tokens + 1, dec))
        self.mask_token = nn.Parameter(torch.zeros(1, 1, dec))
        nn.init.trunc_normal_(self.mask_token, std=0.02)
        nn.init.trunc_normal_(self.decoder_pos_embed, std=0.02)
        self.mask_ratio = cfg.AUG.MASK_RATIO
        self.len_keep = int(self.n_tokens * (1 - self.mask_ratio))  # masked.py:302, float expression kept
        if not 1 < self.len_keep < self.n_tokens:
            raise NotImplementedError(f"AUG.MASK_RATIO {self.mask_ratio} keeps {self.len_keep} of {self.n_tokens} tokens "
                                      "(MAE needs more than one kept and at least one removed token)")
        self.norm_pix = bool(mk.NORM_PRED_PIXEL)

    @staticmethod
    def _reject_mae(cfg):
        """MAE configurations the reference builds but this program does not run fail here, naming the option."""
        mk, mv = cfg.MASK, cfg.MVIT
        ps = list(mv.PATCH_STRIDE)
        crop = cfg.DATA.TRAIN_CROP_SIZE
        n_tokens = (cfg.DATA.NUM_FRAMES // ps[0]) * (crop // ps[-2]) * (crop // ps[-1])
        rel = bool(mv.REL_POS_SPATIAL) or bool(mv.REL_POS_TEMPORAL)
        pooled = any(_is_pool(s["kq"], s["sq"]) or _is_pool(s["kkv"], s["skv"]) for s in block_specs(cfg))
        bad = [
            (bool(mk.PER_FRAME_MASKING), "MASK.PER_FRAME_MASKING (per-frame MAE masking)"),
            (bool(cfg.AUG.MASK_TUBE), "AUG.MASK_TUBE (tube masking)"),
            (not mk.MAE_RND_MASK, "MASK.MAE_ON without MASK.MAE_RND_MASK (a loader-supplied MAE mask)"),
            (bool(mk.DECODER_SEP_POS_EMBED), "MASK.DECODER_SEP_POS_EMBED True (separable decoder position tables)"),
            (bool(mk.DEC_KV_KERNEL) or bool(mk.DEC_KV_STRIDE), "MASK.DEC_KV_KERNEL / DEC_KV_STRIDE (pooled decoder K/V)"),
            (bool(mk.PRED_HOG), "MASK.PRED_HOG with MASK.MAE_ON (HOG targets for MAE)"),
            (bool(mk.SCALE_INIT_BY_DEPTH), "MASK.SCALE_INIT_BY_DEPTH"),
            (bool(cfg.VIS_MASK.ENABLE), "VIS_MASK.ENABLE (mask visualisation)"),
            (not mv.USE_ABS_POS, "MVIT.USE_ABS_POS False with MAE"),
            (not mv.SEP_POS_EMBED, "MVIT.SEP_POS_EMBED False with MAE (a joint encoder pos_embed table)"),
            (len(mk.PRETRAIN_DEPTH) != 1, f"MASK.PRETRAIN_DEPTH {list(mk.PRETRAIN_DEPTH)} (more than one prediction depth)"),
            (n_tokens > MAE_MAX_TOKENS, f"{n_tokens} tokens per clip (the MAE masking kernel holds at most "
                                        f"{MAE_MAX_TOKENS})"),
            (pooled or rel, "pooling or relative positions in the MAE encoder (it runs on a subset of the tokens)"),
            (bool(mv.RESIDUAL_POOLING), "MVIT.RESIDUAL_POOLING with MAE"),
            (float(mv.DROPPATH_RATE) > 0.0, "MVIT.DROPPATH_RATE > 0 with MAE (stochastic depth in the encoder)"),
            (list(mv.PATCH_KERNEL) != ps or any(mv.PATCH_PADDING),
             "an overlapping or padded patch embedding with MAE (the kept patches are packed as rows)"),
        ]
        for cond, what in bad:
            if cond:
                raise NotImplementedError(f"{what} is not on the engine path")

    @torch.jit.ignore
    def no_weight_decay(self):
        """MaskMViT.no_weight_decay (masked.py:129-147), verbatim: it names the joint decoder table
        ``pos_embed_decoder`` and never lists the encoder's position tables."""
        names = []
        if self.cfg.MVIT.ZERO_DECAY_POS_CLS:
            names.extend(["pos_embed_decoder"])
            names.append("cls_token")
        return names

    # ------------------------------------------------------------------------------------------ public forward
    def forward(self, x, return_all=False):
        """x = [frames (B,3,T,H,W)] -> ([pred], [(label, 1.0)]) (masked.py:447-476, 614-621)."""
        assert not return_all
        frames = x[0]
        noise = torch.rand(frames.shape[0], self.n_tokens, device=frames.device)  # masked.py:298
        pred = self._run([frames, noise])
        B = frames.shape[0]
        rows = self.ctx.buf(("mae.rows",), (B * (self.n_tokens - self.len_keep),), I32)
        return [pred], [(self.pixel_targets(frames, rows), 1.0)]

    @torch.no_grad()
    def pixel_targets(self, frames: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
        """_get_pixel_label_3d (masked.py:212-230) for the decoder rows ``rows``: [len(rows), pred_t * p * p * 3]."""
        if frames.device.type != "cuda":
            raise L.NativeLibraryError("slowfast_b200 runs on CUDA devices only (no CPU fallback)")
        B, C, T, H, W = frames.shape
        p = self.pixel_patch
        out = torch.empty((rows.numel(), self.pred_t * p * p * C), dtype=F32, device=frames.device)
        ops.pixel_targets(frames.contiguous().float(), self.patch_stride[0], self.pred_t, p, rows, self.norm_pix, out)
        return out

    # ------------------------------------------------------------------------------------------ forward program
    def _forward_program(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
        x, noise = inputs
        B, cin, t, h, w = x.shape
        Lt, K = self.n_tokens, self.len_keep
        M = Lt - K
        assert tuple(noise.shape) == (B, Lt), (tuple(noise.shape), (B, Lt))
        # ---- masking ------------------------------------------------------------------------------------------
        ids_keep = ctx.buf(("mae.keep",), (B, K), I32)
        ids_restore = ctx.buf(("mae.restore",), (B, Lt), I32)
        mask = ctx.buf(("mae.mask",), (B, Lt))
        rows = ctx.buf(("mae.rows",), (B * M,), I32)
        ops.mae_random_masking(noise, K, ids_keep, ids_restore, mask, rows)
        # ---- patch embedding of the kept patches -> encoder tokens ---------------------------------------------------
        pe = self.patch_embed.proj
        k3, E = tuple(pe.kernel_size), pe.out_channels
        assert (t // k3[0], h // k3[1], w // k3[2]) == (self.T, self.H, self.W)
        Kd = cin * math.prod(k3)
        xin = self._rows_planes(("pe.rows",), B * K, Kd)
        ops.patchify_gather(x.contiguous().float(), k3, ids_keep, K, xin)
        ype = self._mat_fwd(("pe.y",), pe.weight.view(E, Kd), xin)
        x0 = ctx.buf(("x", 0), (B, K + 1, E))
        ops.tokens_assemble_keep(ype, pe.bias, self.cls_token, self.pos_embed_spatial, self.pos_embed_temporal,
                                 self.pos_embed_class, ids_keep, B, K, Lt, self.H * self.W, E, x0)
        # ---- encoder (the kept tokens as a 1 x 1 x K grid) -----------------------------------------------------------
        saved = []
        cur = x0
        for i, (blk, spec) in enumerate(zip(self.blocks, self.specs)):
            cur, _, sv = self._block_forward(i, blk, spec, cur, [1, 1, K], B, None)
            saved.append(sv)
        enc = cur
        Ce = enc.shape[2]
        rows_e = B * (K + 1)
        lat = self._rows_planes(("mae.lat",), rows_e, Ce)
        em, er = ctx.buf(("mae.em",), (rows_e,)), ctx.buf(("mae.er",), (rows_e,))
        self._ln_fwd(enc, Ce, rows_e, Ce, self.norm, lat, None, em, er)
        # ---- decoder ------------------------------------------------------------------------------------------------
        z = self._lin_fwd(("mae.z",), self.decoder_embed, lat)
        D = self.decoder_embed.out_features
        xd = ctx.buf(("mae.xd",), (B, Lt + 1, D))
        ops.decoder_assemble(z, self.decoder_embed.bias, self.mask_token, self.decoder_pos_embed, ids_restore, B, K, Lt, D,
                             xd)
        n_enc = len(self.blocks)
        dec_saved = []
        cur = xd
        head = self.pred_head.transforms[0]
        for j, spec in enumerate(self.dec_specs):
            cur, _, sv = self._block_forward(n_enc + j, head[j], spec, cur, [self.T, self.H, self.W], B, None)
            dec_saved.append(sv)
        # ---- head on the removed tokens -----------------------------------------------------------------------------
        sel = ctx.buf(("mae.sel",), (B * M, D))
        ops.rows_gather(cur, D, rows, B * M, D, None, sel)
        seln = self._rows_planes(("mae.seln",), B * M, D)
        hm, hr = ctx.buf(("mae.hm",), (B * M,)), ctx.buf(("mae.hr",), (B * M,))
        self._ln_fwd(sel, D, B * M, D, head[len(self.dec_specs)], seln, None, hm, hr)
        proj = self.pred_head.projections[0]
        y = self._lin_fwd(("mae.y",), proj, seln)
        nc = proj.out_features
        pred = torch.empty((B * M, nc), dtype=F32, device=ctx.device)
        ops.rows_gather(y, nc, None, B * M, nc, proj.bias, pred)
        object.__setattr__(self, "_saved", dict(B=B, xin=xin, blocks=saved, dec=dec_saved, enc=enc, lat=lat, em=em,
                                                er=er, sel=sel, seln=seln, hm=hm, hr=hr, ids_keep=ids_keep,
                                                ids_restore=ids_restore, rows=rows))
        return pred

    # ------------------------------------------------------------------------------------------ backward program
    def _backward_program(self, dpred: torch.Tensor) -> None:
        ctx = self.ctx
        sv = self._saved
        B = sv["B"]
        Lt, K = self.n_tokens, self.len_keep
        M = Lt - K
        head = self.pred_head.transforms[0]
        proj = self.pred_head.projections[0]
        nc, D = proj.out_features, proj.in_features
        rows = sv["rows"]
        # ---- projection + LayerNorm on the removed rows; kept rows and the cls rows get zero gradient ----------------
        dpp = ctx.scratch_planes("mae.dpred", 1, 1, 1, B * M, nc)
        ops.split_planes(dpred.view(1, 1, 1, B * M, nc), dpp)
        dseln = ctx.scratch("mae.dseln", B * M * D, F32).view(B * M, D)
        self._lin_bwd(proj, dpp, dpred, sv["seln"], dseln)
        dsel = ctx.scratch("mae.dsel", B * M * D, F32).view(B * M, D)
        self._ln_bwd(dseln, D, sv["sel"], D, B * M, D, head[len(self.dec_specs)], sv["hm"], sv["hr"], dsel, D, False)
        dxd = ctx.scratch("mae.dxd", B * (Lt + 1) * D, F32).view(B, Lt + 1, D)
        ops.zero_f32(ops.f32view(dxd.view(B * (Lt + 1), D)))
        ops.rows_scatter(dsel, rows, B * M, D, dxd)
        # ---- decoder blocks --------------------------------------------------------------------------------------
        n_enc = len(self.blocks)
        which = "a"
        dx = dxd
        for j in range(len(self.dec_specs) - 1, -1, -1):
            which = "b" if which == "a" else "a"
            dx = self._block_backward(n_enc + j, head[j], self.dec_specs[j], sv["dec"][j], dx, B, which)
        # ---- decoder assembly: d decoder_embed output, d decoder_pos_embed, d mask_token ---------------------------
        dz = ctx.scratch("mae.dz", B * (K + 1) * D, F32).view(B * (K + 1), D)
        part = ctx.scratch("mae.part", ops.segment_slabs(1, B * M) * D, F32)
        ops.decoder_assemble_bwd(dx, sv["ids_keep"], rows, B, K, Lt, D, dz, ctx.grad_of(self.decoder_pos_embed),
                                 ctx.grad_of(self.mask_token), part)
        rows_e = B * (K + 1)
        dzp = ctx.scratch_planes("mae.dzp", 1, 1, 1, rows_e, D)
        ops.split_planes(dz.view(1, 1, 1, rows_e, D), dzp)
        Ce = sv["enc"].shape[2]
        dlat = ctx.scratch("mae.dlat", rows_e * Ce, F32).view(rows_e, Ce)
        self._lin_bwd(self.decoder_embed, dzp, dz, sv["lat"], dlat)
        dxe = ctx.scratch("mae.dxe", rows_e * Ce, F32).view(B, K + 1, Ce)
        self._ln_bwd(dlat, Ce, sv["enc"], Ce, rows_e, Ce, self.norm, sv["em"], sv["er"], dxe, Ce, False)
        # ---- encoder blocks --------------------------------------------------------------------------------------
        dx = dxe
        for i in range(n_enc - 1, -1, -1):
            which = "b" if which == "a" else "a"
            dx = self._block_backward(i, self.blocks[i], self.specs[i], sv["blocks"][i], dx, B, which)
        # ---- token assembly: positions (on the dense grid), cls, patch-embedding bias and weight ------------------
        pe = self.patch_embed.proj
        E = pe.out_channels
        T, HW = self.T, self.H * self.W
        dense = ctx.scratch("mae.dense", B * (Lt + 1) * E, F32)
        ops.tokens_scatter_keep(dx, sv["ids_restore"], B, K, Lt, E, dense)
        ppart = ctx.scratch("pos.part", T * ops.segment_slabs(T, HW) * E, F32)
        ops.pos_embed_sep_bwd(dense, B, T, HW, E, ctx.grad_of(self.pos_embed_spatial), ctx.grad_of(self.pos_embed_temporal),
                              ctx.grad_of(self.pos_embed_class), ppart)
        dyp, dyf = self._tokens_split_grad(dx, B, K, E)
        self._colsum(dyf, B * K, E, ctx.grad_of(pe.bias))
        self._colsum(dx, B, E, ctx.grad_of(self.cls_token).view(E), pitch=(K + 1) * E)
        xr = sv["xin"]
        gw = ctx.grad_of(pe.weight).view(E, xr.c)
        ops.zero_f32(ops.f32view(gw))
        ops.conv_wgrad(xr, dyp, ops.ConvGeom((1, 1, 1), (1, 1, 1), (0, 0, 0), (xr.t, xr.h, xr.w)), gw, nsplit=ctx.nsplit)
