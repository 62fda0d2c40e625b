"""Single-pathway ResNet video models (C2D / I3D / Slow; video_model_builder.py:445 ResNet) on the engine.

Same building blocks as ``B200SlowFast`` (W-shift stem, wgmma bottleneck blocks, fused BN/ReLU/residual passes),
plus the temporal max-pool the c2d / i3d archs insert after res2 (``pathway0_pool``, _POOL1 :100-103).
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from .. import ops
from ..engine import Act, ConvBN, Namespace, StemConvBN
from .resnet import (POOL1, STAGE_DEPTH, TEMPORAL_KERNELS, BasicHeadModule, StageModule, StemModule,
                     _VideoResNetBase, init_resnet_weights)


class B200ResNet(_VideoResNetBase):
    num_pathways = 1

    def __init__(self, cfg):
        super().__init__(cfg)
        self._check_cfg(cfg)
        assert cfg.MODEL.ARCH in POOL1 and len(POOL1[cfg.MODEL.ARCH]) == 1, cfg.MODEL.ARCH
        ctx = self.ctx
        d2, d3, d4, d5 = STAGE_DEPTH[cfg.RESNET.DEPTH]
        wpg = cfg.RESNET.WIDTH_PER_GROUP
        dim_inner = cfg.RESNET.NUM_GROUPS * wpg
        tk = TEMPORAL_KERNELS[cfg.MODEL.ARCH]
        self._pool1 = tuple(POOL1[cfg.MODEL.ARCH][0])
        cin = cfg.DATA.INPUT_CHANNEL_NUM
        self.s1 = Namespace()
        self.s1.add_module("pathway0_stem", StemModule(cin[0], wpg, tk[0][0] + [7, 7], (1, 2, 2),
                                                       (tk[0][0][0] // 2, 3, 3), 1e-5, 0.1, self._norm))
        widths = [wpg * 4, wpg * 8, wpg * 16, wpg * 32]
        prev = wpg
        for i, (wd, dp) in enumerate(zip(widths, (d2, d3, d4, d5))):
            st = StageModule(f"s{i + 2}", dim_in=[prev], dim_out=[wd], dim_inner=[dim_inner * (2 ** i)],
                             temp_kernel_sizes=tk[i + 1], stride=cfg.RESNET.SPATIAL_STRIDES[i], num_blocks=[dp],
                             num_block_temp_kernel=cfg.RESNET.NUM_BLOCK_TEMP_KERNEL[i],
                             stride_1x1=cfg.RESNET.STRIDE_1X1, ctx=ctx, nonlocal_inds=cfg.NONLOCAL.LOCATION[i],
                             nonlocal_pool=cfg.NONLOCAL.POOL[i], nonlocal_group=cfg.NONLOCAL.GROUP[i],
                             instantiation=cfg.NONLOCAL.INSTANTIATION, norm=self._norm)
            self.add_module(f"s{i + 2}", st)
            if i == 0:
                self.add_module("pathway0_pool", nn.MaxPool3d(kernel_size=list(self._pool1), stride=list(self._pool1),
                                                              padding=[0, 0, 0]))
            prev = wd
        crop32 = cfg.DATA.TRAIN_CROP_SIZE // 32
        p1 = self._pool1
        pools = None if cfg.MULTIGRID.SHORT_CYCLE or cfg.MODEL.MODEL_NAME == "ContrastiveModel" else [[cfg.DATA.NUM_FRAMES // p1[0], crop32 // p1[1], crop32 // p1[2]]]
        self.head = BasicHeadModule([wpg * 32], cfg.MODEL.NUM_CLASSES, cfg.MODEL.DROPOUT_RATE, cfg.MODEL.HEAD_ACT,
                                    pool_size=pools, contrastive=cfg.get("CONTRASTIVE"),
                                    detach_final_fc=cfg.MODEL.DETACH_FINAL_FC)
        init_resnet_weights(self, cfg.MODEL.FC_INIT_STD, cfg.RESNET.ZERO_INIT_FINAL_BN,
                            cfg.RESNET.ZERO_INIT_FINAL_CONV)
        self._stem_saved = {}
        object.__setattr__(self, "_units", None)

    def _engine_units(self):
        if self._units is None:
            stem = self.s1.pathway0_stem
            crop = int(self.cfg.DATA.TRAIN_CROP_SIZE)
            cls = StemConvBN if StemConvBN.supported(stem.conv, crop) else ConvBN
            object.__setattr__(self, "_units", {"stem0": cls("s1.p0", stem.conv, stem.bn, self.ctx)})
        return self._units

    def _forward_program(self, inputs: List[torch.Tensor]) -> torch.Tensor:
        ctx = self.ctx
        u = self._engine_units()
        (x,) = inputs
        n = x.shape[0]
        c0 = u["stem0"].cout
        t, h, w = u["stem0"].out_dims(*x.shape[2:])
        ph, pw = ops.conv_out_size(h, 3, 2, 1), ops.conv_out_size(w, 3, 2, 1)
        cur = Act(ctx.storage(("s1", 0), n, t, ph, pw, c0))
        self._stem_forward(0, x, self.s1.pathway0_stem, u["stem0"], cur)
        self._pool_saved = None
        for i in range(2, 6):
            stage: StageModule = getattr(self, f"s{i}")
            for bi, blk in enumerate(stage.blocks(0)):
                tt, hh, ww = blk.out_dims(*cur.dims[1:])
                out = Act(ctx.storage((f"s{i}", 0, bi), n, tt, hh, ww, blk._dim_out))
                stage.run_block_forward(0, bi, cur, out, (f"s{i}", 0, bi))
                cur = out
            if i == 2 and self._pool1 != (1, 1, 1):
                k = self._pool1
                _, tt, hh, ww = cur.dims
                od = (tt // k[0], hh // k[1], ww // k[2])
                pooled = Act(ctx.storage(("pool1",), n, *od, cur.c))
                argmax = ctx.buf(("pool1.argmax",), (n, *od, cur.c), torch.uint8)
                ops.maxpool3d_fwd(cur.planes, pooled.planes, argmax, k, k, (0, 0, 0))
                self._pool_saved = (cur, pooled, argmax, k)
                cur = pooled
        return self._head_forward([cur])

    def _backward_program(self, dlogits: torch.Tensor) -> None:
        u = self._engine_units()
        if not self._head_backward(dlogits):
            return
        for i in range(5, 1, -1):
            if i == 2 and self._pool_saved is not None:
                src, pooled, argmax, k = self._pool_saved
                assert not src.s.grad_written
                ops.maxpool3d_bwd(pooled.grad_view(), argmax, src.planes, pooled.dims[1:], src.grad_view(), k, k,
                                  (0, 0, 0))
                src.s.grad_written = True
            stage: StageModule = getattr(self, f"s{i}")
            for bi in reversed(range(stage.num_blocks[0])):
                stage.run_block_backward(0, bi)
        self._stem_backward(0, u["stem0"])
