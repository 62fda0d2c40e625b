"""The launch boundary of the model programs and the launch counter behind bench.py's ``gpu_launches``.

  * host: ``slowfast_b200/nets/*.py`` reach the native library only through ``slowfast_b200.ops`` (no ctypes, no
    ``sfb_*`` symbol, no ``check`` / ``_count`` of their own), so every launch passes through a function that counts it;
  * GPU: for each model family one eager training step under torch.profiler issues exactly as many device activities
    of the library as ``ops.launches()`` counted.
"""
import ast
import collections
import os

import pytest
import torch

NETS = os.path.join(os.path.dirname(__file__), os.pardir, "slowfast_b200", "nets")


def test_model_programs_reach_the_library_only_through_ops():
    files = sorted(f for f in os.listdir(NETS) if f.endswith(".py"))
    assert "mvit.py" in files and "resnet.py" in files
    bad = []
    for fn in files:
        tree = ast.parse(open(os.path.join(NETS, fn)).read(), fn)
        for node in ast.walk(tree):
            if isinstance(node, ast.Import) and any(a.name.split(".")[0] == "ctypes" for a in node.names):
                bad.append((fn, node.lineno, "import ctypes"))
            elif isinstance(node, ast.ImportFrom) and (node.module or "").split(".")[0] == "ctypes":
                bad.append((fn, node.lineno, "from ctypes import"))
            elif isinstance(node, ast.Attribute):
                if node.attr.startswith("sfb_"):
                    bad.append((fn, node.lineno, node.attr))
                owner = node.value.id if isinstance(node.value, ast.Name) else getattr(node.value, "attr", None)
                if node.attr in ("check", "_count") and owner in ("L", "lib", "ops"):
                    bad.append((fn, node.lineno, f"{owner}.{node.attr}"))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ GPU
def _family(name):
    """(model, batch, inputs, loss(outputs, batch)) of one family at a small shape, eager (no CUDA graphs)."""
    import torch.nn.functional as F
    from oracle import torch_oracle as TO
    from slowfast_b200.config import get_cfg
    from slowfast_b200.nets.maskfeat import B200MaskMViT
    from test_gpu_replay import FAMILIES, _cls

    def xent(out, b):
        return F.cross_entropy(out, torch.arange(b, device=out.device))

    def mse(out, b):
        preds, labels = out
        return sum(F.mse_loss(p, lab[0]) for p, lab in zip(preds, labels))

    small = dict(NUM_FRAMES=4, TRAIN_CROP_SIZE=64, TEST_CROP_SIZE=64)
    eager = {"NSPLIT": 3, "CUDA_GRAPH": False}
    batch, loss = 2, xent
    if name in FAMILIES:
        preset, over, batch = FAMILIES[name]
        cfg = get_cfg(preset, B200=eager, **over)
    elif name == "vit":
        cfg = get_cfg("VIT_B_16x4_FT", DATA=small, MVIT={"DEPTH": 2}, B200=eager)
    elif name == "mae":
        cfg = get_cfg("VIT_B_16x4_MAE_PT", DATA=small, MVIT={"DEPTH": 2}, MASK={"PRETRAIN_DEPTH": [1]}, B200=eager)
        loss = mse
    elif name == "maskfeat":
        cfg, loss = get_cfg("MVITv2_S_16x4_MaskFeat_PT", DATA=dict(small, NUM_FRAMES=8), B200=eager), mse
    else:
        cfg = get_cfg("MVITv2_T", DATA={"TRAIN_CROP_SIZE": 64, "TEST_CROP_SIZE": 64}, B200=eager)
    if cfg.MVIT.PATCH_2D:
        x = [torch.randn(batch, 3, 64, 64, generator=torch.Generator().manual_seed(3))]
    else:
        x = TO.synthetic_inputs(cfg, batch, 3)
    if name == "maskfeat":   # frames, meta, the loader's cube mask over the token frames
        tt = cfg.DATA.NUM_FRAMES // cfg.MVIT.PATCH_STRIDE[0]
        mask = torch.rand(batch, tt, 8, 8, generator=torch.Generator().manual_seed(4)) < 0.4
        x = [x[0], torch.Tensor(), mask.float()]
    torch.manual_seed(0)
    model = (B200MaskMViT if cfg.MODEL.MODEL_NAME == "MaskMViT" else _cls(cfg))(cfg)
    return model, batch, x, loss


# kernels of csrc/mvit_ops.cu outside namespace sfb: the row-slab merge of LayerNorm / colsum, the cls pass-through and
# the weight-gradient merge of the depthwise pooling
LIBRARY_FILE_SCOPE_KERNELS = ("partial_merge2_kernel", "dwpool_cls_kernel", "dwpool_wmerge_kernel")
FAMILY_NAMES = ["slowfast", "x3d", "mvit", "vit", "mae", "maskfeat", "mvitv2_t_image"]


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILY_NAMES)
def test_launch_counter_matches_the_device_activities_of_one_step(family, cuda_device):
    """``ops.launches()`` advances by exactly the number of device activities the library issues in one eager training
    step (forward, targets, backward).  The library's activities are its kernels - those in namespace ``sfb::`` and the
    three csrc/mvit_ops.cu defines at file scope (LIBRARY_FILE_SCOPE_KERNELS) - and its own ``cudaMemsetAsync`` /
    ``cudaMemset2DAsync`` calls (dwpool / dwconv weight gradients, gemm_batched split-K, zero_f32).  Memsets are told
    apart from any torch issues in the same step by the profiler's
    correlation of each device activity with the host op that was open when it was enqueued: torch's own memsets run
    inside an ``aten::`` op, the library's from a ctypes call that no ``aten::`` op encloses."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from slowfast_b200 import ops
    model, batch, x, loss_fn = _family(family)
    model = model.to(cuda_device).train()
    x = [t.to(cuda_device) for t in x]

    def step():
        model.zero_grad(set_to_none=True)
        loss_fn(model(x), batch).backward()

    step()  # warm-up: module loads and one-time kernel attributes
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        n0 = ops.launches()
        step()
        torch.cuda.synchronize()
        counted = ops.launches() - n0
    events = prof.events()
    device = [e for e in events if e.device_type == DeviceType.CUDA]
    kernels = collections.Counter(e.name for e in device
                                  if "sfb::" in e.name or e.name.split("(")[0] in LIBRARY_FILE_SCOPE_KERNELS)
    memsets = sum(1 for e in device if e.name.startswith("Memset"))
    torch_memsets = sum(1 for e in events if e.device_type == DeviceType.CPU and e.name.startswith("aten::")
                        for k in e.kernels if k.name.startswith("Memset"))
    issued = sum(kernels.values()) + memsets - torch_memsets
    print(f"{family}: counted {counted}, issued {issued} ({sum(kernels.values())} library kernels, {memsets - torch_memsets} "
          f"library memsets, {torch_memsets} torch memsets)")
    if counted != issued:
        for name, n in sorted(kernels.items()):
            print(f"  {n:5d}  {name[:160]}")
    assert counted == issued
