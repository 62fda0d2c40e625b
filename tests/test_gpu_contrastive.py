"""MoCo on the engine (GPU): the in-place momentum update, the MLPHead projection, one MoCo step against the unmodified
reference ContrastiveModel, and CUDA-graph replay across steps.

Bounds: logits / losses 1e-3 relative with argmax exact and parameter gradients median < 0.2, max < 0.5, cosine > 0.9
(the reference comparison of test_gpu_models.py); fast mode (bf16 operands) logits 0.2; the key-encoder update bitwise."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

MOCO = "contrastive_ssl/MoCo_SlowR50_8x8.yaml"
BATCH, CROP, FRAMES = 4, 64, 8
# one GPU, a small clip, a queue that the 4 views x 4 clips of a step divide, a small kNN memory
SHRUNK = ["NUM_GPUS", 1, "DATA.TRAIN_CROP_SIZE", CROP, "DATA.TEST_CROP_SIZE", CROP, "DATA.NUM_FRAMES", FRAMES,
          "CONTRASTIVE.QUEUE_LEN", 64, "CONTRASTIVE.LENGTH", 16, "TRAIN.BATCH_SIZE", BATCH]


def _refshim():
    from oracle import refshim
    if not refshim.reference_available():
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    refshim.install()
    return refshim


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------ momentum update
ANNEALED = [1 - (1 - 0.994) * (math.cos(math.pi * e / 200) + 1.0) * 0.5 for e in (0.0, 0.37, 57.1, 199.9)]


@pytest.mark.parametrize("m", [0.0, 0.5, 0.994, 0.999] + ANNEALED)
def test_momentum_update_is_bitwise_the_reference_expression(m, cuda_device):
    from slowfast_b200 import ops
    g = torch.Generator(device=cuda_device).manual_seed(3)
    shapes = [(1,), (7,), (8191,), (8192,), (8193,), (100003,), (3, 5, 7), (64, 3, 1, 7, 7)]
    qs = [torch.randn(s, device=cuda_device, generator=g) for s in shapes]
    ks = [torch.randn(s, device=cuda_device, generator=g) * 3 for s in shapes]
    want = [q * (1.0 - m) + k * m for q, k in zip(qs, ks)]
    ptrs = [k.data_ptr() for k in ks]
    n0 = ops.launches()
    ops.momentum_update(ops.momentum_table(list(zip(qs, ks))), m)
    assert ops.launches() - n0 == 1
    torch.cuda.synchronize()
    assert [k.data_ptr() for k in ks] == ptrs
    for k, w in zip(ks, want):
        assert torch.equal(k, w)


# ------------------------------------------------------------------------------------------------ MLP head
def _mlp_model(refshim, cuda_device, layers=3):
    from oracle import torch_oracle as TO
    from slowfast_b200.nets.resnet_single import B200ResNet
    cfg = refshim.load_cfg("Kinetics/SLOW_8x8_R50.yaml", ["CONTRASTIVE.NUM_MLP_LAYERS", layers, "MODEL.NUM_CLASSES", 128,
                                                          "MODEL.HEAD_ACT", "none", "MODEL.DROPOUT_RATE", 0.0,
                                                          "DATA.TRAIN_CROP_SIZE", CROP, "DATA.NUM_FRAMES", FRAMES])
    model = B200ResNet(cfg)
    model.load_state_dict(TO.fixture_state(model.state_dict(), 3))
    model.cuda_graphs = False
    return cfg, model.to(cuda_device)


def _mlp64(x, lins):
    h = x.double()
    for i, lin in enumerate(lins):
        h = h @ lin.weight.double().t() + lin.bias.double()
        if i < len(lins) - 1:
            h = torch.relu(h)
    return h


def test_mlp_head_training_path_matches_fp64(cuda_device):
    refshim = _refshim()
    from oracle import torch_oracle as TO
    cfg, model = _mlp_model(refshim, cuda_device)
    model.train()
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, BATCH, 4)]
    logits = model(x)
    pooled = model._head_saved[1][0].clone()
    lins = model.head.linears()
    assert [lin.out_features for lin in lins] == [2048, 2048, 128]
    dlogits = torch.randn(logits.shape, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    logits.backward(dlogits)
    dpooled = model.ctx._bufs[("head.dpooled",)].clone()
    torch.cuda.synchronize()
    p64 = pooled.double().requires_grad_(True)
    w64 = [(lin.weight.detach().double().requires_grad_(True), lin.bias.detach().double().requires_grad_(True))
           for lin in lins]
    h = p64
    for i, (w, b) in enumerate(w64):
        h = h @ w.t() + b
        if i < len(w64) - 1:
            h = torch.relu(h)
    h.backward(dlogits.double())
    assert _rel(logits.detach(), h.detach()) < 1e-5
    assert _rel(dpooled, p64.grad) < 1e-5
    for lin, (w, b) in zip(lins, w64):
        assert _rel(lin.weight.grad, w.grad) < 1e-5 and _rel(lin.bias.grad, b.grad) < 1e-5


def test_mlp_head_windowed_eval_matches_fp64(cuda_device):
    """Test crop larger than the train pool: the MLP runs per window, then the group mean (HEAD_ACT none)."""
    refshim = _refshim()
    from oracle import torch_oracle as TO
    cfg, model = _mlp_model(refshim, cuda_device)
    model.eval()
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, BATCH, 4, crop=96)]   # 3x3 map, 2x2 pool: 4 windows
    with torch.no_grad():
        out = model(x)
    pooled = model.ctx._bufs[("head.pooled.win",)]
    g = pooled.shape[0] // BATCH
    assert g == 4
    want = _mlp64(pooled, model.head.linears()).view(BATCH, g, -1).mean(1)
    assert _rel(out, want) < 1e-5


# ------------------------------------------------------------------------------------------------ one MoCo step
def _moco_models(cuda_device, fast=False, extra=(), start_iter=1):
    refshim = _refshim()
    from oracle import torch_oracle as TO
    from slowfast_b200.nets.contrastive import B200ContrastiveModel
    cfg = refshim.load_cfg(MOCO, SHRUNK + list(extra))
    ref = refshim.build_reference_model(cfg)
    sd = ref.state_dict()
    # fixture weights: query encoder seed 3, key encoder seed 4.  start_iter 1: the EMA mixes two different nets;
    # start_iter 0: the key encoder is first overwritten with the query encoder, then the EMA runs
    q = TO.fixture_state({k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}, 3)
    kk = TO.fixture_state({k[len("backbone_hist."):]: v for k, v in sd.items() if k.startswith("backbone_hist.")}, 4)
    sd.update({"backbone." + k: v for k, v in q.items()})
    sd.update({"backbone_hist." + k: v for k, v in kk.items()})
    sd["iter"] = torch.full_like(sd["iter"], start_iter)
    ref.load_state_dict(sd)
    if fast:
        cfg["B200"] = {"NSPLIT": 1}
    mine = B200ContrastiveModel(cfg)
    mine.load_state_dict({k: v.cpu() for k, v in sd.items()})
    return cfg, ref.to(cuda_device).train(), mine.to(cuda_device).train()


def _clips(cfg, cuda_device, seed=0):
    from oracle import torch_oracle as TO
    return [[t.to(cuda_device) for t in TO.synthetic_inputs(cfg, BATCH, 10 + seed * 4 + i)] for i in range(4)]


def _step(model, cfg, clips, epoch_exact=3.7):
    """contrastive_forward (SEQUENTIAL: 4 key forwards, then forward + backward per query clip, then the enqueue) with
    the batch-shuffle permutation drawn from the same seed for both models."""
    from slowfast.models.contrastive import contrastive_forward

    class _NoScale:
        @staticmethod
        def scale(loss):
            return loss

    index = torch.arange(BATCH, device=clips[0][0].device)
    time = torch.zeros(BATCH, len(clips), 1, device=clips[0][0].device)
    torch.manual_seed(17)
    _, preds, loss, _ = contrastive_forward(model, cfg, clips, index, time, epoch_exact, _NoScale())
    torch.cuda.synchronize()
    return preds.detach(), loss.detach()


def _bn_stats(model, prefix):
    return {k: v for k, v in model.state_dict().items()
            if k.startswith(prefix) and (k.endswith("running_mean") or k.endswith("running_var"))}


@pytest.mark.parametrize("fast,start_iter", [(False, 1), (False, 0), (True, 1)], ids=["parity", "parity-iter0", "fast"])
def test_moco_step_matches_reference(fast, start_iter, cuda_device):
    cfg, ref, mine = _moco_models(cuda_device, fast, start_iter=start_iter)
    clips = _clips(cfg, cuda_device)
    pr, lr = _step(ref, cfg, [[t.clone() for t in c] for c in clips])
    pm, lm = _step(mine, cfg, clips)
    rel = ((pm - pr).abs().max() / pr.abs().max()).item()
    if fast:
        assert _rel(pm, pr) < 0.2
        return
    assert rel < 1e-3 and torch.equal(pm.argmax(1), pr.argmax(1)), rel
    assert abs(lm.item() - lr.item()) / abs(lr.item()) < 1e-3
    rp = dict(ref.named_parameters())
    per = {k: _rel(p.grad, rp[k].grad) for k, p in mine.named_parameters() if k.startswith("backbone.")}
    rels = sorted(per.values())
    cos = min(torch.nn.functional.cosine_similarity(p.grad.double().flatten(), rp[k].grad.double().flatten(),
                                                    dim=0).item()
              for k, p in mine.named_parameters() if k.startswith("backbone."))
    assert rels[len(rels) // 2] < 0.2 and rels[-1] < 0.5 and cos > 0.9, (rels[len(rels) // 2], rels[-1], cos)
    assert not any(p.grad is not None for p in mine.backbone_hist.parameters())
    # the key encoder after the momentum update: bitwise the reference's
    for k, p in mine.backbone_hist.named_parameters():
        assert torch.equal(p, rp["backbone_hist." + k]), k
    assert mine.mmt == ref.mmt and int(mine.iter) == int(ref.iter) == start_iter + 1
    assert torch.equal(mine.ptr, ref.ptr)
    assert _rel(mine.queue_x, ref.queue_x) < 1e-3
    for prefix in ("backbone.", "backbone_hist."):
        sr, sm = _bn_stats(ref, prefix), _bn_stats(mine, prefix)
        assert sr.keys() == sm.keys() and sr
        worst = max(_rel(sm[k], sr[k]) for k in sr)
        assert worst < 1e-2, (prefix, worst)


def test_moco_replay_matches_eager_without_recapture(cuda_device):
    """Five MoCo steps (with an SGD update between them) with CUDA graphs and twice eagerly: the replayed run stays
    within the eager runs' own spread, and after the first step neither encoder captures a new program - the
    in-place momentum update keeps every pointer the programs hold."""
    runs = {}
    programs = []
    for name, graphs in (("eager_a", False), ("eager_b", False), ("graphs", True)):
        cfg, _, mine = _moco_models(cuda_device)
        for enc in (mine.backbone, mine.backbone_hist):
            enc.cuda_graphs = graphs
        opt = torch.optim.SGD([p for p in mine.parameters() if p.requires_grad], lr=0.05)
        out = []
        for step in range(5):
            opt.zero_grad(set_to_none=True)
            pm, _ = _step(mine, cfg, _clips(cfg, cuda_device, step), epoch_exact=step * 0.5)
            opt.step()
            out.append(pm)
            if graphs:
                programs.append({id(p) for enc in (mine.backbone, mine.backbone_hist) for p in enc._graphs.values()})
        runs[name] = out
    assert programs[0] and all(p == programs[0] for p in programs[1:])
    for s in range(5):
        spread = _rel(runs["eager_b"][s], runs["eager_a"][s])
        got = _rel(runs["graphs"][s], runs["eager_a"][s])
        assert got <= max(4 * spread, 1e-5), (s, got, spread)


def test_moco_knn_eval_at_the_test_crop_matches_reference(cuda_device):
    """Eval at a test crop larger than the train crop (the recipe: 256 against 224), as test_net's kNN evaluation runs
    it: inside ContrastiveModel the backbone head pools globally (adaptive 1x1x1), then the MLP; the returned kNN
    similarities and neighbours must match the reference's."""
    cfg, ref, mine = _moco_models(cuda_device, extra=["CONTRASTIVE.LENGTH", 256])   # kNN takes the top 200
    ref.eval()
    mine.eval()
    from oracle import torch_oracle as TO
    x = [t.to(cuda_device) for t in TO.synthetic_inputs(cfg, BATCH, 7, crop=96)]   # 3x3 feature map, train pool 2x2
    index = torch.arange(BATCH, device=cuda_device)
    tm = torch.zeros(BATCH, 1, 1, device=cuda_device)
    with torch.no_grad():
        fr = ref.backbone([t.clone() for t in x])
        fm = mine.backbone(x)
        yd_r, yi_r = ref(x, index, tm)
        yd_m, yi_m = mine(x, index, tm)
    torch.cuda.synchronize()
    assert fm.shape == fr.shape == (BATCH, 128)
    assert ((fm - fr).abs().max() / fr.abs().max()).item() < 1e-3
    assert yd_m.shape == yd_r.shape == (BATCH, 200)
    assert ((yd_m - yd_r).abs().max()).item() < 1e-3
    assert torch.equal(yi_m[:, 0], yi_r[:, 0])


# ------------------------------------------------------------------------------------------------ unmodified drivers
N_TRAIN, N_VAL, DBATCH = 200, 16, 8   # kNN eval takes the top 200 of the memory (contrastive.py:227): >= 200 videos


def _register_moco_dataset():
    from slowfast.datasets import utils as dsutils
    from slowfast.datasets.build import DATASET_REGISTRY
    if "Mocosynthetic" in DATASET_REGISTRY._obj_map:
        return

    class Mocosynthetic(torch.utils.data.Dataset):
        """Seeded clips shaped as kinetics.py yields them for ContrastiveModel (kinetics.py:364-464): in train mode
        TRAIN_CROP_NUM_TEMPORAL clips, each packed per pathway, one label / index per video, time of shape
        [clips, 1]; in val / test mode one packed clip.  ``_labels`` is what init_knn_labels reads."""

        def __init__(self, cfg, mode, num_retries=0):
            self.cfg, self.mode = cfg, mode
            self._n = N_TRAIN if mode == "train" else N_VAL
            self._labels = [i % 7 for i in range(self._n)]

        @property
        def num_videos(self):
            return self._n

        def __len__(self):
            return self._n

        def __getitem__(self, i):
            cfg = self.cfg
            n_clips = cfg.DATA.TRAIN_CROP_NUM_TEMPORAL if self.mode == "train" else 1
            crop = cfg.DATA.TRAIN_CROP_SIZE if self.mode == "train" else cfg.DATA.TEST_CROP_SIZE
            g = torch.Generator().manual_seed(7919 * i + {"train": 1, "val": 2, "test": 3}[self.mode])
            clips = [dsutils.pack_pathway_output(cfg, torch.randn(3, cfg.DATA.NUM_FRAMES, crop, crop, generator=g))
                     for _ in range(n_clips)]
            frames = clips[0] if n_clips == 1 else clips
            return frames, self._labels[i], i, torch.zeros(n_clips, 1), {}

    DATASET_REGISTRY._do_register("Mocosynthetic", Mocosynthetic)


def test_moco_through_the_unmodified_driver_then_finetune(cuda_device, tmp_path):
    """tools/train_net.train on a shrunk MoCo_SlowR50_8x8.yaml (contrastive_forward, contrastive_parameter_surgery,
    init_knn_labels, the kNN eval of eval_epoch, save_checkpoint) with the engine and with the stock model: losses within
    test_gpu_drivers.py's bounds.  Then the engine's checkpoint fine-tunes finetune_ucf_Slow_R50_syn0.yaml on the engine
    with CHECKPOINT_CLEAR_NAME_PATTERN ("backbone.",): every backbone tensor it loads equals the checkpoint's."""
    import glob

    import driver_harness as H
    if H.setup_reference() is None:
        pytest.skip("no reference tree (build() copies it into oracle/_ref)")
    _register_moco_dataset()
    import slowfast.utils.checkpoint as cu
    over = ["TRAIN.DATASET", "mocosynthetic", "TEST.DATASET", "mocosynthetic", "DATA.NUM_FRAMES", FRAMES,
            "DATA.TEST_CROP_SIZE", 96, "CONTRASTIVE.QUEUE_LEN", 64, "CONTRASTIVE.LENGTH", N_TRAIN,
            "TRAIN.MIXED_PRECISION", False, "SOLVER.WARMUP_EPOCHS", 0.0]
    recs = {}
    try:
        for engine in (False, True):
            H.use_engine(engine)
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            out = tmp_path / ("engine" if engine else "stock")
            out.mkdir()
            cfg = H.driver_cfg(MOCO, 1, over, out_dir=str(out), batch=DBATCH, crop=CROP)
            from slowfast.models import build_model
            assert type(build_model(cfg)).__name__ == ("B200ContrastiveModel" if engine else "ContrastiveModel")
            recs[engine], _ = H.run_train(cfg)
        en, st = recs[True], recs[False]
        assert len(en["train"]) == len(st["train"]) == N_TRAIN // DBATCH
        for i, (a, b) in enumerate(zip(en["train"], st["train"])):
            rel = abs(a["loss"] - b["loss"]) / abs(b["loss"])
            assert rel < (1e-3 if i == 0 else 1e-2), (i, a["loss"], b["loss"])
        assert len(en["val"]) == len(st["val"]) == N_VAL // DBATCH    # the kNN evaluation ran

        ckpt = sorted(glob.glob(str(tmp_path / "engine" / "checkpoints" / "*.pyth")))[-1]
        saved = torch.load(ckpt, map_location="cpu", weights_only=False)["model_state"]
        loaded = {}
        orig = cu.load_checkpoint

        def recording_load(path, model, *a, **k):
            epoch = orig(path, model, *a, **k)
            loaded.update({n: v.detach().cpu().clone() for n, v in getattr(model, "module", model).state_dict().items()})
            return epoch

        cu.load_checkpoint = recording_load
        (tmp_path / "finetune").mkdir()
        try:
            H.use_engine(True)
            ft = H.driver_cfg("contrastive_ssl/finetune_ucf_Slow_R50_syn0.yaml", 1,
                              ["TRAIN.DATASET", "synthetic", "TEST.DATASET", "synthetic", "DATA.NUM_FRAMES", FRAMES,
                               "MODEL.DROPOUT_RATE", 0.0, "TRAIN.CHECKPOINT_FILE_PATH", ckpt],
                              out_dir=str(tmp_path / "finetune"), batch=4, crop=CROP)
            from slowfast.models import build_model
            assert type(build_model(ft)).__name__ == "B200ResNet"
            H.run_train(ft)
        finally:
            cu.load_checkpoint = orig
        matched = [k for k in loaded if "backbone." + k in saved and saved["backbone." + k].shape == loaded[k].shape]
        assert len([k for k in matched if not k.startswith("head.")]) == \
            len([k for k in saved if k.startswith("backbone.") and not k.startswith("backbone.head.")])
        for k in matched:
            assert torch.equal(loaded[k], saved["backbone." + k]), k
    finally:
        H.use_engine(False)
