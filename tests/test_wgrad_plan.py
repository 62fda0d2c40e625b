"""CPU: the weight-gradient tiling (sfb_conv_wgrad_plan) of every tensor-core conv_wgrad launch of a SlowFast-8x8-R50
step at batch 8 on a 132-SM H100 keeps the tensor cores on useful work, fills its waves, and adds no more red.add
traffic into dW than the 128-row tiling with the 2 x SMs / tiles split it replaces."""
import importlib.util
import os

import pytest

NUM_SMS = 132


def _launches():
    path = os.path.join(os.path.dirname(__file__), "probes", "wgrad_plan.py")
    spec = importlib.util.spec_from_file_location("wgrad_plan_probe", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, mod.slowfast_wgrad_launches(8)


def _previous_red_bytes(x, dy, geom):
    """red.add bytes of the previous plan: cout in 128-row tiles, up to 128 (tap, ci) columns, 2 x SMs / tiles slices."""
    taps = geom.k[0] * geom.k[1] * geom.k[2]
    ck = 64 if x.c % 64 == 0 else 32 if x.c % 32 == 0 else 16 if x.c % 16 == 0 else 8
    n_chunks = taps * x.c // ck
    ng = min(n_chunks, 128 // ck)
    ng += (ng * ck) % 16 != 0
    tiles = -(-n_chunks // ng) * -(-dy.c // 128)
    k_blocks = -(-dy.rows // 64)
    splits = min(max(1, 2 * NUM_SMS // tiles), max(1, k_blocks // 4))
    per = -(-k_blocks // splits)
    return 4 * -(-k_blocks // per) * dy.c * taps * x.c


def test_slowfast_wgrad_plan_targets():
    from slowfast_b200 import ops
    probe, launches = _launches()
    useful = issued = red = red_before = 0.0
    n_tc = 0
    for name, x, dy, geom in launches:
        plan = ops.conv_wgrad_plan(x, dy, geom, nsplit=3, num_sms=NUM_SMS)
        if plan.direct:
            continue
        n_tc += 1
        r = probe.describe(x, dy, geom, plan, NUM_SMS)
        assert r["useful"] / r["issued"] >= 0.7, (name, r)
        assert r["slot_use"] >= 0.85, (name, r)
        assert plan.k_blocks // plan.slices >= 4 or plan.slices == 1, (name, plan.k_blocks, plan.slices)
        assert plan.ctas == plan.tiles * plan.slices
        useful += r["useful"]
        issued += r["issued"]
        red += r["red_bytes"]
        red_before += _previous_red_bytes(x, dy, geom)
    assert n_tc == 97
    assert useful / issued >= 0.9
    assert red <= red_before


@pytest.mark.parametrize("cout,c,k,expect", [
    (16, 16, (1, 3, 3), (1, 64, 16)),     # narrow output: (tap, ci) rows, cout columns
    (64, 64, (1, 3, 3), (0, 64, 128)),    # 64 output channels: one warpgroup's rows, the positions split between two
    (512, 512, (1, 3, 3), (0, 128, 128)),
])
def test_plan_orientation(cout, c, k, expect):
    from slowfast_b200 import ops
    x = ops.alloc_planes(8, 8, 56, 56, c, 1, "meta")
    geom = ops.fprop_geom(x, k, (1, 1, 1), tuple(kk // 2 for kk in k))
    dy = ops.alloc_planes(8, *geom.out, cout, 1, "meta")
    plan = ops.conv_wgrad_plan(x, dy, geom, nsplit=1, num_sms=NUM_SMS)
    assert (plan.transposed, plan.tile_rows, plan.bn) == expect


def test_plan_rejects_bad_descriptors():
    from slowfast_b200 import lib as L
    from slowfast_b200 import ops
    x = ops.alloc_planes(1, 1, 8, 8, 12, 1, "meta")
    geom = ops.fprop_geom(x, (1, 1, 1), (1, 1, 1), (0, 0, 0))
    dy = ops.alloc_planes(1, *geom.out, 16, 1, "meta")
    with pytest.raises(L.NativeLibraryError, match="multiples of 8"):
        ops.conv_wgrad_plan(x, dy, geom, nsplit=1, num_sms=NUM_SMS)
    x = ops.alloc_planes(1, 1, 8, 8, 16, 1, "meta")
    with pytest.raises(L.NativeLibraryError, match="num_sms"):
        ops.conv_wgrad_plan(x, dy, geom, nsplit=1, num_sms=0)
