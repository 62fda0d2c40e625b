"""The weight-gradient plan (sfb_conv_wgrad_plan) of every conv_wgrad launch of one SlowFast-8x8-R50 train step: tile
orientation and shape, split-K slices, useful / issued MMA work, last-wave fill and red.add bytes into dW.  Runs on a
CPU: the launch shapes come from the model's own conv units, walked in the order of its forward program.
Usage: python tests/probes/wgrad_plan.py [batch] [num_sms]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from slowfast_b200 import ops
from slowfast_b200.config import get_cfg
from slowfast_b200.engine import StemConvBN
from slowfast_b200.nets.resnet import B200SlowFast


def slowfast_wgrad_launches(batch=8):
    """[(name, x planes, dy planes, geom)] of the conv_wgrad calls of a SlowFast-8x8-R50 step (operands on the meta
    device: shapes only)."""
    cfg = get_cfg("SLOWFAST_8x8_R50", B200={"NSPLIT": 3, "CUDA_GRAPH": False})
    model = B200SlowFast(cfg)
    units = model._engine_units()
    crop, T, A = int(cfg.DATA.TRAIN_CROP_SIZE), cfg.DATA.NUM_FRAMES, cfg.SLOWFAST.ALPHA
    launches = []

    def conv(unit, dims):
        x = ops.alloc_planes(batch, *dims, unit.cin_pad, 1, "meta")
        geom = ops.fprop_geom(x, unit.k, unit.stride, unit.pad)
        if not isinstance(unit, StemConvBN):  # the stems' weight gradients run on their own kernels
            launches.append((unit.name, x, ops.alloc_planes(batch, *geom.out, unit.cout_pad, 1, "meta"), geom))
        return geom.out

    dims = []
    for p, t in enumerate((T // A, T)):
        st, sh, sw = conv(units[f"stem{p}"], (t, crop, crop))
        dims.append((st, ops.conv_out_size(sh, 3, 2, 1), ops.conv_out_size(sw, 3, 2, 1)))  # the stem's max pool
    conv(units["fuse1"], dims[1])
    for i in range(2, 6):
        stage = getattr(model, f"s{i}")
        for p in (0, 1):
            for blk in stage.blocks(p):
                u = blk.units()
                conv(u["c"], conv(u["b"], conv(u["a"], dims[p])))
                if "s" in u:
                    conv(u["s"], dims[p])
                dims[p] = blk.out_dims(*dims[p])
        if i < 5:
            conv(units[f"fuse{i}"], dims[1])
    return launches


def describe(x, dy, geom, plan, num_sms):
    """Useful and issued MMA work (GFLOP), last-wave fill and red.add bytes of one planned tensor-core launch."""
    m, taps = dy.rows, geom.k[0] * geom.k[1] * geom.k[2]
    useful = 2.0 * m * dy.c * taps * x.c / 1e9
    issued = 2.0 * plan.tiles * plan.tile_rows * plan.bn * 64 * plan.k_blocks / 1e9
    waves = -(-plan.ctas // num_sms)
    return dict(useful=useful, issued=issued, waves=waves, last_fill=(plan.ctas - (waves - 1) * num_sms) / num_sms,
                slot_use=plan.tiles * plan.k_blocks / (waves * num_sms * -(-plan.k_blocks // plan.slices)),
                red_bytes=4 * plan.slices * dy.c * taps * x.c)


def main():
    batch = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    num_sms = int(sys.argv[2]) if len(sys.argv) > 2 else 132
    tot = dict(useful=0.0, issued=0.0, red_bytes=0)
    print(f"{'layer':28s} {'M':>8s} {'cout':>5s} {'K':>6s}  tile          CK tiles slices ctas  use/iss last_wave  red MB")
    n_tc = 0
    for name, x, dy, geom in slowfast_wgrad_launches(batch):
        plan = ops.conv_wgrad_plan(x, dy, geom, nsplit=3, num_sms=num_sms)
        taps = geom.k[0] * geom.k[1] * geom.k[2]
        if plan.direct:
            print(f"{name:28s} {dy.rows:8d} {dy.c:5d} {taps * x.c:6d}  fp32 SIMT body")
            continue
        n_tc += 1
        r = describe(x, dy, geom, plan, num_sms)
        for k in tot:
            tot[k] += r[k]
        tile = f"{'T' if plan.transposed else 'C'} {plan.tile_rows:3d}x{plan.bn:<3d}"
        print(f"{name:28s} {dy.rows:8d} {dy.c:5d} {taps * x.c:6d}  {tile:12s} {plan.ck:3d} {plan.tiles:5d} {plan.slices:6d} "
              f"{plan.ctas:5d}  {r['useful'] / r['issued']:6.3f} {r['last_fill']:9.2f} {r['red_bytes'] / 1e6:7.1f}")
    print(f"{n_tc} tensor-core launches: useful {tot['useful']:.1f} GFLOP, issued {tot['issued']:.1f} GFLOP "
          f"(ratio {tot['useful'] / tot['issued']:.3f}), red.add {tot['red_bytes'] / 1e9:.3f} GB")


if __name__ == "__main__":
    main()
