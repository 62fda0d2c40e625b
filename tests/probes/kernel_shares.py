"""Per-kernel share of one eager SlowFast train step (CUDA graphs off), from torch.profiler's CUDA activities.
Writes OUT_DIR/kernel_shares_b{B}_n{nsplit}.json (default: the current directory).
Usage: python tests/probes/kernel_shares.py [batch] [nsplit] [OUT_DIR]"""
import json, os, re, sys
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from slowfast_b200.config import get_cfg
from slowfast_b200.nets.resnet import B200SlowFast

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
nsplit = int(sys.argv[2]) if len(sys.argv) > 2 else 3
out_dir = sys.argv[3] if len(sys.argv) > 3 else "."
cfg = get_cfg("SLOWFAST_8x8_R50", B200={"NSPLIT": nsplit, "CUDA_GRAPH": False})
torch.manual_seed(0)
model = B200SlowFast(cfg).cuda().train()
T, A = cfg.DATA.NUM_FRAMES, cfg.SLOWFAST.ALPHA
clip = torch.randn(B, 3, T, 224, 224, device="cuda")
idx = torch.linspace(0, T - 1, T // A).long().cuda()
x = [clip.index_select(2, idx).contiguous(), clip]
y = torch.randint(0, 400, (B,), device="cuda")


def step():
    model.zero_grad(set_to_none=True)
    F.cross_entropy(model(x), y).backward()


for _ in range(3):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()


def kernel_class(name):
    """Template arguments and parameter lists stripped: 'void sfb::conv_igemm_kernel<3>(sfb::ConvParams)' ->
    'conv_igemm_kernel'."""
    n = re.sub(r"^void ", "", name)
    n = n.split("(")[0]
    n = re.sub(r"<.*>$", "", n)
    return n.split("::")[-1]


agg = {}
for ev in prof.events():
    if ev.device_type != torch.autograd.DeviceType.CUDA:
        continue
    k = kernel_class(ev.name)
    a = agg.setdefault(k, dict(us=0.0, launches=0))
    a["us"] += ev.time_range.elapsed_us()
    a["launches"] += 1
total = sum(a["us"] for a in agg.values())
rows = sorted(([k, a["us"], a["launches"]] for k, a in agg.items()), key=lambda r: -r[1])
out = dict(batch=B, nsplit=nsplit, device=torch.cuda.get_device_name(), cuda_us_per_step=total,
           kernels=[dict(kernel=k, us=round(us, 1), launches=n, share=round(us / total, 4)) for k, us, n in rows])
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, f"kernel_shares_b{B}_n{nsplit}.json"), "w") as f:
    json.dump(out, f, indent=1)
print(f"CUDA time per step {total / 1e3:.2f} ms")
for k, us, n in rows[:15]:
    print(f"  {us / total * 100:5.1f} %  {us / 1e3:8.2f} ms  {n:5d}  {k}")
