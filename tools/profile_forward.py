"""Per-kernel device time of one eval forward of the bench workload (B=256 SMPL-size meshes, fp16x3), from
torch.profiler with CUDA activities: kernel name, launches, total time and share of the forward's kernel time.
Usage: python tools/profile_forward.py [--batch 256] [--iters 5] [--trace DIR]  (times are per forward, averaged over
--iters profiled forwards after two warm-up ones; --trace also writes a chrome trace under DIR)."""
import argparse
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from pose2mesh_release_b200.meshnet import Pose2Mesh  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--trace", default=None)
args = ap.parse_args()

graph_L, perm_rev = bench.build_problem("smpl")
torch.manual_seed(123)
model = Pose2Mesh(5, 3, graph_L, joint_set="human36")
model.load_state_dict(bench.randomize_bn_({k: v.clone() for k, v in model.state_dict().items()}))
model = model.cuda().set_precision("fp16x3").eval()
x = torch.randn(args.batch, 17, 5, generator=torch.Generator().manual_seed(1000)).cuda()
with torch.no_grad():
    for _ in range(2):
        model(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            model(x)
        torch.cuda.synchronize()

tot = defaultdict(float)
cnt = defaultdict(int)
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        name = e.name if len(e.name) < 90 else e.name[:87] + "..."
        tot[name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        cnt[name] += 1
all_us = sum(tot.values())
print(f"{torch.cuda.get_device_name(0)}; eval forward B={args.batch}: {all_us / args.iters / 1e3:.3f} ms of kernel time "
      f"per forward")
print(f"{'kernel':90s} {'launches':>8s} {'ms':>8s} {'share':>6s}")
for name, us in sorted(tot.items(), key=lambda kv: -kv[1]):
    print(f"{name:90s} {cnt[name] // args.iters:8d} {us / args.iters / 1e3:8.3f} {100 * us / all_us:5.1f}%")
if args.trace:
    os.makedirs(args.trace, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.trace, "forward.pt.trace.json"))
