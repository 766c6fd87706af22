"""Timing aid (needs a GPU): PoseNet's train-mode forward + backward, the native path against the module's torch path.

    python tools/time_posenet_train.py [--iters 200] [--out DIR]

J = 17, H = 4096, two stages, p = 0.5, at B = 64 (the reference's default batch) and B = 256.  Both paths run in one
process, alternated round by round after a warm-up; every forward + backward is timed with device events.  Prints the
card's name and power limit, the median and range per path, and the per-kernel split of the native path from one
separate torch.profiler pass (the trace goes to --out when given)."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from pose2mesh_release_b200 import posenet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_posenet_train: no GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else
          torch.cuda.get_device_name(0) + " (power limit unknown)")
    torch.manual_seed(0)
    net = posenet.get_model(17, 4096, 2, 0.5).cuda().train()
    for B in (64, 256):
        x = torch.randn(B, 34, device="cuda")
        d_out = torch.randn(B, 51, device="cuda")

        def step(fwd):
            for prm in net.parameters():
                prm.grad = None
            fwd(x).backward(d_out)

        paths = {"native": net.forward_train_native, "torch": net._forward_torch}
        for fwd in paths.values():                       # warm-up: module loads, cuBLAS / cuDNN algorithm choice
            for _ in range(10):
                step(fwd)
        torch.cuda.synchronize()
        times = {k: [] for k in paths}
        for _ in range(args.iters):
            for k, fwd in paths.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step(fwd)
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
        for k, t in times.items():
            t = sorted(t)
            print(f"B={B:4d} {k:6s} forward+backward ms: median {t[len(t) // 2]:.3f}  min {t[0]:.3f}  max {t[-1]:.3f}"
                  f"  ({args.iters} iterations)")
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                step(net.forward_train_native)
            torch.cuda.synchronize()
        print(f"B={B}: kernels of 5 native forward+backward steps")
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=14, max_name_column_width=60))
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.out, f"posenet_train_B{B}.json"))


if __name__ == "__main__":
    main()
