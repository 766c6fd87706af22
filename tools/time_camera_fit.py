#!/usr/bin/env python
"""Time the demo's camera fit on the GPU: the native one-launch fit (pose2mesh_release_b200.camera.fit_cameras) at
B in {1, 16, 256}, against the reference's loop restated in torch ops on the same GPU at B = 1 (OptimzeCamLayer,
lib/models/project_net.py, with torch.optim.Adam at its default settings and the demo's 1500 steps and lr schedule,
demo/run.py:161-189).  Seeded synthetic poses; prints one JSON line.

    python tools/time_camera_fit.py [--repeats 5]

Each time is the median over `repeats` runs.  A native run is CUDA events around back-to-back calls after a warm-up
(at least --min-seconds of work); a torch-loop run is one full 1500-step fit timed by the host clock and ended with a
device synchronise, as the demo runs it.  The card's name, power limit and SM clock limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pose2mesh_release_b200.camera import LR_SCHEDULE, N_ITER, fit_cameras  # noqa: E402


def device_ms(fn, min_seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    iters = 4
    while True:
        beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        beg.record()
        for _ in range(iters):
            fn()
        end.record()
        end.synchronize()
        total = beg.elapsed_time(end)
        if total >= 1000.0 * min_seconds:
            return total / iters
        iters *= 2


def gpu_query(field):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


class OptimzeCamLayer(torch.nn.Module):
    """lib/models/project_net.py:7-17."""

    def __init__(self, crop_size):
        super().__init__()
        self.img_res = crop_size / 2
        self.cam_param = torch.nn.Parameter(torch.rand((1, 3)))

    def forward(self, pose3d):
        output = pose3d[:, :, :2] + self.cam_param[None, :, 1:]
        return output * self.cam_param[None, :, :1] * self.img_res + self.img_res


def torch_loop(pred_3d_joint, target_joint):
    """demo/run.py:161-189 for one person."""
    project_net = OptimzeCamLayer(500).to(pred_3d_joint.device)
    criterion = torch.nn.L1Loss()
    optimizer = torch.optim.Adam(project_net.parameters(), lr=0.1)
    project_net.train()
    for j in range(0, 1500):
        loss = criterion(project_net(pred_3d_joint.detach()), target_joint[:, :17, :])
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        if j == 500:
            for g in optimizer.param_groups:
                g["lr"] = 0.05
        if j == 1000:
            for g in optimizer.param_groups:
                g["lr"] = 0.001
    return project_net.cam_param


def synthetic(B, seed):
    g = np.random.default_rng(seed)
    p3d = g.normal(0, 0.3, (B, 17, 3)).astype(np.float32)
    s, t = g.uniform(0.6, 1.3, (B, 1, 1)), g.normal(0, 0.1, (B, 1, 2))
    px = (p3d[:, :, :2] + t) * s * g.uniform(80, 300, (B, 1, 1)) + g.uniform(100, 600, (B, 1, 2))
    return px + g.normal(0, 3, (B, 17, 2)), p3d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_camera_fit.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    native = {}
    for B in (1, 16, 256):
        px, p3d = synthetic(B, B)
        x, p = torch.from_numpy(px).to(dev), torch.from_numpy(p3d).to(dev)
        init = torch.rand((B, 3)).to(dev)
        runs = [device_ms(lambda: fit_cameras(x, p, init=init, n_iter=N_ITER, lr_schedule=LR_SCHEDULE),
                          args.min_seconds) for _ in range(args.repeats)]
        native[f"B{B}"] = {"median_ms": round(statistics.median(runs), 4), "runs_ms": [round(r, 4) for r in runs]}
    px, p3d = synthetic(1, 1)
    x, p = torch.from_numpy(px).to(dev), torch.from_numpy(p3d).to(dev)
    target = fit_cameras(x, p, init=torch.rand((1, 3)).to(dev), n_iter=0)["target"]      # the same crop target
    torch_loop(p, target)                                                                 # warm-up
    torch.cuda.synchronize()
    runs = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        torch_loop(p, target)
        torch.cuda.synchronize()
        runs.append(1e3 * (time.perf_counter() - t0))
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(dev), "power_limit": gpu_query("power.limit"),
        "sm_clock_max": gpu_query("clocks.max.sm"), "n_iter": N_ITER, "native_fit": native,
        "torch_loop_b1": {"median_ms": round(statistics.median(runs), 2), "runs_ms": [round(r, 2) for r in runs]},
        "host_cpus": os.cpu_count(), "torch": torch.__version__,
    }))


if __name__ == "__main__":
    main()
