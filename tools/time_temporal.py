#!/usr/bin/env python
"""Device time of the temporal metrics (SURVEY.md §8 row f8), one JSON line:

  * evaluate_video on a seeded 3DPW-sized set (37 videos, about 35 k frames, 14 joints, float32, smoothed);
  * smooth_sequences on 1000 SMPL-mesh frames (4 sequences of 250 frames x 6890 x 3, float32);
  * the host baseline: oracle/temporal_oracle.py's float64 per-video loop (numpy) on the same 3DPW-sized set;
  * the card's name and power limit, read in the same run.

CUDA events around `iters` calls after `warmup` calls; median of `reps` windows.

    python tools/time_temporal.py [--iters 20] [--warmup 5] [--reps 5] [--host-videos 37]
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

from oracle import temporal_oracle as to  # noqa: E402
from pose2mesh_release_b200 import temporal as T  # noqa: E402


def device_ms(fn, iters, warmup, reps):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-videos", type=int, default=37, help="videos of the host baseline (all 37 by default)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_temporal.py measures on a GPU; none is available")
    rng = np.random.default_rng(2026)
    lengths = rng.integers(600, 1300, 37)
    lengths = (lengths * 35000 / lengths.sum()).astype(np.int64)
    n = int(lengths.sum())
    gt = (rng.standard_normal((1, 14, 3)) * 300 + np.cumsum(rng.standard_normal((n, 14, 3)) * 8, 0)).astype(np.float32)
    pred = (gt + rng.standard_normal(gt.shape) * 40).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(lengths)])
    videos = [np.arange(off[i], off[i + 1]) for i in range(37)]
    dev = torch.device("cuda:0")
    g, p = torch.from_numpy(gt).to(dev), torch.from_numpy(pred).to(dev)
    ev_ms = device_ms(lambda: T.evaluate_video(p, g, videos), args.iters, args.warmup, args.reps)

    mesh = torch.randn((1000, 6890, 3), device=dev).cumsum(0)
    sm_ms = device_ms(lambda: T.smooth_sequences(mesh, [250] * 4, 0.004, 0.7), args.iters, args.warmup, args.reps)

    hv = videos[:args.host_videos]
    t0 = time.perf_counter()
    to.evaluate_video_f64(pred, gt, hv)
    host_s = (time.perf_counter() - t0) * 37 / len(hv)
    print(json.dumps({"card": card(), "frames": n, "videos": 37, "joints": 14,
                      "evaluate_video_ms": round(ev_ms, 4), "smooth_smpl_1000_frames_ms": round(sm_ms, 4),
                      "host_oracle_loop_s": round(host_s, 3), "host_videos_timed": len(hv)}))


if __name__ == "__main__":
    main()
