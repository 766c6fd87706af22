#!/usr/bin/env python
"""Device time of the FreiHAND scores (SURVEY.md §8 row f9), one JSON line:

  * FreiHANDEvaluator.update + compute over a FreiHAND-evaluation-sized set (3960 seeded samples, 21 keypoints and
    778 vertices each, metres), fed in batches of `--batch`;
  * f_scores at SMPL size: B=256 samples of 6890 vs 6890 points, float32, and the pairs per second it reaches
    (pairs = B n m; each pair is scored once for both directions);
  * the host baseline: oracle/freihand_oracle.py's float64 script loop on `--host-samples` of the 3960 samples and
    on `--host-smpl` of the SMPL-size samples, scaled to the full sets, with the CPU count;
  * the card's name and power limit, read in the same run.

CUDA events around `iters` calls after `warmup` calls; median of `reps` windows.

    python tools/time_freihand.py [--iters 5] [--warmup 2] [--reps 3] [--host-samples 200] [--host-smpl 2]
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

from oracle import freihand_oracle as fo  # noqa: E402
from pose2mesh_release_b200 import freihand as F  # noqa: E402


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
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--host-samples", type=int, default=200, help="FreiHAND-size samples of the host baseline")
    ap.add_argument("--host-smpl", type=int, default=2, help="SMPL-size samples of the host baseline")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_freihand.py measures on a GPU; none is available")
    rng = np.random.default_rng(3960)
    N = 3960
    gt_v = (rng.normal(0, 0.03, (N, 778, 3)) + rng.normal(0, 0.1, (N, 1, 3))).astype(np.float32)
    pred_v = (gt_v + rng.normal(0, 0.004, gt_v.shape)).astype(np.float32)
    gt_x, pred_x = gt_v[:, :21].copy(), pred_v[:, :21].copy()
    dev = torch.device("cuda:0")
    gx, gv, px, pv = (torch.from_numpy(a).to(dev) for a in (gt_x, gt_v, pred_x, pred_v))

    def evaluate():
        ev = F.FreiHANDEvaluator()
        for a in range(0, N, args.batch):
            ev.update(px[a:a + args.batch], pv[a:a + args.batch], gx[a:a + args.batch], gv[a:a + args.batch])
        return ev.compute()

    ev_ms = device_ms(evaluate, args.iters, args.warmup, args.reps)

    B, n = 256, 6890
    P = torch.randn((B, n, 3), device=dev) * 0.3
    Q = P + torch.randn((B, n, 3), device=dev) * 0.01
    fs_ms = device_ms(lambda: F.f_scores(P, Q), args.iters, args.warmup, args.reps)

    hs = args.host_samples
    t0 = time.perf_counter()
    fo.evaluate(gt_x[:hs], gt_v[:hs], pred_x[:hs], pred_v[:hs])
    host_eval_s = (time.perf_counter() - t0) * N / hs
    Ph, Qh = P[:args.host_smpl].cpu().numpy(), Q[:args.host_smpl].cpu().numpy()
    t0 = time.perf_counter()
    for b in range(len(Ph)):
        d = fo.nearest(Ph[b], Qh[b])
        for th in F.FSCORE_THRESHOLDS:
            fo.fscore_from_distances(*d, th)
    host_fs_s = (time.perf_counter() - t0) * B / len(Ph)
    print(json.dumps({"card": card(), "evaluator_samples": N, "evaluator_batch": args.batch,
                      "evaluator_ms": round(ev_ms, 3),
                      "f_scores_smpl_b256_ms": round(fs_ms, 3),
                      "f_scores_smpl_pairs_per_s": float(f"{B * n * n / (fs_ms * 1e-3):.4g}"),
                      "host_oracle_evaluator_s": round(host_eval_s, 2), "host_samples_timed": hs,
                      "host_oracle_f_scores_smpl_b256_s": round(host_fs_s, 1), "host_smpl_samples_timed": len(Ph),
                      "host_cpus": os.cpu_count()}))


if __name__ == "__main__":
    main()
