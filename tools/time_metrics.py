#!/usr/bin/env python
"""Time the evaluation metrics on the GPU against the reference's host-side numpy evaluation, at configs[1]'s size:
B = 256 SMPL meshes (6890 vertices), the 17-joint H36M regressor (tests/golden/eval_metrics.npz) and a seeded 24-joint
mesh regressor.  Seeded inputs; prints one JSON line.

    python tools/time_metrics.py [--min-seconds 1.0]

Device times come from CUDA events around >= min_seconds of back-to-back calls after a warm-up.  compute_both_err
includes its one host synchronisation (reading back the two means).  The host times are the oracle's float64 restatement of
the reference's per-sample evaluate loop (oracle/metrics_oracle.py, reference order of operations, with PA-MPVPE) and
its compute_both_err, on the same data already on the host (the reference also pays the device-to-host copies).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import metrics_oracle as mo  # noqa: E402
from pose2mesh_release_b200 import metrics  # noqa: E402

H36M_EVAL = metrics.H36M_EVAL_JOINT


def device_ms(fn, min_seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    iters, total = 8, 0.0
    while True:
        beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        beg.record()
        for _ in range(iters):
            fn()
        end.record()
        end.synchronize()
        total = beg.elapsed_time(end)
        if total >= 1000.0 * min_seconds:
            return total / iters, iters
        iters *= 2


def gpu_power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    B, V = args.batch, 6890
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    Jh = np.load(os.path.join(ROOT, "tests", "golden", "eval_metrics.npz"))["J_regressor_h36m"]
    Jm = np.zeros((24, V))
    for j in range(24):
        cols = rng.choice(V, 30, replace=False)
        w = rng.random(30)
        Jm[j, cols] = w / w.sum()
    pred = (rng.standard_normal((B, V, 3)) * 300.0 + [0.0, 0.0, 4000.0]).astype(np.float32)
    gt = (pred + rng.standard_normal((B, V, 3)) * 30.0).astype(np.float32)
    pj, gj = np.einsum("jv,bvc->bjc", Jh, pred).astype(np.float32), np.einsum("jv,bvc->bjc", Jh, gt).astype(np.float32)

    P, G = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    PJ, GJ = torch.from_numpy(pj).to(dev), torch.from_numpy(gj).to(dev)
    Jm_t, Jh_t = torch.from_numpy(Jm).float().to(dev), torch.from_numpy(Jh).float().to(dev)
    eval_ms, eval_iters = device_ms(lambda: metrics.evaluate_meshes(P, G, Jm_t, 0, Jh_t, 0, H36M_EVAL), args.min_seconds)
    both_ms, both_iters = device_ms(lambda: metrics.compute_both_err(P, G, PJ, GJ, H36M_EVAL), args.min_seconds)

    t0 = time.perf_counter()
    for b in range(B):
        mo.evaluate_sample(pred[b], gt[b], Jm, 0, Jh, 0, H36M_EVAL, None, pa_mesh=True)
    host_eval_ms = 1e3 * (time.perf_counter() - t0)
    t0 = time.perf_counter()
    mo.both_err(pred, gt, pj, gj, H36M_EVAL)
    host_both_ms = 1e3 * (time.perf_counter() - t0)

    print(json.dumps({
        "gpu": torch.cuda.get_device_name(dev), "power_limit": gpu_power_limit(), "batch": B, "n_vertex": V,
        "evaluate_meshes_ms": round(eval_ms, 4), "evaluate_meshes_iters": eval_iters,
        "compute_both_err_ms": round(both_ms, 4), "compute_both_err_iters": both_iters,
        "host_numpy_evaluate_loop_ms": round(host_eval_ms, 2), "host_numpy_compute_both_err_ms": round(host_both_ms, 2),
        "host_cpus": os.cpu_count(),
    }))


if __name__ == "__main__":
    main()
