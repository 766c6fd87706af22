#!/usr/bin/env python
"""Time Human36MTargets (the human36m camera-frame call plus the Human3.6M assembly, six launches) at B = 256 on the
seeded synthetic SMPL model of tests/body_models.py with the regressors of tests/golden/targets.npz, and the float64
oracle's per-sample host loop (oracle/targets_oracle.py, B = 1 per call as the datasets' __getitem__ runs) on the same
host.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/time_targets.py [--min-seconds 1.0] [--host-samples 16]

Device times come from CUDA events around >= min_seconds of back-to-back calls after a warm-up (each call includes its
output and workspace allocations).  The host loop is a float64 port of the reference, not the reference itself.
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import body_model_oracle as bo  # noqa: E402
import body_models as bm  # noqa: E402
from oracle import targets_oracle as to  # noqa: E402
from pose2mesh_release_b200.body_model import SMPLLayer  # noqa: E402
from pose2mesh_release_b200.targets import Human36MTargets  # noqa: E402


def device_ms(fn, min_seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    iters = 8
    while True:
        beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        beg.record()
        for _ in range(iters):
            fn()
        end.record()
        torch.cuda.synchronize()
        total = beg.elapsed_time(end)
        if total >= 1e3 * min_seconds:
            return total / iters
        iters *= 2


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--host-samples", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_targets.py needs a GPU")
    golden = np.load(os.path.join(ROOT, "tests", "golden", "targets.npz"))
    m = bm.smpl_model()
    layer = SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                      m["betas"])
    rng = np.random.RandomState(0)
    B = 256
    f32 = lambda x: np.asarray(x, np.float32)  # noqa: E731
    pose = f32(rng.normal(0, 0.4, (B, 72)))
    betas = f32(rng.normal(0, 1.0, (B, 10)))
    trans = f32(rng.normal(0, 0.3, (B, 3)))
    R = np.repeat(np.eye(3, dtype=np.float32)[None], B, 0)
    t = f32(rng.normal(0, 300, (B, 3)) + [0, 0, 4000])
    f = f32(np.full((B, 2), 1150))
    c = f32(np.full((B, 2), 512))
    joint_cam = f32(rng.normal(0, 300, (B, 17, 3)) + [0, 0, 4000])
    host = (pose, betas, trans, R, t, f, c, joint_cam)
    dev = torch.device("cuda:0")
    args = [torch.from_numpy(x).to(dev) for x in host]
    out = {"device": card(), "B": B}
    for js in ("human36", "coco"):
        mod = Human36MTargets(layer, golden["reg_h36m"], golden["reg_coco"], js)
        out[f"h36m_targets_{js}_ms"] = round(device_ms(lambda: mod(*args), a.min_seconds), 4)
    fwd = lambda q, b, tr: bo.smpl_forward(m, q, b, tr)  # noqa: E731
    n = a.host_samples
    t0 = time.perf_counter()
    for i in range(n):
        one = [x[i:i + 1] for x in host]
        mesh, _ = to.camera_frame(fwd, m["betas"], "human36m", *one[:5])
        to.h36m_targets(mesh, one[7], one[5], one[6], golden["reg_h36m"], golden["reg_coco"], "coco")
    host_ms = 1e3 * (time.perf_counter() - t0) / n
    out["oracle_host_ms_per_sample"] = round(host_ms, 3)
    out["oracle_host_ms_per_batch"] = round(host_ms * B, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
