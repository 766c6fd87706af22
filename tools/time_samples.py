#!/usr/bin/env python
"""Time a training sample's device assembly at B = 256 on the seeded synthetic SMPL model of tests/body_models.py with
the regressors of tests/golden/targets.npz: each dataset's targets call (Human36MTargets, COCOTargets, MuCoTargets,
AMASSTargets, coco joint set, with augm_params' rotation and flip: six launches each), augm_params (one launch) and
training_pose2d with the COCO noise, a rotation and a flip (one launch); and the float64 oracle's per-sample host loop
(oracle/targets_oracle.py camera frame + oracle/samples_oracle.py assembly, B = 1 per call as __getitem__ runs) on the
same host.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/time_samples.py [--min-seconds 1.0] [--host-samples 16]

Device times come from CUDA events around >= min_seconds of back-to-back calls after a warm-up (each call includes its
output and workspace allocations).  The host loop is a float64 port of the reference, not the reference itself.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import body_model_oracle as bo  # noqa: E402
import body_models as bm  # noqa: E402
from oracle import samples_oracle as so  # noqa: E402
from oracle import targets_oracle as to  # noqa: E402
from pose2mesh_release_b200.body_model import SMPLLayer  # noqa: E402
from pose2mesh_release_b200.inputs import augm_params, training_pose2d  # noqa: E402
from pose2mesh_release_b200.targets import AMASSTargets, COCOTargets, Human36MTargets, MuCoTargets  # noqa: E402
from time_targets import card, device_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--host-samples", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_samples.py needs a GPU")
    golden = np.load(os.path.join(ROOT, "tests", "golden", "targets.npz"))
    reg = (golden["reg_h36m"], golden["reg_coco"])
    m = bm.smpl_model()
    layer = SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                      m["betas"])
    rng = np.random.RandomState(0)
    B = 256
    f32 = lambda x: np.asarray(x, np.float32)  # noqa: E731
    pose = f32(rng.normal(0, 0.4, (B, 72)))
    betas = f32(rng.normal(0, 1.0, (B, 10)))
    trans = f32(rng.normal(0, 0.3, (B, 3)) + [0, 0, 4])
    R = np.repeat(np.eye(3, dtype=np.float32)[None], B, 0)
    t = f32(rng.normal(0, 0.3, (B, 3)) + [0, 0, 4])
    f, c = f32(np.full((B, 2), 1150)), f32(np.full((B, 2), 512))
    joint_cam = f32(rng.normal(0, 300, (B, 17, 3)) + [0, 0, 4000])
    s, tt = f32(rng.uniform(180, 260, B)), f32(rng.uniform(300, 500, (B, 2)))
    kps, vis = f32(rng.uniform(100, 600, (B, 17, 2))), f32(rng.uniform(size=(B, 17)) < 0.7)
    dev = torch.device("cuda:0")
    d = lambda x: torch.from_numpy(x).to(dev)  # noqa: E731
    seed = torch.tensor([1234, 5678], dtype=torch.int64, device=dev)
    flip, rot = augm_params(B, True, 30.0, seed)
    calls = {
        "human36m": (Human36MTargets, (pose, betas, trans, R, t * 1000, f, c, joint_cam)),
        "coco": (COCOTargets, (pose, betas, s, tt, kps, vis)),
        "muco": (MuCoTargets, (pose, betas, trans, f, c)),
        "amass": (AMASSTargets, (pose, betas, R, t, f, c)),
    }
    out = {"device": card(), "B": B}
    for name, (cls, host) in calls.items():
        mod, args = cls(layer, *reg, "coco"), [d(x) for x in host]
        out[f"{name}_targets_ms"] = round(device_ms(lambda: mod(*args, rot=rot, flip=flip), a.min_seconds), 4)
    out["augm_params_ms"] = round(device_ms(lambda: augm_params(B, True, 30.0, seed), a.min_seconds), 4)
    px = d(f32(rng.uniform(100, 900, (B, 19, 2))))
    out["training_pose2d_coco_aug_ms"] = round(
        device_ms(lambda: training_pose2d(px, "coco", seed=seed, rot=rot, flip=flip), a.min_seconds), 4)
    fwd = lambda q, b, tr: bo.smpl_forward(m, q, b, tr)  # noqa: E731
    n = a.host_samples
    rot_h, flip_h = rot.cpu().numpy(), flip.cpu().numpy()
    t0 = time.perf_counter()
    for i in range(n):
        mesh, _ = to.camera_frame(fwd, m["betas"], "coco", pose[i:i + 1], betas[i:i + 1], None, None, None)
        tg = so.sample_targets("coco", mesh, *reg, "coco", s=s[i:i + 1], t=tt[i:i + 1], keypoints=kps[i:i + 1],
                               keypoints_valid=vis[i:i + 1])
        so.j3d_processing(tg["lift_pose3d"], rot_h[i:i + 1], flip_h[i:i + 1], "coco")
    host_ms = 1e3 * (time.perf_counter() - t0) / n
    out["oracle_host_ms_per_sample"] = round(host_ms, 3)
    out["oracle_host_ms_per_batch"] = round(host_ms * B, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
