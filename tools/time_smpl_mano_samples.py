#!/usr/bin/env python
"""Time the SURREAL, FreiHAND and 3DPW sample assembly on the device, on the seeded synthetic SMPL and MANO models of
tests/body_models.py with the regressors of tests/golden/targets.npz: each targets call at B = 256 (SURREALTargets with
augm_params' rotation and flip, FreiHANDTargets, PW3DTargets: six launches each), FreiHANDTargets also at B = 1024 (the
MANO bench batch), and training_pose2d on the 'smpl' set with a rotation and a flip (one launch); and the float64
oracle's per-sample host loop (tests/targets_oracle camera frame + tests/smpl_mano_oracle.py assembly, B = 1 per call as
__getitem__ runs) on the same host.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/time_smpl_mano_samples.py [--min-seconds 1.0] [--host-samples 16]

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
import smpl_mano_oracle as smo  # noqa: E402
from oracle import targets_oracle as to  # noqa: E402
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer  # noqa: E402
from pose2mesh_release_b200.inputs import augm_params, training_pose2d  # noqa: E402
from pose2mesh_release_b200.targets import FreiHANDTargets, PW3DTargets, SURREALTargets  # noqa: E402
from time_targets import card, device_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--host-samples", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_smpl_mano_samples.py needs a GPU")
    golden = np.load(os.path.join(ROOT, "tests", "golden", "targets.npz"))
    reg = (golden["reg_h36m"], golden["reg_coco"])
    m, mm = bm.smpl_model(), bm.mano_model("right", False)
    smpl = SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                     m["betas"])
    mano = ManoLayer(mm["v_template"], mm["shapedirs"], mm["posedirs"], mm["J_regressor"], mm["weights"], mm["betas"],
                     mm["hands_mean"], flat_hand_mean=False, side="right")
    rng = np.random.RandomState(0)
    f32 = lambda x: np.asarray(x, np.float32)  # noqa: E731
    dev = torch.device("cuda:0")
    d = lambda x: torch.from_numpy(x).to(dev)  # noqa: E731

    def smpl_args(B):
        return (f32(rng.normal(0, 0.4, (B, 72))), f32(rng.normal(0, 1.0, (B, 10))),
                f32(rng.normal(0, 0.3, (B, 3)) + [0, 0, 4]), f32(np.full((B, 2), 1150)), f32(np.full((B, 2), 512)))

    def mano_args(B):
        return (f32(rng.normal(0, 0.4, (B, 48))), f32(rng.normal(0, 1.0, (B, 10))),
                np.repeat(np.eye(3, dtype=np.float32)[None], B, 0), f32(rng.normal(0, 0.05, (B, 3)) + [0, 0, 0.5]))

    B = 256
    seed = torch.tensor([1234, 5678], dtype=torch.int64, device=dev)
    flip, rot = augm_params(B, True, 30.0, seed)
    out = {"device": card(), "B": B}
    s_host = smpl_args(B)
    sm, sargs = SURREALTargets(smpl), [d(x) for x in s_host]
    out["surreal_targets_ms"] = round(device_ms(lambda: sm(*sargs, rot=rot, flip=flip), a.min_seconds), 4)
    fm = FreiHANDTargets(mano)
    for n in (B, 1024):
        fargs = [d(x) for x in mano_args(n)]
        out[f"freihand_targets_B{n}_ms"] = round(device_ms(lambda: fm(*fargs), a.min_seconds), 4)
    pm, pargs = PW3DTargets(smpl, *reg), [d(x) for x in smpl_args(B)]
    out["pw3d_targets_ms"] = round(device_ms(lambda: pm(*pargs), a.min_seconds), 4)
    px = d(f32(rng.uniform(100, 900, (B, 24, 2))))
    out["training_pose2d_smpl_aug_ms"] = round(
        device_ms(lambda: training_pose2d(px, "smpl", noise=False, rot=rot, flip=flip), a.min_seconds), 4)
    fwd = lambda q, b, tr: bo.smpl_forward(m, q, b, tr)  # noqa: E731
    pose, betas, trans, f, c = s_host
    n = a.host_samples
    rot_h, flip_h = rot.cpu().numpy(), flip.cpu().numpy()
    t0 = time.perf_counter()
    for i in range(n):
        mesh, joints = to.camera_frame(fwd, m["betas"], "surreal", pose[i:i + 1], betas[i:i + 1], trans[i:i + 1],
                                       None, None)
        smo.surreal_targets(mesh, joints, f[i:i + 1], c[i:i + 1], rot_h[i:i + 1], flip_h[i:i + 1])
    host_ms = 1e3 * (time.perf_counter() - t0) / n
    out["oracle_host_ms_per_sample"] = round(host_ms, 3)
    out["oracle_host_ms_per_batch"] = round(host_ms * B, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
