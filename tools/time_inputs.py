#!/usr/bin/env python
"""Time the training inputs on the device: training_pose2d at B = 256 for both joint sets (COCO with the synthetic
detector errors, Human3.6M with the error model) and synthesize_pose at B = 4096, with the card's name and power limit
read in the same run.  Beside them, on the same run's host: the float64 oracle's synthesize_pose per sample
(oracle/inputs_oracle.py, one sample per call) and, when P2M_REFERENCE_ROOT names a reference checkout, the
reference's lib/noise_utils.synthesize_pose per sample.  Prints one JSON line.

    python tools/time_inputs.py [--min-seconds 1.0] [--host-samples 50]

Device times come from CUDA events around >= min_seconds of back-to-back calls after a warm-up (each call includes its
output allocation).
"""
import argparse
import json
import os
import random
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from inputs_cases import case, error_table  # noqa: E402
from oracle import inputs_oracle as io  # noqa: E402
from pose2mesh_release_b200.inputs import Human36MErrorModel, synthesize_pose, training_pose2d  # noqa: E402
from time_targets import card, device_ms  # noqa: E402


def host_ms(fn, n):
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    return 1e3 * (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--host-samples", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_inputs.py needs a GPU")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    out = {"device": card()}
    B = 256
    base = rng.uniform(200, 600, (B, 1, 2))
    px = torch.from_numpy((base + rng.uniform(0, [300, 500], (B, 19, 2))).astype(np.float32)).to(dev)
    px17 = px[:, :17].contiguous()
    seed = torch.tensor([1, 2], dtype=torch.int64, device=dev)
    model = Human36MErrorModel(*error_table())
    out["training_pose2d_coco_B256_ms"] = round(device_ms(lambda: training_pose2d(px, "coco", seed=seed),
                                                          a.min_seconds), 4)
    out["training_pose2d_human36_B256_ms"] = round(device_ms(
        lambda: training_pose2d(px17, "human36", error_model=model, seed=seed), a.min_seconds), 4)
    joints, area, _ = case("all_visible")
    Bs = 4096
    realistic = joints.copy()            # the fixture's skeleton at a typical crop-space area: overlapping sources
    jt = torch.from_numpy(np.repeat(realistic[None], Bs, 0).astype(np.float32)).to(dev)
    at = torch.full((Bs,), 60000.0, device=dev)
    out["synthesize_pose_B4096_ms"] = round(device_ms(lambda: synthesize_pose(jt, at, seed), a.min_seconds), 4)
    one = realistic[None].astype(np.float64)
    out["oracle_host_ms_per_sample"] = round(host_ms(lambda: io.synthesize_pose(one, np.array([60000.0]), (1, 2)),
                                                     a.host_samples), 3)
    ref = os.environ.get("P2M_REFERENCE_ROOT", "")
    if ref:
        shim = types.ModuleType("easydict")
        shim.EasyDict = type("EasyDict", (dict,), {"__getattr__": dict.__getitem__, "__setattr__": dict.__setitem__})
        sys.modules.setdefault("easydict", shim)
        sys.path.insert(0, os.path.join(ref, "lib"))
        import noise_utils
        np.random.seed(0)
        random.seed(0)
        out["reference_host_ms_per_sample"] = round(host_ms(
            lambda: noise_utils.synthesize_pose(realistic.copy(), 60000.0, num_overlap=0), a.host_samples), 3)
    else:
        out["reference_host_ms_per_sample"] = "not measured (P2M_REFERENCE_ROOT unset)"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
