"""Timing aid (needs a GPU): the Trainer's objective as one op (loss.Pose2MeshLoss) against the torch composition a
user writes without it (advanced-index gather of the real rows, torch.matmul regression, CoordLoss x 3 and MeshLosses).

    python tools/time_pose2mesh_loss.py [--iters 50]

Sizes: SMPL (6890 of 12288 rows, 17 joints) at B = 64 (the reference's batch) and B = 256, MANO (778 of 1088 rows,
21 joints) at B = 1024.  Each step is forward + backward with the edge term on; the two are alternated step by step
after a warm-up and every step is timed with device events.  Prints one JSON line: the card's name and power limit
(read in the same run), the median / min / max step time in milliseconds per setting and size, and the library
launches of one step (p2m_launch_count; the composition's torch launches are not counted there)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from pose2mesh_loss_cases import INPUTS, make_case
from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200 import loss as L

WEIGHTS = (0.1, 20.0, 1e-3)
SIZES = {"smpl_b64": (6890, 12288, 64, 17, 17), "smpl_b256": (6890, 12288, 256, 17, 17),
         "mano_b1024": (778, 1088, 1024, 21, 21)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def steps(c, dev):
    x = {k: c[k].to(dev) for k in INPUTS}
    nv = int(c["face"].max()) + 1
    rows = torch.as_tensor(c["perm_reverse"][:nv], dtype=torch.long, device=dev)
    jr = c["joint_regressor"].to(dev)
    crit = L.Pose2MeshLoss(c["face"], c["joint_regressor"], c["perm_reverse"], *WEIGHTS)
    coord, mesh_losses = L.CoordLoss(has_valid=True), L.MeshLosses(c["face"])

    def native():
        cam, lift = x["cam_mesh"].detach().requires_grad_(True), x["lift_pose"].detach().requires_grad_(True)
        loss, _ = crit(cam, lift, *(x[k] for k in INPUTS[2:]), edge=True)
        loss.backward()

    def composed():
        cam, lift = x["cam_mesh"].detach().requires_grad_(True), x["lift_pose"].detach().requires_grad_(True)
        pred_mesh = cam[:, rows]
        pred_pose = torch.matmul(jr[None], pred_mesh * 1000)
        normal, edge = mesh_losses(pred_mesh, x["gt_mesh"])
        loss = (coord(pred_mesh, x["gt_mesh"], x["mesh_valid"]) + WEIGHTS[0] * normal
                + WEIGHTS[2] * coord(pred_pose, x["gt_reg3dpose"], x["reg3dpose_valid"])
                + WEIGHTS[2] * coord(lift, x["gt_lift3dpose"], x["lift3dpose_valid"]) + WEIGHTS[1] * edge)
        loss.backward()

    return {"pose2mesh_loss": native, "torch_composition": composed}


def launches(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    with torch.autograd.set_multithreading_enabled(False):   # the counter is per thread: backward on this one
        lib.p2m_launch_count_reset()
        fn()
        n = int(lib.p2m_launch_count())
    torch.cuda.synchronize()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "iters": args.iters, "sizes": {}}
    for name, size in SIZES.items():
        fns = steps(make_case(*size, seed=1), dev)
        for fn in fns.values():
            for _ in range(5):
                fn()
        times = {k: [] for k in fns}
        for _ in range(args.iters):
            for k, fn in fns.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
        out["sizes"][name] = {k: {"median_ms": round(statistics.median(v), 4), "min_ms": round(min(v), 4),
                                  "max_ms": round(max(v), 4), "library_launches": launches(fns[k])}
                              for k, v in times.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
