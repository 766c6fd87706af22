"""Timing aid (needs a GPU): training steps with default BatchNorms against frozen BatchNorms.

    python tools/time_bn_modes.py [--iters 30]

Two steps, each in two settings alternated round by round after a warm-up, every step timed with device events:
  - MeshNet at B = 256 on the SMPL-size hierarchy of bench.py (6890 vertices, levels 9): forward + L1 loss + backward,
    default (batch statistics) against every BatchNorm in eval mode inside the train-mode model (frozen statistics);
  - PoseNet (J = 17, H = 4096, two stages, p = 0.5) at B = 256: forward + backward, default against frozen BatchNorms
    with every Dropout in eval mode.
Prints one JSON line: the card's name and power limit (read in the same run) and the median / min / max step time in
milliseconds per setting."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn as nn

from pose2mesh_release_b200 import graph as pg
from pose2mesh_release_b200.meshnet import Pose2Mesh
from pose2mesh_release_b200.posenet import LinearModel


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def freeze(model, frozen, dropout_too=False):
    for m in model.modules():
        if isinstance(m, nn.BatchNorm1d) or (dropout_too and isinstance(m, nn.Dropout)):
            m.train(not frozen)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_bn_modes: no GPU")
    dev = torch.device("cuda:0")
    B = 256
    torch.manual_seed(0)
    face = pg.synthetic_sphere_faces(6890, 2)
    _, graph_L, _, _ = pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=9)
    mesh = Pose2Mesh(5, 3, graph_L).to(dev).train()
    x = torch.randn(B, 17, 5, device=dev)
    tgt = torch.randn(B, mesh.num_vertices, 3, device=dev)
    pose = LinearModel(17, 4096, 2, 0.5).to(dev).train()
    x2 = torch.randn(B, 34, device=dev)
    d_out = torch.randn(B, 51, device=dev)

    def mesh_step():
        mesh.zero_grad(set_to_none=True)
        (mesh(x) - tgt).abs().mean().backward()

    def pose_step():
        pose.zero_grad(set_to_none=True)
        pose(x2).backward(d_out)

    cases = {"meshnet_default": (mesh, False, False, mesh_step), "meshnet_frozen_bn": (mesh, True, False, mesh_step),
             "posenet_default": (pose, False, True, pose_step),
             "posenet_frozen_bn_no_dropout": (pose, True, True, pose_step)}
    times = {k: [] for k in cases}
    for it in range(args.warmup + args.iters):
        for name, (model, frozen, dropout_too, step) in cases.items():
            freeze(model, frozen, dropout_too)
            t = timed(step)
            if it >= args.warmup:
                times[name].append(t)
    res = {"tool": "time_bn_modes", "card": card(), "batch": B, "iters": args.iters,
           "step_ms": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
