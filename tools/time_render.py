#!/usr/bin/env python
"""Device time of the mesh overlay (SURVEY.md §8 row f10, pose2mesh_release_b200.render.render_meshes), one JSON line.

Three workloads of seeded synthetic meshes (a closed ellipsoid of SMPL's 6890 vertices / 13776 faces, or of MANO's
778 / 1552, wound outward):

  * demo:  one 1920 x 1080 image with 8 people of different sizes and places;
  * video: 256 frames of 1920 x 1080 with one person each (the same mesh and camera on every frame);
  * hands: 1024 crops of 224 x 224 with one hand each (the same mesh and camera on every crop).

For each: the device time of one call (CUDA events around `iters` calls after `warmup`, median of `reps` windows),
pixels/s (output pixels), fragments/s (covered pixel centres of front faces inside the clip planes, counted by
oracle/render_oracle.py: over the whole demo image, and over one frame / crop times the count of the others, which are
identical), and the oracle's host time on `--host-items` frames / crops (the whole demo image), with the CPU count.
The card's name and power limit are read in the same run.

    python tools/time_render.py [--iters 10] [--warmup 3] [--reps 5] [--host-items 4]
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
from scipy.spatial import ConvexHull

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import render_oracle as ro  # noqa: E402
from pose2mesh_release_b200.render import render_meshes  # noqa: E402


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
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times), times


def gpu_query(field):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


def ellipsoid(n_vertex, half, seed):
    """[n, 3] float32 points on an ellipsoid with half-axes `half`, faces [2 n - 4, 3] wound outward."""
    p = np.random.default_rng(seed).normal(size=(n_vertex, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    f = ConvexHull(p).simplices.astype(np.int64)
    a, b, c = p[f[:, 0]], p[f[:, 1]], p[f[:, 2]]
    flip = np.einsum("ij,ij->i", np.cross(b - a, c - a), a + b + c) < 0
    f[flip, 1], f[flip, 2] = f[flip, 2], f[flip, 1].copy()
    return (p * np.asarray(half)).astype(np.float32), f


def workloads():
    g = np.random.default_rng(0)
    body, body_f = ellipsoid(6890, (0.35, 0.85, 0.15), 0)
    hand, hand_f = ellipsoid(778, (0.04, 0.1, 0.02), 1)
    P = 8  # demo: people 300 .. 800 px tall across the image
    h = g.uniform(300, 800, P)
    cx, cy = g.uniform(200, 1720, P), g.uniform(400, 680, P)
    s = h / 1.7
    demo_cams = np.stack([s * 2 / 1920, s * 2 / 1080, (cx - 960) / s, (cy - 540) / s], 1).astype(np.float32)
    s1 = 700 / 1.7
    video_cam = np.array([s1 * 2 / 1920, s1 * 2 / 1080, 0.2, 0.0], np.float32)
    s2 = 180 / 0.2
    hand_cam = np.array([s2 * 2 / 224, s2 * 2 / 224, 0.0, 0.0], np.float32)
    return {
        "demo": dict(N=1, H=1080, W=1920, verts=np.repeat(body[None], P, 0), faces=body_f, cams=demo_cams,
                     index=np.zeros(P, np.int32)),
        "video": dict(N=256, H=1080, W=1920, verts=np.repeat(body[None], 256, 0), faces=body_f,
                      cams=np.repeat(video_cam[None], 256, 0), index=np.arange(256, dtype=np.int32)),
        "hands": dict(N=1024, H=224, W=224, verts=np.repeat(hand[None], 1024, 0), faces=hand_f,
                      cams=np.repeat(hand_cam[None], 1024, 0), index=np.arange(1024, dtype=np.int32)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-items", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_render.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit": gpu_query("power.limit"),
           "sm_clock_max": gpu_query("clocks.max.sm"), "host_cpus": os.cpu_count(), "torch": torch.__version__}
    for name, w in workloads().items():
        N, H, W, P = w["N"], w["H"], w["W"], len(w["verts"])
        rng = np.random.default_rng(1)
        imgs = torch.from_numpy(rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)).to(dev)
        verts, cams = torch.from_numpy(w["verts"]).to(dev), torch.from_numpy(w["cams"]).to(dev)
        faces = torch.from_numpy(w["faces"].astype(np.int32)).to(dev)
        colors = torch.from_numpy(rng.uniform(0.3, 1.0, (P, 3)).astype(np.float32)).to(dev)
        idx = torch.from_numpy(w["index"]).to(dev)
        med, runs = device_ms(lambda: render_meshes(imgs, verts, faces, cams, colors, image_index=idx),
                              args.iters, args.warmup, args.reps)
        covered = int((render_meshes(imgs, verts, faces, cams, colors, image_index=idx, return_maps=True)[1] >= 0).sum())
        k = P if name == "demo" else min(args.host_items, P)   # people (= images) the oracle draws on the host
        kn = 1 if name == "demo" else k
        t0 = time.perf_counter()
        ro.render(imgs[:kn].cpu().numpy(), w["verts"][:k], w["faces"], w["cams"][:k], colors[:k].cpu().numpy(),
                  np.arange(k) if name != "demo" else None)
        host_s = time.perf_counter() - t0
        _, frags = ro.raster_keys(w["verts"][:k], w["faces"], w["cams"][:k], None if name == "demo" else np.arange(k),
                                  kn, H, W, return_count=True)
        frags = frags if name == "demo" else frags // k * P
        out[name] = {"images": N, "size": [H, W], "people": P, "faces": int(len(w["faces"])),
                     "device_ms": round(med, 4), "runs_ms": [round(r, 4) for r in runs],
                     "pixels_per_s": N * H * W / (med * 1e-3), "fragments": int(frags),
                     "fragments_per_s": frags / (med * 1e-3), "covered_pixels": covered,
                     "oracle_host_s": round(host_s, 3), "oracle_host_subset": f"{kn} of {N} images, {k} of {P} people"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
