#!/usr/bin/env python
"""Time the batched body-model layers on the GPU: SMPLLayer.forward at B = 256 and ManoLayer.forward at B = 1024, on
the seeded synthetic models of tests/body_models.py (SMPL and MANO sizes).  Seeded inputs; prints one JSON line.

    python tools/time_body_model.py [--min-seconds 1.0]

Device times come from CUDA events around >= min_seconds of back-to-back forwards after a warm-up (each forward is
the layer's three kernels plus its output and workspace allocations).  Achieved rates use the shape-derived counts
of the blend-shape product: 2 B (S + P) 3V flops, and the basis read once plus the vertices written once in bytes.
The host baseline is the float64 numpy oracle (tests/body_model_oracle.py) called per sample (B = 1), as the
datasets call the reference layer; it is a port of the reference, not the reference itself.
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
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer  # noqa: E402


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


def measure(name, layer, model, B, width, trans_sd, oracle_fwd, min_seconds, dev):
    rng = np.random.RandomState(B)
    pose = rng.normal(0.0, 0.6, (B, width)).astype(np.float32)
    betas = rng.normal(0.0, 1.5, (B, 10)).astype(np.float32)
    trans = rng.normal(0.0, trans_sd, (B, 3)).astype(np.float32)
    P, Bt, T = (torch.from_numpy(a).to(dev) for a in (pose, betas, trans))
    ms, iters = device_ms(lambda: layer(P, Bt, T), min_seconds)
    V, K = layer.n_vertex, layer.n_betas + 9 * (layer.num_joints - 1)
    flops = 2.0 * B * K * 3 * V
    nbytes = 4.0 * (K * 3 * V + B * 3 * V)
    n_host = 20
    t0 = time.perf_counter()
    for b in range(n_host):
        oracle_fwd(model, pose[b:b + 1], betas[b:b + 1], trans[b:b + 1])
    host_ms = 1e3 * (time.perf_counter() - t0) / n_host
    return {f"{name}_batch": B, f"{name}_forward_ms": round(ms, 4), f"{name}_iters": iters,
            f"{name}_blend_tflops": round(flops / ms / 1e9, 3), f"{name}_blend_gbytes_per_s": round(nbytes / ms / 1e6, 1),
            f"{name}_host_oracle_per_sample_ms": round(host_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    smpl, mano = bm.smpl_model(), bm.mano_model("right", False)
    sl = SMPLLayer(smpl["v_template"], smpl["shapedirs"], smpl["posedirs"], smpl["J_regressor"], smpl["weights"],
                   smpl["parents"], smpl["betas"])
    ml = ManoLayer(mano["v_template"], mano["shapedirs"], mano["posedirs"], mano["J_regressor"], mano["weights"],
                   mano["betas"], mano["hands_mean"], flat_hand_mean=False)
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit": gpu_power_limit(), "host_cpus": os.cpu_count()}
    out.update(measure("smpl", sl, smpl, 256, 72, 0.5, bo.smpl_forward, args.min_seconds, dev))
    out.update(measure("mano", ml, mano, 1024, 48, 0.1, bo.mano_forward, args.min_seconds, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
