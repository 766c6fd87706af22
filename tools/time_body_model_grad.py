#!/usr/bin/env python
"""Device time of the body-model backward (pose2mesh_release_b200.body_model with differentiable=True), one JSON line.

Two workloads on the seeded synthetic models of tests/body_models.py: SMPL at B=256 and MANO (right hand) at B=1024,
random pose, betas and trans, cotangents on vertices and joints.  For each, the device time of one call (CUDA events
around `iters` calls after `warmup`, median of `reps` windows) of:

  * forward:   the default (forward-only) layer;
  * backward:  p2m_body_model_backward alone, through the C ABI;
  * fwd+bwd:   forward and autograd backward through the differentiable layer, eager;
  * graph:     the same step captured once in a CUDA graph and replayed;

and the host time of the float64 torch restatement's forward + autograd backward (tests/body_model_grad_ref.py, the
reference layers' maths) on `--host-batch` samples, with the CPU thread count.  The card's name and power limit are read
in the same run.

    python tools/time_body_model_grad.py [--iters 20] [--warmup 5] [--reps 5] [--host-batch 8]
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import body_model_grad_ref as gr  # noqa: E402
import body_models as bm  # noqa: E402
from pose2mesh_release_b200 import _lib  # noqa: E402
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer  # noqa: E402


def device_ms(fn, iters, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return round(statistics.median(times), 4)


def gpu_query(field):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except Exception:
        return None


def layer(kind, differentiable):
    if kind == "smpl":
        m = bm.smpl_model()
        return m, SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"],
                            m["parents"], m["betas"], differentiable=differentiable)
    m = bm.mano_model("right", False)
    return m, ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                        m["hands_mean"], flat_hand_mean=False, differentiable=differentiable)


def workload(kind, B, args, dev):
    m, fwd_layer = layer(kind, False)
    _, grad_layer = layer(kind, True)
    rng = np.random.RandomState(B)
    width, nv, nj = (72, 6890, 24) if kind == "smpl" else (48, 778, 21)
    t = lambda a: torch.as_tensor(np.asarray(a, np.float32), device=dev)  # noqa: E731
    pose, betas = t(rng.normal(0, 0.6, (B, width))), t(rng.normal(0, 1.5, (B, 10)))
    trans = t(rng.normal(0, 0.3, (B, 3)))
    gv, gj = t(rng.normal(0, 1, (B, nv, 3))), t(rng.normal(0, 1, (B, nj, 3)))
    out = {"model": kind, "batch": B}
    out["forward_ms"] = device_ms(lambda: fwd_layer(pose, betas, trans), args.iters, args.warmup, args.reps)

    lib, h = _lib.load(), grad_layer.handle(dev.index)
    rule = _lib.P2M_BETAS_ZERO_MEANS_MODEL if kind == "smpl" else _lib.P2M_BETAS_AS_GIVEN
    gp, gb, gt = torch.empty_like(pose), torch.empty_like(betas), torch.empty_like(trans)
    nbytes = lib.p2m_body_model_backward_workspace_bytes(h, B)
    ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def bwd():
        _lib.check(lib.p2m_body_model_backward(h, pose.data_ptr(), betas.data_ptr(), rule, trans.data_ptr(), -1,
                                               gv.data_ptr(), gj.data_ptr(), gp.data_ptr(), gb.data_ptr(),
                                               gt.data_ptr(), B, ws.data_ptr(), nbytes, stream))

    out["backward_ms"] = device_ms(bwd, args.iters, args.warmup, args.reps)
    out["backward_workspace_mb"] = round(nbytes / 2 ** 20, 1)
    params = [pose.clone().requires_grad_(True), betas.clone().requires_grad_(True), trans.clone().requires_grad_(True)]

    def step():
        for p in params:
            p.grad = None
        v, j = grad_layer(*params)
        torch.autograd.backward([v, j], [gv, gj])

    out["fwd_bwd_ms"] = device_ms(step, args.iters, args.warmup, args.reps)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    out["fwd_bwd_graph_ms"] = device_ms(g.replay, args.iters, args.warmup, args.reps)

    hb = args.host_batch
    cpu = lambda x: x[:hb].cpu().numpy()  # noqa: E731
    t0 = time.perf_counter()
    gr.vjp(kind, m, cpu(pose), cpu(betas), cpu(trans), None, cpu(gv), cpu(gj))
    out["host_f64_fwd_bwd_s"] = round(time.perf_counter() - t0, 3)
    out["host_batch"] = hb
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_body_model_grad.py measures the GPU; no CUDA device is visible")
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit": gpu_query("power.limit"),
           "cpu_threads": torch.get_num_threads(), "workloads": []}
    for kind, B in (("smpl", 256), ("mano", 1024)):
        out["workloads"].append(workload(kind, B, args, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
