"""Timing aid (needs a GPU): the native RMSprop step (pose2mesh_release_b200.optim.RMSprop) against
torch.optim.RMSprop (its default, the foreach path), alternated round by round in one process.

    python tools/time_rmsprop.py [--rounds 100] [--warmup 10]

Three workloads, each with torch's default RMSprop options (alpha 0.99, eps 1e-8, lr 1e-3, as every released config):
  posenet      the 22 tensors (20 with gradients) of PoseNet, J = 17, H = 4096, two stages;
  flat_smpl    the 106 tensors (104 with gradients) of FlatPose2Mesh with the SMPL-size (6890-vertex) MeshNet;
  lift_step    a LiftTrainer step at B = 64 (lib/core/base.py:253-265): native PoseNet train forward + backward, the
               masked L1 loss and the optimizer step, one model copy per optimizer.
The step sets use fixed synthetic gradients, the same on both sides.  Every timed region is bracketed by CUDA events
after a 256 MiB buffer is written (L2 flushed, outside the events).  Prints one JSON line: per workload and side the
median and range in ms and the median host time of step(); for the step sets the algorithmic bytes (5 floats per
parameter: p, g, square_avg read, p, square_avg written), the GB/s they imply, and the native launches per step
(p2m_launch_count); the card, its power limit and the SM clocks sampled during the timed rounds."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from pose2mesh_release_b200 import _lib  # noqa: E402
from pose2mesh_release_b200.loss import CoordLoss  # noqa: E402
from pose2mesh_release_b200.optim import RMSprop  # noqa: E402

LR = 1e-3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    return torch.cuda.get_device_name(0), "unknown"


def stats(ts):
    ts = sorted(ts)
    return {"median_ms": round(ts[len(ts) // 2], 4), "min_ms": round(ts[0], 4), "max_ms": round(ts[-1], 4)}


def timed(sides, rounds, warmup, flush):
    """sides: {name: fn}.  Alternates the sides round by round; returns {name: (device ms list, host us list)}."""
    for fn in sides.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    out = {k: ([], []) for k in sides}
    for _ in range(rounds):
        for k, fn in sides.items():
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            h = time.perf_counter()
            fn()
            h = time.perf_counter() - h
            b.record()
            b.synchronize()
            out[k][0].append(a.elapsed_time(b))
            out[k][1].append(h * 1e6)
    return out


def posenet_model():
    from pose2mesh_release_b200 import posenet

    torch.manual_seed(0)
    return posenet.get_model(17, 4096, 2, 0.5)


def flat_smpl_model():
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200.pose2mesh_net import FlatPose2Mesh

    face = pg.synthetic_sphere_faces(6890, 2)
    _, graph_L, _, _ = pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=9)
    torch.manual_seed(0)
    return FlatPose2Mesh(17, graph_L)


def step_set(model, rounds, warmup, flush):
    """The optimizer step alone over the model's parameter set (PoseNet's unused batch_norm1 gets no gradient)."""
    model = model.cuda()
    skip = {id(p) for m in model.modules() if hasattr(m, "batch_norm1") and hasattr(m, "linear_stages")
            for p in m.batch_norm1.parameters()}
    gen = torch.Generator(device="cuda").manual_seed(1)
    src = [p.detach() for p in model.parameters()]
    grads = [None if id(p) in skip else torch.randn(p.shape, device="cuda", generator=gen) * 1e-2
             for p in model.parameters()]
    sides = {}
    for name, cls in (("native", RMSprop), ("torch", torch.optim.RMSprop)):
        ps = [torch.nn.Parameter(t.clone()) for t in src]
        for p, g in zip(ps, grads):
            p.grad = g
        sides[name] = cls(ps, lr=LR).step
    n_param = sum(g.numel() for g in grads if g is not None)
    lib = _lib.load()
    lib.p2m_launch_count_reset()
    sides["native"]()
    launches = lib.p2m_launch_count()
    res = timed(sides, rounds, warmup, flush)
    nbytes = 5 * 4 * n_param
    out = {"tensors": len(grads), "tensors_with_grad": sum(g is not None for g in grads), "parameters": n_param,
           "algorithmic_bytes": nbytes, "native_launches_per_step": launches}
    for k, (dev_ms, host_us) in res.items():
        s = stats(dev_ms)
        s["gb_per_s"] = round(nbytes / (s["median_ms"] * 1e-3) / 1e9, 1)
        s["host_us_median"] = round(sorted(host_us)[len(host_us) // 2], 1)
        out[k] = s
    out["torch_over_native"] = round(out["torch"]["median_ms"] / out["native"]["median_ms"], 3)
    return out


def lift_step(rounds, warmup, flush, B=64):
    """LiftTrainer.train's step: PoseNet train forward + backward (native), masked L1 (native CoordLoss), step."""
    gen = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(B, 34, device="cuda", generator=gen)
    tgt = torch.randn(B, 51, device="cuda", generator=gen)
    valid = (torch.rand(B, 51, device="cuda", generator=gen) > 0.1).float()
    loss_fn = CoordLoss(has_valid=True)
    sides = {}
    for name, cls in (("native", RMSprop), ("torch", torch.optim.RMSprop)):
        net = posenet_model().cuda().train()
        opt = cls(net.parameters(), lr=LR)

        def step(net=net, opt=opt):
            opt.zero_grad(set_to_none=True)
            loss_fn(net(x), tgt, valid).backward()
            opt.step()

        sides[name] = step
    res = timed(sides, rounds, warmup, flush)
    out = {"batch": B}
    for k, (dev_ms, host_us) in res.items():
        s = stats(dev_ms)
        s["host_us_median"] = round(sorted(host_us)[len(host_us) // 2], 1)
        out[k] = s
    out["torch_over_native"] = round(out["torch"]["median_ms"] / out["native"]["median_ms"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_rmsprop: no GPU")
    name, power = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > the H100's 50 MB L2
    clocks = ClockSampler(torch.cuda.current_device())
    clocks.start()
    clocks.mark()
    result = {"card": name, "power_limit": power, "lr": LR, "rounds": args.rounds,
              "l2": "256 MiB buffer written before every timed region (outside the events)",
              "posenet": step_set(posenet_model(), args.rounds, args.warmup, flush),
              "flat_smpl": step_set(flat_smpl_model(), args.rounds, args.warmup, flush),
              "lift_step_b64": lift_step(args.rounds, args.warmup, flush)}
    result["sm_clocks"] = clocks.stop()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
