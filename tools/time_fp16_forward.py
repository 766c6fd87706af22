"""Timing aid (needs a GPU): the eval forward at the single-pass fp16 precision against fp16x3.

    python tools/time_fp16_forward.py [--rounds 20] [--steps 20] [--out FILE]

The bench.py workload (SMPL-size hierarchy, seeded weights, randomised BatchNorm, B = 256) and the MANO-size one
(B = 1024): the eval forward of each precision is captured once as a CUDA graph and the two graphs are replayed
alternately, round by round after a warm-up, each round timed with device events over --steps replays.  Then each
precision runs eagerly with per-layer profiling (p2m_model_layer_times_ms; median over --rounds forwards).  Records,
per workload: median / min / max ms per step and meshes/s per precision, the per-layer device times, and the largest
per-mesh deviation max|y_fp16 - y_fp16x3| / max|y_fp16x3|; and the card's name, power limit and the SM clock sampled
during the timed rounds, all read in the same run.  Prints one JSON line (also written to --out)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from pose2mesh_release_b200.meshnet import Pose2Mesh  # noqa: E402

PRECISIONS = ("fp16x3", "fp16")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(mesh, B, dev):
    graph_L, _ = bench.build_problem(mesh)
    torch.manual_seed(123)
    model = Pose2Mesh(5, 3, graph_L, joint_set="mano" if mesh == "mano" else "human36")
    model.load_state_dict(bench.randomize_bn_({k: v.clone() for k, v in model.state_dict().items()}))
    model = model.to(dev).eval()
    n_joint = 21 if mesh == "mano" else 17
    x = torch.randn(B, n_joint, 5, generator=torch.Generator().manual_seed(1000)).to(dev)
    return model, x


def capture(model, x, precision):
    model.set_precision(precision)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            model(x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        y = model(x)
    return g, y


def measure(mesh, B, rounds, steps, warmup, dev, sampler):
    model, x = workload(mesh, B, dev)
    graphs = {p: capture(model, x, p) for p in PRECISIONS}
    times = {p: [] for p in PRECISIONS}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if sampler is not None:
        sampler.mark()
    for r in range(warmup + rounds):
        order = PRECISIONS if r % 2 == 0 else PRECISIONS[::-1]
        for p in order:
            g = graphs[p][0]
            a.record()
            for _ in range(steps):
                g.replay()
            b.record()
            b.synchronize()
            if r >= warmup:
                times[p].append(a.elapsed_time(b) / steps)
    clocks = sampler.stop() if sampler is not None else None
    y3, y16 = graphs["fp16x3"][1].double(), graphs["fp16"][1].double()
    dev_mesh = ((y16 - y3).abs().flatten(1).max(dim=1).values / y3.abs().flatten(1).max(dim=1).values).max().item()
    # per-layer device times, eager forwards with profiling on
    d = dev.index or 0
    model._hier.set_profiling(d, True)
    layers = {}
    info = model._hier.layer_info(d)
    for p in PRECISIONS:
        model.set_precision(p)
        per = []
        with torch.no_grad():
            for r in range(warmup + rounds):
                model(x)
                if r >= warmup:
                    per.append(model._hier.layer_times_ms(d))
        layers[p] = [statistics.median(v[i] for v in per) for i in range(len(info))]
    model._hier.set_profiling(d, False)
    res = {"batch": B, "step_ms": {}, "meshes_per_s": {}, "max_per_mesh_dev_fp16_vs_fp16x3": dev_mesh,
           "layers": [{"layer": i, "V": L["V"], "fin": L["fin"], "fout": L["fout"],
                       **{f"{p}_ms": layers[p][i] for p in PRECISIONS}} for i, L in enumerate(info)]}
    for p in PRECISIONS:
        t = times[p]
        res["step_ms"][p] = {"median": statistics.median(t), "min": min(t), "max": max(t)}
        res["meshes_per_s"][p] = {"median": B * 1e3 / statistics.median(t), "min": B * 1e3 / max(t),
                                  "max": B * 1e3 / min(t)}
    res["speedup_median"] = statistics.median(times["fp16x3"]) / statistics.median(times["fp16"])
    res["fp16_faster_every_round"] = all(t16 < t3 for t16, t3 in zip(times["fp16"], times["fp16x3"]))
    res["sm_clock"] = clocks
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_fp16_forward: no GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"tool": "time_fp16_forward", "card": card(), "rounds": args.rounds, "steps_per_round": args.steps}
    for mesh, B in (("smpl", 256), ("mano", 1024)):
        sampler = bench.ClockSampler(0)
        sampler.start()
        res[f"{mesh}_b{B}"] = measure(mesh, B, args.rounds, args.steps, args.warmup, dev, sampler)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
