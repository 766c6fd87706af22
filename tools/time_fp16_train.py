"""Timing aid (needs a GPU): the training step at the single-pass mixed precision (fp16_mixed) against fp16x3.

    python tools/time_fp16_train.py [--rounds 10] [--steps 10] [--warmup 3] [--out FILE]

bench.py's training workload: the seeded SMPL-size model (randomised BatchNorm) at B = 256, and the MANO-size one at
B = 1024; one step is a train-mode forward, an L1 loss to seeded random targets and the backward.  After a warm-up the
two precisions alternate round by round in one process, each round timed with device events over --steps steps.
Records, per workload:
  * median / min / max ms per step and meshes/s per precision, and whether fp16_mixed was faster in every round;
  * a torch.profiler pass of its own (two steps per precision), whose kernels are split into the forward convs, the
    T1 passes, backward-data (the convs and dT GEMMs of the backward), dW, BatchNorm and elementwise work, and the rest
    (with every kernel's total, so that the split can be checked);
  * the deviation of one step from fp16x3's, from the same parameters and inputs: the largest per-mesh
    max|dy| / max|y|, both losses, and per parameter tensor max|dg| / max|g|;
  * the card's name, power limit and the SM clock sampled during the timed rounds, read in the same run.
Prints one JSON line (also written to --out)."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

import bench  # noqa: E402
from time_fp16_forward import card, workload  # noqa: E402

PRECISIONS = ("fp16x3", "fp16_mixed")


def make_step(model, x, tgt):
    def step():
        model.zero_grad(set_to_none=True)
        y = model(x)
        loss = (y - tgt).abs().mean()
        loss.backward()
        return y, loss
    return step


def kernel_class(name, backward):
    n = name.lower()
    if "k_cheb_dw" in n:
        return "dw"
    if "k_cheb_t1" in n:
        return "t1"
    if "k_cheb_conv" in n:
        return "backward_data" if backward else "forward_conv"
    if any(k in n for k in ("bn", "affine", "relu", "elementwise", "reduce", "absmax", "scale", "fill", "unpool",
                            "resample", "abs", "mean")):
        return "batchnorm_elementwise"
    return "rest"


def profile(model, step, precision, reps=2):
    """Device time per class (ms per step) and per kernel, from torch.profiler: the forward and the backward are
    profiled apart, so a conv kernel is counted as forward or backward-data by the pass that launched it."""
    from torch.profiler import ProfilerActivity, profile as prof

    model.set_precision(precision)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    classes, kernels = {}, {}
    for _ in range(reps):
        model.zero_grad(set_to_none=True)
        with prof(activities=[ProfilerActivity.CUDA]) as pf:
            y = model(step.x)
            loss = (y - step.tgt).abs().mean()
            torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as pb:
            loss.backward()
            torch.cuda.synchronize()
        for p, bwd in ((pf, False), (pb, True)):
            for e in p.key_averages():
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                if t <= 0 or e.key.startswith("cuda") or e.key.startswith("Memcpy"):
                    continue
                c = kernel_class(e.key, bwd)
                classes[c] = classes.get(c, 0.0) + t / 1e3 / reps
                k = ("bwd " if bwd else "fwd ") + e.key[:120]
                kernels[k] = kernels.get(k, 0.0) + t / 1e3 / reps
    return {"classes_ms": classes, "kernels_ms": dict(sorted(kernels.items(), key=lambda kv: -kv[1]))}


def deviation(model, step):
    """One step at each precision from the same parameters, buffers and inputs."""
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    out = {}
    for p in PRECISIONS:
        model.load_state_dict(sd)
        model.set_precision(p)
        y, loss = step()
        torch.cuda.synchronize()
        out[p] = (y.detach().double(), float(loss),
                  {n: q.grad.detach().double() for n, q in model.named_parameters() if q.grad is not None})
    model.load_state_dict(sd)
    (y3, l3, g3), (ym, lm, gm) = out["fp16x3"], out["fp16_mixed"]
    per_mesh = ((ym - y3).abs().flatten(1).max(dim=1).values / y3.abs().flatten(1).max(dim=1).values).max().item()
    grads = {n: ((gm[n] - g3[n]).abs().max() / g3[n].abs().max().clamp_min(1e-30)).item() for n in g3}
    worst = max(grads, key=grads.get)
    return {"max_per_mesh_dy": per_mesh, "loss": {"fp16x3": l3, "fp16_mixed": lm},
            "grad_rel_max": grads, "grad_rel_worst": [worst, grads[worst]]}


def measure(mesh, B, rounds, steps, warmup, dev, sampler):
    model, x = workload(mesh, B, dev)
    model.train()
    tgt = torch.randn(B, model.num_vertices, 3, generator=torch.Generator().manual_seed(7)).to(dev)
    step = make_step(model, x, tgt)
    step.x, step.tgt = x, tgt
    res = {"batch": B, "deviation": deviation(model, step)}
    times = {p: [] for p in PRECISIONS}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if sampler is not None:
        sampler.mark()
    for r in range(warmup + rounds):
        order = PRECISIONS if r % 2 == 0 else PRECISIONS[::-1]
        for p in order:
            model.set_precision(p)
            step()                      # the first step after a switch is not timed
            a.record()
            for _ in range(steps):
                step()
            b.record()
            b.synchronize()
            if r >= warmup:
                times[p].append(a.elapsed_time(b) / steps)
    res["sm_clock"] = sampler.stop() if sampler is not None else None
    res["step_ms"], res["meshes_per_s"] = {}, {}
    for p in PRECISIONS:
        t = times[p]
        res["step_ms"][p] = {"median": statistics.median(t), "min": min(t), "max": max(t), "all": t}
        res["meshes_per_s"][p] = {"median": B * 1e3 / statistics.median(t), "min": B * 1e3 / max(t),
                                  "max": B * 1e3 / min(t)}
    res["speedup_median"] = statistics.median(times["fp16x3"]) / statistics.median(times["fp16_mixed"])
    res["rounds_fp16_mixed_not_faster"] = [i for i, (tm, t3) in enumerate(zip(times["fp16_mixed"], times["fp16x3"]))
                                           if tm >= t3]
    res["profile"] = {p: profile(model, step, p) for p in PRECISIONS}
    model.set_precision("fp16x3")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_fp16_train: no GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"tool": "time_fp16_train", "card": card(), "rounds": args.rounds, "steps_per_round": args.steps}
    for mesh, B in (("smpl", 256), ("mano", 1024)):
        sampler = bench.ClockSampler(0)
        sampler.start()
        res[f"{mesh}_b{B}"] = measure(mesh, B, args.rounds, args.steps, args.warmup, dev, sampler)
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
