"""PoseNet's train step layer by layer against float64: every operation of p2m_posenet_train_forward_opts and of the
backward (p2m_debug_posenet_backward_capture) from the fp32 tensors the device itself produced, with one float64 value
and one element-wise bound per operation (fp64_ref's precision models).  Nothing is chained: each layer's inputs are
the device's, so a bound never grows with depth.  The ReLU masks are the device's own, reproduced bit for bit from
the saved pre-activation statistics (fp64_ref.relu_mask), so no entry near zero can take the other branch in float64.

check_step returns, per quantity, the worst max |err| / bound (<= 1 passes), the bitwise checks that failed, and the
number of pre-activations whose float64 value is within its own forward bound of zero (the entries a chained float64
reference cannot place on either side of the ReLU)."""
from __future__ import annotations

import numpy as np

import fp64_ref as R
from posenet_train_ref import dropout_multiplier

U32 = R.U32
ALIGN = 256                # every array of `saved` starts at a multiple of 256 bytes (include/p2m_b200.h)
BATCH_UPDATE, BATCH, RUNNING = 0, 1, 2


def parse_saved(saved: np.ndarray, B: int, H: int, S: int):
    """`saved` (uint8) as include/p2m_b200.h lays it out: (y [S + 1] of [B, H], z2 [S] of [B, H], stats[s][bn] = (mean,
    invstd, scale, shift) [H] each, the bytes the layout covers)."""
    off = 0

    def take(n):
        nonlocal off
        a = saved[off:off + 4 * n].view(np.float32)
        off += -(-4 * n // ALIGN) * ALIGN
        return a

    y = [take(B * H).reshape(B, H) for _ in range(S + 1)]
    z2 = [take(B * H).reshape(B, H) for _ in range(S)]
    stats = [[tuple(take(H) for _ in range(4)) for _ in range(2)] for _ in range(S)]
    return y, z2, stats, off


def activation(z, scale, shift, mult):
    """drop(relu(fmaf(z, scale, shift))) as k_pn_bn_relu_drop computes it, up to the double rounding of the float64 sum
    (at most one ulp of the pre-activation), and the device's exact ReLU mask."""
    f32 = np.float32
    pre = (np.asarray(z, f32).astype(np.float64) * np.asarray(scale, f32) + np.asarray(shift, f32)).astype(f32)
    return (np.maximum(pre, f32(0)) * mult.astype(f32)).astype(f32), R.relu_mask(z, scale, shift)


class Checks:
    """Collects max |err| / bound per quantity class, and the names of failed bitwise checks."""

    def __init__(self):
        self.ratio, self.bitwise = {}, []

    def bound(self, cls, got, ref, bd):
        r = R.bound_ratio(got, ref, bd)
        self.ratio[cls] = max(self.ratio.get(cls, 0.0), r)
        return r

    def equal(self, name, got, want):
        if not np.array_equal(np.asarray(got), np.asarray(want)):
            self.bitwise.append(name)


def _gemm(chk, cls, got, A, Bm, prec, b_side="fixed", add=None, res=None):
    """got ~ A @ Bm (+ add, a bias row, + res, a residual) with the GEMM's bound and one rounding per addition."""
    o = np.asarray(A, np.float64) @ np.asarray(Bm, np.float64)
    bd = R.dense_gemm_bound(A, Bm, prec, b_side)
    ref = o
    if add is not None:
        ref = ref + add
        bd = bd + U32 * np.abs(ref)
    if res is not None:
        ref = ref + res
        bd = bd + U32 * np.abs(ref)
    return chk.bound(cls, got, ref, bd)


def check_step(sd, sd_after, x, d_out, seed, modes, p_stage, res, J: int, H: int, S: int, saved_bytes: int):
    """sd / sd_after: the module's state_dict (numpy) before / after the step; modes: per BatchNorm (bn1 of stage s at
    2 s, bn2 at 2 s + 1) a dict(stats, cumulative, momentum, eps); p_stage: each stage's dropout p; res: the numpy
    results of posenet.debug_train_step_capture with every field captured.  Returns (Checks, near-zero count)."""
    f32, f64 = np.float32, np.float64
    chk = Checks()
    x = np.asarray(x, f32)
    B = x.shape[0]
    tc = H % 64 == 0
    prec = "fp16x3" if tc else "fp32"
    W = {k: np.asarray(v, f64) for k, v in sd.items()}
    y, z2, stats, nbytes = parse_saved(res["saved"], B, H, S)
    chk.equal("saved layout covers p2m_posenet_train_saved_bytes", nbytes, saved_bytes)
    near_zero = 0

    # ------------------------------------------------------------------------------------------------------ forward
    _gemm(chk, "fwd.y0", y[0], x, W["w1.weight"].T, "fp32", add=W["w1.bias"])
    acts = []
    for s in range(S):
        p = f"linear_stages.{s}."
        pair = []
        for which, (name, z) in enumerate((("batch_norm1.", y[s]), ("batch_norm2.", z2[s]))):
            o = modes[2 * s + which]
            bn = p + name
            gam, bet, rm, rv = (W[bn + k] for k in ("weight", "bias", "running_mean", "running_var"))
            mean, invstd, scale, shift = stats[s][which]
            nbt0, nbt1 = int(sd[bn + "num_batches_tracked"]), int(sd_after[bn + "num_batches_tracked"])
            eps = o["eps"]
            if o["stats"] == RUNNING:        # k_bn_fold_eval: running statistics, buffers untouched
                sc64 = gam / np.sqrt(rv + eps)
                chk.equal(bn + "frozen mean", mean, sd[bn + "running_mean"])
                chk.bound("fwd.bn.invstd", invstd, 1 / np.sqrt(rv + eps), 4 * U32 / np.sqrt(rv + eps))
                chk.bound("fwd.bn.scale", scale, sc64, 4 * U32 * np.abs(sc64))
                sh64 = bet - rm * sc64
                chk.bound("fwd.bn.shift", shift, sh64, 5 * U32 * np.abs(rm * sc64) + U32 * np.abs(sh64))
                pre64 = z.astype(f64) * sc64 + sh64
                e_pre = (np.abs(z) * 4 * U32 * np.abs(sc64) + 5 * U32 * np.abs(rm * sc64) + U32 * np.abs(sh64)
                         + U32 * np.abs(pre64))
            else:
                mom = 1.0 / nbt1 if o["cumulative"] and o["stats"] == BATCH_UPDATE else o["momentum"]
                y64, mean64, var64, rm64, rv64 = R.bn_train_fwd(z, gam, bet, rm, rv, eps=eps, momentum=mom)
                bd = R.bn_train_fwd_bound(z, np.zeros_like(z, f64), gam, bet, rm, rv, eps=eps, momentum=mom)
                is64 = 1 / np.sqrt(var64 + eps)
                chk.bound("fwd.bn.mean", mean, mean64, bd["mean"])
                chk.bound("fwd.bn.invstd", invstd, is64, bd["invstd"])
                sc64 = gam * is64
                e_sc = np.abs(gam) * bd["invstd"] + U32 * np.abs(sc64)
                chk.bound("fwd.bn.scale", scale, sc64, e_sc)
                sh64 = bet - mean64 * sc64
                chk.bound("fwd.bn.shift", shift, sh64, np.abs(sc64) * bd["mean"] + np.abs(mean64) * e_sc
                          + 2 * U32 * np.abs(mean64 * sc64) + U32 * np.abs(sh64))
                if o["stats"] == BATCH_UPDATE:
                    chk.bound("fwd.bn.running_mean", sd_after[bn + "running_mean"], rm64, bd["rm"])
                    chk.bound("fwd.bn.running_var", sd_after[bn + "running_var"], rv64, bd["rv"])
                pre64, e_pre = y64, bd["y"]
            if o["stats"] != BATCH_UPDATE:
                for k in ("running_mean", "running_var"):
                    chk.equal(bn + k + " unchanged", sd_after[bn + k], sd[bn + k])
            chk.equal(bn + "num_batches_tracked", nbt1, nbt0 + (o["stats"] == BATCH_UPDATE))
            near_zero += int((np.abs(pre64) <= e_pre).sum())
            mult = dropout_multiplier(seed, 2 * s + which, B * H, p_stage[s]).reshape(B, H)
            a_dev = res["a1" if which == 0 else "a2"][s]
            a_emu, mask = activation(z, scale, shift, mult)
            chk.equal(bn + "activation zero pattern", a_dev != 0, mask & (mult != 0))
            chk.bound("fwd.act.ulp", a_dev, a_emu.astype(f64), np.spacing(np.abs(a_emu)).astype(f64))
            a64 = np.maximum(pre64, 0.0) * mult
            chk.bound("fwd.act.fp64", a_dev, a64, mult * e_pre + U32 * np.abs(a64))
            pair.append((a_dev, mask, mult))
        a1, a2 = pair[0][0], pair[1][0]
        _gemm(chk, "fwd.z2", z2[s], a1, W[p + "w1.weight"].T, prec, add=W[p + "w1.bias"])
        _gemm(chk, "fwd.y", y[s + 1], a2, W[p + "w2.weight"].T, prec, add=W[p + "w2.bias"], res=y[s].astype(f64))
        acts.append(pair)
    out_prec = "fp16x3" if tc and 3 * J <= 64 else "fp32"
    _gemm(chk, "fwd.out", res["out"], y[S], W["w2.weight"].T, out_prec, add=W["w2.bias"])
    comb = res["combine"].reshape(B, J, 5)
    chk.equal("pose_combine pose2d", comb[..., :2], x.reshape(B, J, 2))
    chk.equal("pose_combine pose3d / 1000", comb[..., 2:], (res["out"].reshape(B, J, 3) / f32(1000)).astype(f32))

    # ----------------------------------------------------------------------------------------------------- backward
    grads = res["grads"]          # LinearModel._trained_tensors() order
    d_out = np.asarray(d_out, f32)

    def col_sum(cls, got, g):
        chk.bound(cls, got, g.astype(f64).sum(axis=0), R.col_sum_bound(g))

    col_sum("bwd.db2", grads[3], d_out)
    _gemm(chk, "bwd.dW2", grads[2], d_out.T, y[S], "fp32")
    g_top = res["g_y"][S - 1] if S else res["g_y0"]
    _gemm(chk, "bwd.g_y", g_top, d_out, W["w2.weight"], "fp32")
    for s in reversed(range(S)):
        p = f"linear_stages.{s}."
        gs = grads[4 + 8 * s:12 + 8 * s]    # w1_w, w1_b, w2_w, w2_b, bn1_w, bn1_b, bn2_w, bn2_b
        g_y = res["g_y"][s]
        (a1, mask1, mult1), (a2, mask2, mult2) = acts[s]
        if tc:
            want = [R._pow2_scale(float(np.abs(t).max())) for t in (a2, g_y, a1, res["g_z2"][s])]
            chk.equal(p + "range-normalisation scales", res["scale"][s], np.asarray(want, f32))
        col_sum("bwd.db_b", gs[3], g_y)
        _gemm(chk, "bwd.dW_b", gs[2], g_y.T, a2, prec, b_side="normalised")
        _gemm(chk, "bwd.g_a2", res["g_a2"][s], g_y, W[p + "w2.weight"], prec)
        for which, (z, g_a, g_z, dgam, dbet, mask, mult) in (
                (1, (z2[s], res["g_a2"][s], res["g_z2"][s], gs[6], gs[7], mask2, mult2)),
                (0, (y[s], res["g_a1"][s], res["g_bn1"][s], gs[4], gs[5], mask1, mult1))):
            bn = p + ("batch_norm1." if which == 0 else "batch_norm2.")
            o = modes[2 * s + which]
            gam, bet = W[bn + "weight"], W[bn + "bias"]
            gp = (g_a * mult.astype(f32)).astype(f32)           # k_pn_drop_bwd: one fp32 product
            if o["stats"] == RUNNING:
                gm = np.where(mask, gp, f32(0))
                ref = R.bn_frozen_bwd(z, gm, gam, W[bn + "running_mean"], W[bn + "running_var"], o["eps"])
                bds = R.bn_frozen_bwd_bound(z, gm, gam, W[bn + "running_mean"], W[bn + "running_var"], o["eps"])
            else:
                ref = R.bn_train_bwd(z, gp, gam, bet, eps=o["eps"], mask=mask)[:3]
                bds = R.bn_train_bwd_bound(z, gp, gam, bet, eps=o["eps"], mask=mask)
            for cls, got, r, b in zip(("bwd.g_z", "bwd.dgamma", "bwd.dbeta"), (g_z, dgam, dbet), ref, bds):
                chk.bound(cls, got, r, b)
            if which == 1:
                col_sum("bwd.db_a", gs[1], g_z)
                _gemm(chk, "bwd.dW_a", gs[0], g_z.T, a1, prec, b_side="normalised")
                _gemm(chk, "bwd.g_a1", res["g_a1"][s], g_z, W[p + "w1.weight"], prec)
        below = res["g_y"][s - 1] if s else res["g_y0"]
        chk.equal(p + "residual gradient g_y + g_bn1", below, (g_y + res["g_bn1"][s]).astype(f32))
    g0 = res["g_y0"]
    col_sum("bwd.db1", grads[1], g0)
    _gemm(chk, "bwd.dW1", grads[0], g0.T, x, "fp32")
    _gemm(chk, "bwd.dx", res["dx"], g0, W["w1.weight"], "fp32")
    return chk, near_zero
