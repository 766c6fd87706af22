"""TEST INFRASTRUCTURE ONLY — numpy restatement of the temporal-metric kernels (csrc/temporal.cu, SURVEY.md §8 f8).

    one_euro(x, ...)         k_one_euro: smooth_utils.smooth_pose / OneEuroFilter (lib/smooth_utils.py:5-72), in the
                             input's dtype T, one operation at a time in the kernel's order
    accel_error(gt, pred)    k_accel_error: coord_utils.compute_error_accel (lib/coord_utils.py:194-222) per window,
                             with the window-valid flags instead of the compaction
    row_sum(v)               numpy's np.add.reduce over the last axis of a C-contiguous [M, n] array (n <= 128)
    segment_means(...)       k_segment_mean in fp64 (summation order differs from the kernel's; compare with rtol)
    evaluate_video_f64(...)  the video block of PW3D.evaluate (data/PW3D/dataset.py:387-415), float64, per video

The keyword switches of one_euro and accel_error are mutations: tests/test_temporal_cpu.py shows the reference
fixture tells each of them from the reference's arithmetic.
"""
import math

import numpy as np

from oracle import metrics_oracle


def one_euro(x, min_cutoff, beta, d_cutoff=1.0, t=None, fma=False, weights_swapped=False, cutoff_2pi_in_double=False,
             beta_on_raw_dx=False, unit_te=False):
    """The One-Euro filter along axis 0 of x [N, ...] in x's dtype.  t: per-frame times [N] (default: the frame
    index, as smooth_pose passes); frame 0 is copied and starts the filter with x_prev = x[0], dx_prev = 0,
    t_prev = 0 (smooth_pose's zeros_like(pred_pose[0]); a OneEuroFilter built with t0 = t[0] is the same filter on
    t - t[0])."""
    x = np.asarray(x)
    T = x.dtype.type
    one = T(1)
    two_pi, two_pi_d = T(2 * math.pi), T(2 * math.pi * d_cutoff)
    mc, b = T(min_cutoff), T(beta)
    times = np.arange(len(x)) if t is None else np.asarray(t)
    y = np.empty_like(x)
    y[0] = x[0]
    x_prev, dx_prev, t_prev = x[0].copy(), np.zeros_like(x[0]), np.zeros_like(x[0])
    if t is not None:
        t_prev = t_prev + T(times[0])
    with np.errstate(all="ignore"):
        for i in range(1, len(x)):
            tt = np.full_like(x[0], T(times[i]))
            te = np.ones_like(tt) if unit_te else tt - t_prev
            r_d = two_pi_d * te
            a_d = r_d / (r_d + one)
            dx = (x[i] - x_prev) / te
            dx_hat = a_d * dx + (one - a_d) * dx_prev
            cutoff = mc + b * np.abs(dx if beta_on_raw_dx else dx_hat)
            if cutoff_2pi_in_double:
                r = (2 * math.pi * cutoff.astype(np.float64)).astype(T) * te
            else:
                r = (two_pi * cutoff) * te
            a = r / (r + one)
            if weights_swapped:
                x_hat = a * x_prev + (one - a) * x[i]
            elif fma:  # a * x + c with one rounding: the product is exact in the wider type
                wide = np.longdouble if T is np.float64 else np.float64
                x_hat = (a.astype(wide) * x[i].astype(wide) + ((one - a) * x_prev).astype(wide)).astype(T)
            else:
                x_hat = a * x[i] + (one - a) * x_prev
            y[i] = x_hat
            x_prev, dx_prev, t_prev = x_hat, dx_hat, tt
    return y


def row_sum(v):
    """np.add.reduce(v, axis=-1) for C-contiguous v [M, n], n <= 128, restated: the identity 0 plus numpy's pairwise
    sum of all n values (sequential below 8; else eight strided accumulators, a fixed tree, the tail in order)."""
    v = np.asarray(v)
    T = v.dtype.type
    n = v.shape[-1]
    with np.errstate(all="ignore"):
        if n < 8:
            res = np.zeros(v.shape[:-1], v.dtype)
            for i in range(n):
                res = res + v[..., i]
        else:
            r = [v[..., j].copy() for j in range(8)]
            i = 8
            while i < n - n % 8:
                for j in range(8):
                    r[j] = r[j] + v[..., i + j]
                i += 8
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            for k in range(i, n):
                res = res + v[..., k]
        return T(0) + res


def accel_error(gt, pred, vis=None, vis_first_frame_only=False, naive_mean=False):
    """(per_window [N - 2], valid [N - 2]) of one sequence [N, J, 3], in the input's dtype; N < 3 gives empty arrays."""
    gt, pred = np.asarray(gt), np.asarray(pred)
    T = gt.dtype.type
    n = max(len(gt) - 2, 0)
    with np.errstate(all="ignore"):
        ag = (gt[:-2] - T(2) * gt[1:-1]) + gt[2:]
        ap = (pred[:-2] - T(2) * pred[1:-1]) + pred[2:]
        d = (ap - ag)[:n]
        e = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
        J = gt.shape[1]
        if naive_mean:
            s = np.zeros(n, gt.dtype)
            for j in range(J):
                s = s + e[:, j]
        else:
            s = row_sum(e)
        per_window = (s / T(J)).astype(gt.dtype)
    if vis is None:
        valid = np.ones(n, bool)
    else:
        v = np.asarray(vis).astype(bool)
        valid = v[:n].copy() if vis_first_frame_only else (v[:n] & v[1:n + 1] & v[2:n + 2])
    return per_window, valid


def segment_means(values, lengths, valid=None, width=1):
    """fp64 mean of each segment's (valid) rows; NaN for a segment with none."""
    values = np.asarray(values, dtype=np.float64).reshape(-1, width)
    out, start = [], 0
    for n in lengths:
        rows = values[start:start + n]
        if valid is not None:
            rows = rows[np.asarray(valid[start:start + n], bool)]
        out.append(rows.mean() if rows.size else np.nan)
        start += n
    return np.array(out)


def evaluate_video_f64(pred_j3d, gt_j3d, video_indices, smooth=True, min_cutoff=0.004, beta=0.005):
    """The reference's video block in float64, one video at a time: smooth, accel error, MPJPE, per-frame Procrustes.
    -> (per-video accel, per-video MPJPE, per-frame PA-MPJPE [n, J], accel total, MPJPE total, PA-MPJPE total)."""
    pred_j3d, gt_j3d = np.asarray(pred_j3d, np.float64), np.asarray(gt_j3d, np.float64)
    accel, mpjpe, pa = [], [], []
    with np.errstate(all="ignore"):
        for vid in video_indices:
            pred, gt = pred_j3d[vid], gt_j3d[vid]
            if smooth:
                pred = one_euro(pred, min_cutoff, beta)
            per_window, _ = accel_error(gt, pred)
            accel.append(per_window.mean() if per_window.size else np.nan)
            mpjpe.append(np.sqrt(((pred - gt) ** 2).sum(2)).mean())
            for i in range(len(pred)):
                aligned = metrics_oracle.rigid_align(pred[i], gt[i])
                pa.append(np.sqrt(((aligned - gt[i]) ** 2).sum(1)))
    pa = np.array(pa)
    return np.array(accel), np.array(mpjpe), pa, np.mean(accel), np.mean(mpjpe), pa.mean()
