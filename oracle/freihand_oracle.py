"""TEST INFRASTRUCTURE ONLY — float64 numpy restatement of the FreiHAND evaluation script (eval.py and
utils/eval_util.py of the FreiHAND repository) for MANO predictions, written as the script's per-sample loop.

    nearest(P, Q)                      brute-force nearest distances both ways, in row chunks
    fscore(gt, pred, th)               calculate_fscore -> (F, frac_gt, frac_pred)
    align_w_scale(gt, pred)            centre, Frobenius-normalise, scipy.linalg.orthogonal_procrustes, rescale
    EvalUtil                           per-keypoint errors, get_measures' PCK / AUC / mean EPE
    evaluate(...)                      the script's main loop over samples -> the reported measures

Every distance is np.sqrt((dx*dx + dy*dy) + dz*dz) in float64 on the inputs' values.  A sample holding a non-finite
coordinate gets NaN distances, NaN fractions and NaN F-scores (the script itself would stop in scipy's finiteness check).
"""
import numpy as np
from scipy.linalg import orthogonal_procrustes


def point_dist(a, b):
    """|a - b| per row, float64, ((dx^2 + dy^2) + dz^2)."""
    d = np.asarray(a, np.float64) - np.asarray(b, np.float64)
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def nearest(P, Q, chunk=512):
    """d_p[i] = min_j |P_i - Q_j|, d_q[j] = min_i |Q_j - P_i| for one sample ([n, 3], [m, 3])."""
    P, Q = np.asarray(P, np.float64), np.asarray(Q, np.float64)
    if not (np.isfinite(P).all() and np.isfinite(Q).all()):
        return np.full(len(P), np.nan), np.full(len(Q), np.nan)
    # squared distances ((dx*dx + dy*dy) + dz*dz) per chunk of rows; sqrt is correctly rounded and monotone, so the
    # sqrt of the minimum is the minimum of the distances, bit for bit
    d_p = np.empty(len(P))
    s_q = np.full(len(Q), np.inf)
    for i in range(0, len(P), chunk):
        p = P[i:i + chunk]
        s = np.subtract.outer(p[:, 0], Q[:, 0])
        s *= s
        for c in (1, 2):
            d = np.subtract.outer(p[:, c], Q[:, c])
            d *= d
            s += d
        d_p[i:i + chunk] = s.min(axis=1)
        np.minimum(s_q, s.min(axis=0), out=s_q)
    return np.sqrt(d_p), np.sqrt(s_q)


def fscore_from_distances(d_gt, d_pr, th):
    """calculate_fscore from both directed distance arrays: strict `<`, F = ((2 a) b) / (a + b), 0 when a + b = 0."""
    if np.isnan(d_gt).all() and np.isnan(d_pr).all():
        return np.nan, np.nan, np.nan
    a = float(np.sum(d_gt < th)) / float(len(d_gt))
    b = float(np.sum(d_pr < th)) / float(len(d_pr))
    f = ((2 * a) * b) / (a + b) if a + b > 0 else 0.0
    return f, a, b


def fscore(gt, pred, th):
    d_gt, d_pr = nearest(gt, pred)
    return fscore_from_distances(d_gt, d_pr, th)


def align_w_scale(gt, pred):
    """The script's align_w_scale(mtx1=gt, mtx2=pred): pred aligned onto gt, no reflection correction."""
    gt, pred = np.asarray(gt, np.float64), np.asarray(pred, np.float64)
    if not (np.isfinite(gt).all() and np.isfinite(pred).all()):
        return np.full(pred.shape, np.nan)
    t1, t2 = gt.mean(0), pred.mean(0)
    A, P = gt - t1, pred - t2
    s1 = np.linalg.norm(A) + 1e-8
    A = A / s1
    s2 = np.linalg.norm(P) + 1e-8
    P = P / s2
    R, s = orthogonal_procrustes(A, P)
    return (P @ R.T) * s * s1 + t1


class EvalUtil:
    """utils/eval_util.py: per-keypoint error lists (every point visible) and get_measures."""

    def __init__(self, num_kp):
        self.data = [[] for _ in range(num_kp)]

    def feed(self, gt, pred):
        e = point_dist(gt, pred)
        for k in range(len(self.data)):
            self.data[k].append(e[k])

    def counts(self, thresholds):
        """#(e <= t) over every (sample, keypoint) per threshold (int64)."""
        e = np.asarray(self.data, np.float64).reshape(-1)
        return np.array([np.sum(e <= t) for t in thresholds], np.int64)

    def get_measures(self, val_min, val_max, steps):
        thresholds = np.linspace(val_min, val_max, steps)
        norm = np.trapezoid(np.ones_like(thresholds), thresholds)
        auc_all, pck_all, epe_all = [], [], []
        for d in self.data:
            d = np.asarray(d)
            epe_all.append(np.mean(d))
            pck = np.array([np.mean((d <= t).astype("float")) for t in thresholds])
            pck_all.append(pck)
            auc_all.append(np.trapezoid(pck, thresholds) / norm)
        return float(np.mean(epe_all)), float(np.mean(auc_all)), np.mean(np.array(pck_all), 0), thresholds


def evaluate(gt_xyz, gt_verts, pred_xyz, pred_verts, thresholds=(0.005, 0.015), pck=(0.0, 0.05, 100)):
    """The script's loop over samples (MANO branch: keypoints and vertices aligned separately) -> dict with
    {kind}_mean3d, {kind}_auc3d, {kind}_pck, {kind}_counts for kind in xyz, pa_xyz, mesh, pa_mesh, and the mean F per
    threshold f_score / f_score_aligned."""
    n_kp, n_v = np.asarray(gt_xyz).shape[1], np.asarray(gt_verts).shape[1]
    ev = {"xyz": EvalUtil(n_kp), "pa_xyz": EvalUtil(n_kp), "mesh": EvalUtil(n_v), "pa_mesh": EvalUtil(n_v)}
    f, fa = [[] for _ in thresholds], [[] for _ in thresholds]
    for i in range(len(gt_xyz)):
        xyz, verts = gt_xyz[i], gt_verts[i]
        xyz_al = align_w_scale(xyz, pred_xyz[i])
        verts_al = align_w_scale(verts, pred_verts[i])
        ev["xyz"].feed(xyz, pred_xyz[i])
        ev["pa_xyz"].feed(xyz, xyz_al)
        ev["mesh"].feed(verts, pred_verts[i])
        ev["pa_mesh"].feed(verts, verts_al)
        d = nearest(verts, pred_verts[i])
        d_al = nearest(verts, verts_al)
        for j, th in enumerate(thresholds):
            f[j].append(fscore_from_distances(*d, th)[0])
            fa[j].append(fscore_from_distances(*d_al, th)[0])
    out = {"n_samples": len(gt_xyz)}
    for k, e in ev.items():
        mean, auc, curve, t = e.get_measures(*pck)
        out[f"{k}_mean3d"], out[f"{k}_auc3d"], out[f"{k}_pck"] = mean, auc, curve
        out[f"{k}_counts"] = e.counts(t)
    out["f_score"] = np.array([np.mean(x) for x in f])
    out["f_score_aligned"] = np.array([np.mean(x) for x in fa])
    return out
