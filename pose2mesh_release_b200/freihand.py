"""The FreiHAND benchmark's scores on the GPU (SURVEY.md §8 row f9), as the dataset's evaluation script (eval.py and
utils/eval_util.py of the FreiHAND repository) defines them for MANO predictions:

    nearest_distances(P, Q)               per point, the distance to the nearest point of the other set, both ways
    f_scores(gt, pred, thresholds)        calculate_fscore: F and both directed fractions per threshold
    align_w_scale(gt, pred)               centre, Frobenius-normalise, orthogonal Procrustes (reflections allowed)
    mano_eval_regressor(J_regressor)      the 21-row evaluation regressor of lib/_mano.py:22-30
    FreiHANDEvaluator                     the script's measures over a test set, fed batch by batch

Everything runs in libp2m_b200.so (p2m_nearest_distances, p2m_align_w_scale, p2m_pck_accumulate, p2m_segment_mean);
CUDA tensors only.  Point sets are [B, n, 3] or [n, 3] (one sample), in the unit of the data (FreiHAND: metres).  All
arithmetic is fp64 on the float32 (or float64) inputs; distances equal the float64 brute force bit for bit, and counts
and F-scores do not depend on how samples are batched.  install() does not rebind anything: the reference's
evaluation writes pred.json and takes numpy arrays per sample.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .temporal import _segment_mean

FSCORE_THRESHOLDS = (0.005, 0.015)  # F@5 mm and F@15 mm, in metres
PCK_RANGE = (0.0, 0.05, 100)        # EvalUtil.get_measures(0.0, 0.05, 100)
# lib/_mano.py:22-30: fingertip one-hot rows appended to the MANO J_regressor, then reordered to FreiHAND's 21 joints.
# The middle tip is vertex 445 there, although fingertip_vertex_idx lists 444.
MANO_EVAL_TIPS = (745, 317, 445, 556, 673)
MANO_EVAL_ORDER = (0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20)
_DTYPES = {torch.float32: _lib.P2M_DTYPE_F32, torch.float64: _lib.P2M_DTYPE_F64}
_MAX_F_THRESHOLDS = 16
_MAX_PCK_THRESHOLDS = 128


def _points(x, what: str, dtypes=(torch.float32,)) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.dim() == 2:
        x = x.unsqueeze(0)
    if x.dim() != 3 or x.shape[-1] != 3 or x.shape[0] == 0 or x.shape[1] == 0:
        raise ValueError(f"{what} must be [B, n, 3] or [n, 3] with B, n > 0; got {tuple(x.shape)}")
    if x.dtype not in dtypes:
        raise ValueError(f"{what} must be {' or '.join(str(d) for d in dtypes)}; got {x.dtype}")
    return x.contiguous()


def _same_batch(a, b, names):
    if a.shape[0] != b.shape[0] or a.device != b.device:
        raise ValueError(f"{names[0]} {tuple(a.shape)} on {a.device} and {names[1]} {tuple(b.shape)} on {b.device} "
                         "must hold the same number of samples on one device")


def _thresholds(t, max_n: int, what: str = "thresholds"):
    """Host thresholds -> ctypes double array; finite, >= 0, sorted ascending, 1 .. max_n values."""
    a = np.asarray(t, dtype=np.float64).reshape(-1)
    if a.size == 0 or a.size > max_n:
        raise ValueError(f"{what}: need 1 .. {max_n} values; got {a.size}")
    if not np.isfinite(a).all() or (a < 0).any() or (np.diff(a) < 0).any():
        raise ValueError(f"{what} must be finite, non-negative and sorted ascending; got {a.tolist()}")
    return (C.c_double * a.size)(*a.tolist()), a


def _nearest(P, Q, thr=None, n_thr=0, dist=True, counts=False, frac=False, fscore=False):
    """One p2m_nearest_distances call on contiguous [B, n, 3] / [B, m, 3] tensors of one dtype."""
    B, n, m, dev = P.shape[0], P.shape[1], Q.shape[1], P.device
    f64 = dict(device=dev, dtype=torch.float64)
    dp = torch.empty((B, n), **f64) if dist else None
    dq = torch.empty((B, m), **f64) if dist else None
    cnt = torch.empty((B, 2, n_thr), device=dev, dtype=torch.int64) if counts else None
    fr = torch.empty((B, 2, n_thr), **f64) if frac else None
    fs = torch.empty((B, n_thr), **f64) if fscore else None
    _lib.call("p2m_nearest_distances", dev, _DTYPES[P.dtype], P, Q, B, n, m, thr, n_thr, dp, dq, cnt, fr, fs)
    return dp, dq, cnt, fr, fs


def _align(gt, pred, aligned_dtype=torch.float32, aligned=True, err=False):
    """One p2m_align_w_scale call on contiguous float32 [B, n, 3] tensors."""
    B, n = gt.shape[0], gt.shape[1]
    Y = torch.empty((B, n, 3), device=gt.device, dtype=aligned_dtype) if aligned else None
    E = torch.empty((B, n), device=gt.device, dtype=torch.float64) if err else None
    _lib.call("p2m_align_w_scale", gt.device, gt, pred, B, n, _DTYPES[aligned_dtype], Y, E)
    return Y, E


def _pck(hist, thr, n_thr, err=None, pred=None, gt=None, err_out=None):
    """One p2m_pck_accumulate call into hist (int64 [n_thr], accumulated)."""
    x = err if err is not None else pred
    _lib.call("p2m_pck_accumulate", x.device, err, pred, gt, x.numel() // (1 if err is not None else 3), thr, n_thr,
              err_out, hist)


# ---------------------------------------------------------------------------------------------- public functions
def nearest_distances(P: torch.Tensor, Q: torch.Tensor):
    """d_p [B, n] = min_j |P_i - Q_j| and d_q [B, m] = min_i |Q_j - P_i| (float64) for P [B, n, 3], Q [B, m, 3]
    (float32 or float64, one dtype; [n, 3] for one sample gives [n] / [m]).  Bit for bit the float64 brute force;
    a sample holding a non-finite coordinate gets NaN throughout."""
    squeeze = P.dim() == 2
    dts = tuple(_DTYPES)
    P, Q = _points(P, "P", dts), _points(Q, "Q", dts)
    _same_batch(P, Q, ("P", "Q"))
    if P.dtype != Q.dtype:
        raise ValueError(f"P ({P.dtype}) and Q ({Q.dtype}) must have one dtype")
    dp, dq = _nearest(P, Q)[:2]
    return (dp[0], dq[0]) if squeeze else (dp, dq)


def f_scores(gt: torch.Tensor, pred: torch.Tensor, thresholds=FSCORE_THRESHOLDS):
    """calculate_fscore of the FreiHAND script for every sample and threshold -> (F, frac_gt, frac_pred), each
    [B, T] float64: frac_gt = #(d_gt < t) / n_gt with d_gt the distance of each gt point to the nearest prediction,
    frac_pred the same for the predicted points, F = ((2 frac_gt) frac_pred) / (frac_gt + frac_pred) (0 when both are
    0; symmetric in gt and pred).  thresholds: 1 .. 16 values, sorted, in the points' unit.  A sample holding a
    non-finite coordinate gets NaN."""
    squeeze = gt.dim() == 2
    dts = tuple(_DTYPES)
    gt, pred = _points(gt, "gt", dts), _points(pred, "pred", dts)
    _same_batch(gt, pred, ("gt", "pred"))
    if gt.dtype != pred.dtype:
        raise ValueError(f"gt ({gt.dtype}) and pred ({pred.dtype}) must have one dtype")
    thr, t = _thresholds(thresholds, _MAX_F_THRESHOLDS)
    _, _, _, fr, fs = _nearest(gt, pred, thr, t.size, dist=False, frac=True, fscore=True)
    out = (fs, fr[:, 0], fr[:, 1])
    return tuple(o[0] for o in out) if squeeze else out


def align_w_scale(gt: torch.Tensor, pred: torch.Tensor) -> torch.Tensor:
    """The FreiHAND script's align_w_scale(gt, pred) per sample: pred aligned onto gt by the similarity of the
    Frobenius-normalised orthogonal Procrustes problem, with no reflection correction (det R = -1 is kept).  float32
    [B, n, 3] or [n, 3] in, float32 of pred's shape out.  A sample holding a non-finite coordinate gets NaN."""
    squeeze = gt.dim() == 2
    gt, pred = _points(gt, "gt"), _points(pred, "pred")
    if gt.shape != pred.shape or gt.device != pred.device:
        raise ValueError(f"gt {tuple(gt.shape)} and pred {tuple(pred.shape)} must match in shape and device")
    Y, _ = _align(gt, pred)
    return Y[0] if squeeze else Y


def mano_eval_regressor(J_regressor) -> torch.Tensor:
    """The 21 x 778 joint regressor Pose2Mesh evaluates FreiHAND with (lib/_mano.py:22-30): MANO's 16-row J_regressor
    plus one-hot rows for the fingertip vertices 745, 317, 445, 556, 673, in FreiHAND's joint order.  float32 on the
    input's device (CPU for a numpy array); predicted joints are then postprocess.regress_joints(verts, it)."""
    device = J_regressor.device if isinstance(J_regressor, torch.Tensor) else torch.device("cpu")
    J = np.asarray(J_regressor.detach().cpu() if isinstance(J_regressor, torch.Tensor) else J_regressor)
    if J.shape != (16, 778):
        raise ValueError(f"J_regressor must be MANO's [16, 778]; got {J.shape}")
    tips = np.zeros((5, 778), dtype=np.float32)
    tips[np.arange(5), MANO_EVAL_TIPS] = 1
    out = np.concatenate((J, tips))[list(MANO_EVAL_ORDER), :].astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(out)).to(device)


class FreiHANDEvaluator:
    """The FreiHAND script's measures over a test set, accumulated on the device:

        ev = FreiHANDEvaluator()
        for batch in loader:
            ev.update(pred_xyz, pred_verts, gt_xyz, gt_verts)   # [B, 21, 3], [B, 778, 3] float32 CUDA, metres
        scores = ev.compute()

    update() enqueues a fixed number of launches and never synchronises with the host; compute() reads the results
    back once.  Counts are integers and F means reduce over samples in sample order, so splitting the same samples
    into different batches gives bitwise-identical counts, AUCs and F means."""

    KINDS = ("xyz", "pa_xyz", "mesh", "pa_mesh")

    def __init__(self, thresholds=FSCORE_THRESHOLDS, pck=PCK_RANGE, device=None):
        self._f_thr, t = _thresholds(thresholds, _MAX_F_THRESHOLDS)
        self.thresholds = tuple(t.tolist())
        lo, hi, steps = pck
        self.pck_thresholds = np.linspace(lo, hi, int(steps))
        self._pck_thr, _ = _thresholds(self.pck_thresholds, _MAX_PCK_THRESHOLDS, "pck thresholds")
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("pose2mesh_release_b200 runs on CUDA (sm_90a) only; no CUDA device")
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"pose2mesh_release_b200 runs on CUDA (sm_90a) only; device {self.device}")
        self.reset()

    def reset(self):
        self._hist = torch.zeros((len(self.KINDS), len(self.pck_thresholds)), device=self.device, dtype=torch.int64)
        self._err = {k: [] for k in self.KINDS}
        self._f = {"f_score": [], "f_score_aligned": []}
        self.n_samples = 0

    def update(self, pred_xyz, pred_verts, gt_xyz, gt_verts):
        px, pv = _points(pred_xyz, "pred_xyz"), _points(pred_verts, "pred_verts")
        gx, gv = _points(gt_xyz, "gt_xyz"), _points(gt_verts, "gt_verts")
        if px.shape != gx.shape or pv.shape != gv.shape or px.shape[0] != pv.shape[0]:
            raise ValueError(f"pred_xyz {tuple(px.shape)}, gt_xyz {tuple(gx.shape)}, pred_verts {tuple(pv.shape)} and "
                             f"gt_verts {tuple(gv.shape)}: keypoints and vertices must match and share the batch")
        for t in (px, pv, gx, gv):
            if t.device != self.device:
                raise ValueError(f"the evaluator runs on {self.device}; got a tensor on {t.device}")
        n_pck = len(self.pck_thresholds)
        f64 = dict(device=self.device, dtype=torch.float64)
        for k, (g, p) in enumerate(((gx, px), (gv, pv))):
            e = torch.empty(g.shape[:2], **f64)
            _pck(self._hist[2 * k], self._pck_thr, n_pck, pred=p, gt=g, err_out=e)
            aligned, e_al = _align(g, p, torch.float64, aligned=k == 1, err=True)
            _pck(self._hist[2 * k + 1], self._pck_thr, n_pck, err=e_al)
            self._err[self.KINDS[2 * k]].append(e)
            self._err[self.KINDS[2 * k + 1]].append(e_al)
        n_t = len(self.thresholds)
        self._f["f_score"].append(_nearest(gv, pv, self._f_thr, n_t, fscore=True)[4])
        self._f["f_score_aligned"].append(_nearest(gv.double(), aligned, self._f_thr, n_t, fscore=True)[4])
        self.n_samples += px.shape[0]

    def compute(self) -> dict:
        """The script's measures: for each of xyz, pa_xyz (keypoints after align_w_scale), mesh and pa_mesh, the mean
        end-point error ``{kind}_mean3d`` (mean over points of each point's mean over samples), the PCK curve
        ``{kind}_pck`` over ``pck_thresholds`` (fraction of errors <= t), its integer ``{kind}_counts`` and the
        normalised area under it ``{kind}_auc3d``; the mean F per threshold ``f_score`` / ``f_score_aligned``; and
        ``n_samples``.  PA-MPJPE = pa_xyz_mean3d, PA-MPVPE = pa_mesh_mean3d, F@5 / F@15 = f_score_aligned[0 / 1]
        with the default thresholds.  One device-to-host copy."""
        N = self.n_samples
        if N == 0:
            raise ValueError("FreiHANDEvaluator.compute: no samples; call update() first")
        means = []
        for k in self.KINDS:
            E = torch.cat(self._err[k]).t().contiguous()  # [points, samples]
            K = E.shape[0]
            per_point = _segment_mean(E, (C.c_int64 * (K + 1))(*range(0, (K + 1) * N, N)), K)
            means.append(_segment_mean(per_point, (C.c_int64 * 2)(0, K), 1))
        T = len(self.thresholds)
        for k in self._f:
            F = torch.cat(self._f[k]).t().contiguous()  # [thresholds, samples]
            means.append(_segment_mean(F, (C.c_int64 * (T + 1))(*range(0, (T + 1) * N, N)), T))
        host = torch.cat([self._hist.flatten()] + [m.view(torch.int64) for m in means]).cpu().numpy()
        n_pck = len(self.pck_thresholds)
        hist = host[:len(self.KINDS) * n_pck].reshape(len(self.KINDS), n_pck)
        f = host[len(self.KINDS) * n_pck:].view(np.float64)
        t = self.pck_thresholds
        norm = np.trapezoid(np.ones_like(t), t)
        out = {"n_samples": N, "pck_thresholds": t, "thresholds": self.thresholds}
        for i, k in enumerate(self.KINDS):
            n_pts = self._err[k][0].shape[1] * N
            counts = np.cumsum(hist[i])
            pck = counts / n_pts
            out[f"{k}_counts"] = counts
            out[f"{k}_pck"] = pck
            out[f"{k}_auc3d"] = float(np.trapezoid(pck, t) / norm)
            out[f"{k}_mean3d"] = float(f[i])
        out["f_score"] = f[len(self.KINDS):len(self.KINDS) + T].copy()
        out["f_score_aligned"] = f[len(self.KINDS) + T:].copy()
        return out
