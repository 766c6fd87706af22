"""The temporal metrics of the reference's 3DPW video evaluation on the GPU (SURVEY.md §8 row f8):

    smooth_pose(pred_pose, ...)              lib/smooth_utils.py:49-72 (OneEuroFilter, :5-46), one sequence
    smooth_sequences(x, lengths, ...)        the same over a ragged batch of sequences, one launch
    compute_error_accel(gt, pred, vis)       lib/coord_utils.py:194-222, one sequence
    accel_errors(gt, pred, lengths, vis)     the same over a ragged batch, with per-sequence means, no host sync
    evaluate_video(pred, gt, video_indices)  the video block of PW3D.evaluate (data/PW3D/dataset.py:383-417) for
                                             every video at once

Everything runs in libp2m_b200.so (p2m_one_euro_smooth, p2m_accel_error, p2m_segment_mean, and p2m_point_errors /
p2m_rigid_align of the evaluation metrics).  Data are float32 or float64 CUDA tensors; sequence lengths and video
indices are host values.  Smoothing and per-window acceleration errors are the reference's bits in the input's dtype;
means are fp64.  install() does not rebind the reference's functions: they take numpy arrays.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .metrics import _align, _errors

_DTYPES = {torch.float32: _lib.P2M_DTYPE_F32, torch.float64: _lib.P2M_DTYPE_F64}


def _data(x, what: str) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.dtype not in _DTYPES:
        raise ValueError(f"{what} must be float32 or float64; got {x.dtype}")
    if x.dim() == 0 or x.shape[0] == 0:
        raise ValueError(f"{what} must be [N, ...] with N > 0 frames; got {tuple(x.shape)}")
    return x.contiguous()


def _joints(gt, pred):
    gt, pred = _data(gt, "joints_gt"), _data(pred, "joints_pred")
    if gt.shape != pred.shape or gt.dim() != 3 or gt.shape[-1] != 3 or not 0 < gt.shape[1] <= 32:
        raise ValueError(f"joints_gt {tuple(gt.shape)} and joints_pred {tuple(pred.shape)} must both be [N, J, 3] "
                         "with J <= 32")
    if gt.dtype != pred.dtype or gt.device != pred.device:
        raise ValueError(f"joints_gt ({gt.dtype}, {gt.device}) and joints_pred ({pred.dtype}, {pred.device}) differ")
    return gt, pred


def _offsets(lengths, n_frames: int):
    """Host sequence lengths -> (ctypes int64 offsets [n + 1], n).  They must cover the n_frames frames exactly."""
    n = np.asarray(lengths.cpu() if isinstance(lengths, torch.Tensor) else lengths).reshape(-1)
    if n.size == 0 or not (np.issubdtype(n.dtype, np.integer) or n.dtype == object) or (n < 0).any():
        raise ValueError(f"lengths must be one or more non-negative integers; got {lengths!r}")
    off = np.concatenate([[0], np.cumsum(n.astype(np.int64))])
    if off[-1] != n_frames:
        raise ValueError(f"lengths sum to {int(off[-1])} frames; the input has {n_frames}")
    return (C.c_int64 * off.size)(*off.tolist()), int(n.size)


def _vis(vis, n_frames: int, device):
    if vis is None:
        return None
    _lib.cuda_tensor(vis, "vis")
    if vis.dim() != 1 or vis.shape[0] != n_frames or vis.device != device:
        raise ValueError(f"vis must be [{n_frames}] on {device}, one flag per frame; got {tuple(vis.shape)}")
    return (vis != 0).to(torch.uint8).contiguous()


def _segment_mean(values: torch.Tensor, offsets, n_seg: int, width: int = 1, valid=None) -> torch.Tensor:
    """fp64 mean per segment of a [rows, width] float32 / float64 tensor (one p2m_segment_mean launch)."""
    out = torch.empty((n_seg,), device=values.device, dtype=torch.float64)
    n_rows = values.numel() // width
    _lib.call("p2m_segment_mean", values.device, _DTYPES[values.dtype], values, width, offsets, n_seg, n_rows, valid,
              out)
    return out


def _one_segment(n: int):
    return (C.c_int64 * 2)(0, n)


# ---------------------------------------------------------------------------------------------- public functions
def smooth_sequences(x: torch.Tensor, lengths, min_cutoff: float, beta: float, d_cutoff: float = 1.0) -> torch.Tensor:
    """smooth_pose on every sequence of x [N, ...] (sequences concatenated along dim 0, `lengths` frames each, host
    values), in one launch.  Returns x's dtype and shape; each value is the bits smooth_pose gives on that sequence."""
    x = _data(x, "x")
    off, n_seq = _offsets(lengths, x.shape[0])
    y = torch.empty_like(x)
    n_ch = x[0].numel()
    if n_ch == 0:
        raise ValueError(f"x must hold at least one channel per frame; got {tuple(x.shape)}")
    _lib.call("p2m_one_euro_smooth", x.device, _DTYPES[x.dtype], x, y, n_ch, off, n_seq, x.shape[0], float(min_cutoff),
              float(beta), float(d_cutoff))
    return y


def smooth_pose(pred_pose: torch.Tensor, min_cutoff: float = 0.004, beta: float = 0.7) -> torch.Tensor:
    """smooth_utils.smooth_pose: the One-Euro filter along dim 0 of pred_pose [N, ...] (N > 0; the reference raises
    IndexError for N = 0, this raises ValueError).  Same dtype and shape, bit for bit the reference's values."""
    pred_pose = _data(pred_pose, "pred_pose")
    return smooth_sequences(pred_pose, [pred_pose.shape[0]], min_cutoff, beta)


def accel_errors(gt: torch.Tensor, pred: torch.Tensor, lengths, vis: torch.Tensor = None):
    """compute_error_accel on every sequence of gt, pred [N, J, 3] (concatenated along frames, `lengths` host values),
    without a host synchronisation.  Returns

      per_window  [sum max(n - 2, 0)]  every window's error in the input's dtype (the reference's bits), in order;
      valid       [same] bool          the window's three frames are visible (all True without vis);
      seq_mean    [n_seq] float64      the mean of the sequence's valid windows, NaN when it has none.

    vis: [N] per-frame flags (bool or integer) on the same device, or None."""
    gt, pred = _joints(gt, pred)
    off, n_seq = _offsets(lengths, gt.shape[0])
    n_win = sum(max(off[i + 1] - off[i] - 2, 0) for i in range(n_seq))
    v = _vis(vis, gt.shape[0], gt.device)
    per_window = torch.empty((n_win,), device=gt.device, dtype=gt.dtype)
    valid = torch.empty((n_win,), device=gt.device, dtype=torch.uint8)
    seq_mean = torch.empty((n_seq,), device=gt.device, dtype=torch.float64)
    _lib.call("p2m_accel_error", gt.device, _DTYPES[gt.dtype], gt, pred, gt.shape[1], off, n_seq, gt.shape[0], v,
              per_window, valid, seq_mean)
    return per_window, valid.view(torch.bool), seq_mean


def compute_error_accel(joints_gt: torch.Tensor, joints_pred: torch.Tensor, vis: torch.Tensor = None) -> torch.Tensor:
    """coord_utils.compute_error_accel: the per-window acceleration errors [M] of one sequence [N, J, 3], compacted to
    the windows whose three frames are visible, bit for bit the reference's values.  With vis given, the compaction
    reads the window count back to the host (one synchronisation); accel_errors is the sync-free form."""
    per_window, valid, _ = accel_errors(joints_gt, joints_pred, [_data(joints_gt, "joints_gt").shape[0]], vis)
    return per_window if vis is None else per_window[valid]


def _video_frames(video_indices, n_frames: int):
    """The dataset's video_indices (boolean masks or index arrays over frames) -> (frame index array, lengths).
    A mask selects its frames in ascending order; an index array keeps its own order, as numpy indexing does."""
    idx, lengths = [], []
    for k, v in enumerate(video_indices):
        a = np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v).reshape(-1)
        if a.dtype == bool:
            if a.size != n_frames:
                raise ValueError(f"video {k}: a mask must have one flag per frame ({n_frames}); got {a.size}")
            a = np.flatnonzero(a)
        elif a.size and not np.issubdtype(a.dtype, np.integer):
            raise ValueError(f"video {k}: indices must be integers or a boolean mask; got {a.dtype}")
        a = a.astype(np.int64)
        if a.size and (a.min() < -n_frames or a.max() >= n_frames):
            raise ValueError(f"video {k}: frame index out of range for {n_frames} frames")
        idx.append(a % n_frames if a.size else a)
        lengths.append(a.size)
    if not lengths:
        raise ValueError("video_indices holds no video")
    return np.concatenate(idx), lengths


def evaluate_video(pred_j3d: torch.Tensor, gt_j3d: torch.Tensor, video_indices, smooth: bool = True,
                   min_cutoff: float = 0.004, beta: float = 0.005):
    """The video block of PW3D.evaluate (data/PW3D/dataset.py:387-415) for every video at once.  pred_j3d, gt_j3d
    [frames, J, 3] (float32 or float64 CUDA tensors) hold the evaluation joints of every frame; video_indices is the
    dataset's list of per-video boolean masks or index arrays.  Each video's prediction is smoothed (smooth_pose with
    min_cutoff, beta; smooth=False scores the raw prediction), then scored.  Returns a dict of device tensors:

      accel_error [n_video] f64   mean acceleration error of the video (NaN with fewer than 3 frames, as np.mean of
                                  the reference's empty array)
      mpjpe       [n_video] f64   mean joint error of the video (NaN for an empty video; the reference raises there)
      pa_mpjpe    [n, J] f32      per-frame joint errors after Procrustes, videos in order (n = frames of all videos)
      accel_error_total, mpjpe_total, pa_mpjpe_total   0-d f64: the means of the per-video accel errors, of the
                                  per-video MPJPEs and of all per-frame PA-MPJPE values, as the block prints them

    The joint errors and Procrustes run in the evaluation-metric kernels, which take float32 points: a float64 input
    is rounded to float32 for those two.  Nine launches at most (eight with smooth=False), whatever the number of
    videos, and no host synchronisation after the index gather."""
    pred, gt = _joints(gt_j3d, pred_j3d)[::-1]
    frames, lengths = _video_frames(video_indices, pred.shape[0])
    if frames.size == 0:
        raise ValueError("video_indices select no frame")
    sel = torch.from_numpy(frames).to(pred.device)
    pred, gt = pred.index_select(0, sel), gt.index_select(0, sel)
    if smooth:
        pred = smooth_sequences(pred, lengths, min_cutoff, beta)
    _, _, accel = accel_errors(gt, pred, lengths)
    off, n_vid = _offsets(lengths, pred.shape[0])
    p32, g32 = pred.float().contiguous(), gt.float().contiguous()
    mpjpe_pp = _errors(p32, g32, fp64=pred.dtype == torch.float64)
    mpjpe = _segment_mean(mpjpe_pp, off, n_vid, width=gt.shape[1])
    pa = _align(p32, g32, err=True)[2]
    return {"accel_error": accel, "mpjpe": mpjpe, "pa_mpjpe": pa,
            "accel_error_total": _segment_mean(accel, _one_segment(n_vid), 1)[0],
            "mpjpe_total": _segment_mean(mpjpe, _one_segment(n_vid), 1)[0],
            "pa_mpjpe_total": _segment_mean(pa, _one_segment(pa.numel()), 1)[0]}
