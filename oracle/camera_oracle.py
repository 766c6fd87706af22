"""TEST INFRASTRUCTURE ONLY — CPU restatement of the demo's camera fit.

Only tests/ and tools/ may import this package.

    demo/run.py:149-153 (optimize_cam_param)         crop target: get_bbox, process_bbox(aspect 1.0, scale 1.25),
      lib/coord_utils.py:7-18,21-39,42-66            j2d_processing to a crop x crop patch
      lib/aug_utils.py:51-64,140-185
    demo/run.py:161-189, lib/models/project_net.py  1500 Adam steps on (s, tx, ty) against an L1 loss
    demo/run.py:24-43                               convert_crop_cam_to_orig_img

Two restatements of the fit:
  fit_f64               the reference's loop in float64, with switches for the mutations tests/test_camera_cpu.py uses
                        to show what the parity bound rejects;
  fit_f32_kernel_order  float32 numpy in csrc/camera.cu's exact operation order and xor-shuffle reduction tree, so the
                        GPU kernel must reproduce it bit for bit.

cv2.getAffineTransform is restated as OpenCV's LUImpl (6 x 6, partial pivoting, elimination a += alpha b, back
substitution by division) and np.dot(trans, (x, y, 1)) as (t0 x + t1 y) + t2; both reproduce the reference's bits.

Parity status: PINNED — tests/golden/camera_fit.npz holds the outputs of the unmodified reference functions
(tests/golden/make_golden_camera.py) and tests/test_camera_cpu.py checks these restatements against them.
"""
from __future__ import annotations

import math

import numpy as np

from . import demo_oracle as do

CROP = 500
LR_SCHEDULE = ((0, 0.1), (501, 0.05), (1001, 0.001))
N_ITER = 1500
f32 = np.float32


# ----------------------------------------------------------------------------------------------- crop target
def affine_lu(bbox: np.ndarray, res) -> np.ndarray:
    """get_center_scale + get_affine_transform(rot = 0): the float32 point pairs, solved as cv2.getAffineTransform
    solves them (OpenCV's LUImpl).  -> [2, 3] float64, or None where OpenCV finds the system singular."""
    x, y, w, h = bbox
    center = np.array([x + w * 0.5, y + h * 0.5], dtype=np.float32)
    src_w, dst_w, dst_h = np.float32(w * 1.0), res[0], res[1]
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0] = center
    src[1] = center + np.array([0.0, np.float64(src_w * -0.5)])          # get_dir(...) is a float64 list
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5]) + np.array([0, dst_w * -0.5], np.float32)
    for p in (src, dst):
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], dtype=np.float32)
    A = np.zeros((6, 6))
    b = np.zeros(6)
    for i in range(3):
        A[2 * i, 0:3] = (src[i, 0], src[i, 1], 1.0)
        A[2 * i + 1, 3:6] = (src[i, 0], src[i, 1], 1.0)
        b[2 * i], b[2 * i + 1] = dst[i, 0], dst[i, 1]
    for i in range(6):
        k = i
        for j in range(i + 1, 6):
            if abs(A[j, i]) > abs(A[k, i]):
                k = j
        if abs(A[k, i]) < np.finfo(np.float64).eps * 100:
            return None
        if k != i:
            A[[i, k], i:] = A[[k, i], i:]
            b[[i, k]] = b[[k, i]]
        d = -1.0 / A[i, i]
        for j in range(i + 1, 6):
            alpha = A[j, i] * d
            for c in range(i + 1, 6):
                A[j, c] = A[j, c] + alpha * A[i, c]
            b[j] = b[j] + alpha * b[i]
    for i in range(5, -1, -1):
        s = b[i]
        for c in range(i + 1, 6):
            s = s - A[i, c] * b[c]
        b[i] = s / A[i, i]
    return b.reshape(2, 3)


def get_bbox(joint_img: np.ndarray) -> np.ndarray:
    """coord_utils.py:21-39 as written: the width and height are taken AFTER re-centring (xmax' - xmin'), in the
    input's arithmetic (float64 for integer and float64 arrays, float32 for float32 arrays)."""
    x_img, y_img = joint_img[:, 0], joint_img[:, 1]
    xmin, ymin, xmax, ymax = min(x_img), min(y_img), max(x_img), max(y_img)
    x_center, width = (xmin + xmax) / 2., xmax - xmin
    xmin, xmax = x_center - 0.5 * width, x_center + 0.5 * width
    y_center, height = (ymin + ymax) / 2., ymax - ymin
    ymin, ymax = y_center - 0.5 * height, y_center + 0.5 * height
    return np.array([xmin, ymin, xmax - xmin, ymax - ymin]).astype(np.float32)


def crop_target(joint_input: np.ndarray, crop: int = CROP, scale: float = 1.25, aspect: float = 1.0):
    """run.py:150-153 -> (bbox1 float32 [4], target float32 [Jin, 2]), or (None, None) where process_bbox rejects the
    box or a joint is NaN.  The input's dtype matters as in the reference: integer arrays truncate the transformed
    points, float32 arrays take their box in float32."""
    xy = np.asarray(joint_input)[:, :2]
    if np.isnan(xy.astype(np.float64)).any():
        return None, None
    bbox = do.process_bbox(get_bbox(joint_input).copy(), aspect_ratio=aspect, scale=scale)
    if bbox is None:
        return None, None
    t = affine_lu(bbox, (crop, crop))
    if t is None:
        return None, None
    x, y = xy[:, 0].astype(np.float64), xy[:, 1].astype(np.float64)
    X, Y = (t[0, 0] * x + t[0, 1] * y) + t[0, 2], (t[1, 0] * x + t[1, 1] * y) + t[1, 2]
    if xy.dtype.kind in "iu":
        X, Y = np.trunc(X), np.trunc(Y)
    return np.asarray(bbox, dtype=np.float32), np.stack([X, Y], 1).astype(np.float32)


def crop_targets(joints: np.ndarray, crop: int = CROP, **kw):
    """crop_target over a batch [B, Jin, C] -> bbox [B, 4], target [B, Jin, 2] (NaN for rejected people)."""
    B, n = joints.shape[0], joints.shape[1]
    bbox = np.full((B, 4), np.nan, np.float32)
    tgt = np.full((B, n, 2), np.nan, np.float32)
    for i in range(B):
        b, t = crop_target(joints[i], crop, **kw)
        if b is not None:
            bbox[i], tgt[i] = b, t
    return bbox, tgt


def orig_cam_f32(cam: np.ndarray, bbox: np.ndarray, img_width, img_height) -> np.ndarray:
    """convert_crop_cam_to_orig_img (run.py:24-43) in float32; img sizes are numbers or [B] arrays of integers."""
    cam, bbox = cam.astype(np.float32), bbox.astype(np.float32)
    W = np.broadcast_to(np.asarray(img_width, dtype=np.float32), cam.shape[:1])
    H = np.broadcast_to(np.asarray(img_height, dtype=np.float32), cam.shape[:1])
    x, y, w, h = bbox[:, 0], bbox[:, 1], bbox[:, 2], bbox[:, 3]
    cx, cy = x + w / f32(2), y + h / f32(2)
    hw, hh = W / f32(2), H / f32(2)
    sx = cam[:, 0] * (f32(1) / (W / h))
    sy = cam[:, 0] * (f32(1) / (H / h))
    tx = ((cx - hw) / hw / sx) + cam[:, 1]
    ty = ((cy - hh) / hh / sy) + cam[:, 2]
    return np.stack([sx, sy, tx, ty]).T.astype(np.float32)


def _lr(schedule, it):
    lr = schedule[0][1]
    for start, r in schedule:
        if start <= it:
            lr = r
    return lr


# ----------------------------------------------------------------------------------------------- float64 loop
def fit_f64(p3d, target, init, crop: int = CROP, n_iter: int = N_ITER, schedule=LR_SCHEDULE,
            bias_correction: bool = True, eps_inside_sqrt: bool = False, sign_of_zero: float = 0.0):
    """run.py:161-189 in float64 for a batch: p3d [B, J, >= 2], target [B, >= J, 2] (its first J rows are used),
    init [B, 3].  -> (cam [B, 3], L1 loss of the final camera [B]).  Switches restate mutations of the loop."""
    P = np.asarray(p3d, np.float64)[:, :, :2]
    J = P.shape[1]
    T = np.asarray(target, np.float64)[:, :J]
    p = np.asarray(init, np.float64).copy()
    m, v = np.zeros_like(p), np.zeros_like(p)
    res = crop / 2
    for it in range(n_iter):
        lr = _lr(schedule, it)
        q = P + p[:, None, 1:]
        d = q * p[:, None, :1] * res + res - T
        g_out = np.where(d == 0, sign_of_zero, np.sign(d)) / (2 * J)
        ga = g_out * res
        g = np.stack([(ga * q).sum((1, 2)), (ga[..., 0] * p[:, None, 0]).sum(1), (ga[..., 1] * p[:, None, 0]).sum(1)], 1)
        step = it + 1
        m = m + (1 - 0.9) * (g - m)
        v = v * 0.999 + (1 - 0.999) * g * g
        bc1, bc2 = 1 - 0.9 ** step, 1 - 0.999 ** step
        if not bias_correction:
            bc1 = bc2 = 1.0
        if eps_inside_sqrt:
            denom = np.sqrt(v / bc2 + 1e-8)
        else:
            denom = np.sqrt(v) / math.sqrt(bc2) + 1e-8
        p = p - (lr / bc1) * m / denom
    q = P + p[:, None, 1:]
    loss = np.abs(q * p[:, None, :1] * res + res - T).mean((1, 2))
    return p, loss


# ----------------------------------------------------------------------------------------------- kernel order
def _tree(v: np.ndarray) -> np.ndarray:
    """csrc/camera.cu warp_sum: xor butterfly over 32 lanes, float32."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lanes ^ o]
    return v[:, 0]


def fit_f32_kernel_order(p3d, target, init, crop: int = CROP, n_iter: int = N_ITER, schedule=LR_SCHEDULE):
    """k_fit_camera's fit in float32 numpy, operation for operation: p3d [B, J, 3] float32, target [B, Jin, 2] float32
    (NaN rows for rejected people), init [B, 3] float32.  -> (cam [B, 3], loss [B]) with the kernel's bits."""
    p3d, target = np.asarray(p3d, np.float32), np.asarray(target, np.float32)
    B, J = p3d.shape[0], p3d.shape[1]
    ok = ~np.isnan(target).any((1, 2))
    px, py, tx, ty = (np.zeros((B, 32), np.float32) for _ in range(4))
    px[:, :J], py[:, :J] = p3d[:, :, 0], p3d[:, :, 1]
    tx[:, :J], ty[:, :J] = target[:, :J, 0], target[:, :J, 1]
    on = np.arange(32)[None] < J
    zero = f32(0)
    res = f32(crop / 2.0)
    inv_n = f32(1) / f32(2 * J)
    w1, b2, w2, eps = f32(1.0 - 0.9), f32(0.999), f32(1.0 - 0.999), f32(1e-8)
    p = np.where(ok[:, None], np.asarray(init, np.float32), f32(np.nan)).astype(np.float32)
    m, v = np.zeros((B, 3), np.float32), np.zeros((B, 3), np.float32)
    b1t = b2t = 1.0
    for it in range(n_iter):
        lr = _lr(schedule, it)
        s = p[:, 0:1]
        qx, qy = px + p[:, 1:2], py + p[:, 2:3]
        ox, oy = (qx * s) * res + res, (qy * s) * res + res
        gax, gay = (np.sign(ox - tx) * inv_n) * res, (np.sign(oy - ty) * inv_n) * res
        g = np.stack([_tree(np.where(on, gax * qx + gay * qy, zero)), _tree(np.where(on, gax * s, zero)),
                      _tree(np.where(on, gay * s, zero))], 1)
        b1t, b2t = b1t * 0.9, b2t * 0.999
        step_size = lr / (1.0 - b1t)
        bc2_sqrt = f32(math.sqrt(1.0 - b2t))
        neg_step = -f32(step_size)
        m = m + w1 * (g - m)
        v = v * b2 + (w2 * g) * g
        denom = np.sqrt(v) / bc2_sqrt + eps
        p = p + (neg_step * m) / denom
    s = p[:, 0:1]
    dx = ((px + p[:, 1:2]) * s) * res + res - tx
    dy = ((py + p[:, 2:3]) * s) * res + res - ty
    loss = _tree(np.where(on, np.abs(dx) + np.abs(dy), zero)) / f32(2 * J)
    return p.astype(np.float32), loss.astype(np.float32)
