"""Float64 CPU restatement of the training sample's augmentation on the device (pose2mesh_release_b200.inputs
augm_params / training_pose2d(rot, flip), targets.Human36MTargets(rot, flip)):

    augm_params       lib/aug_utils.py:98-117 on the augmentation's streams of include/p2m_b200.h's counter rule
    training_pose2d   oracle/inputs_oracle.py's training_pose2d with the rotation in the crop's affine map
                      (get_affine_transform, lib/aug_utils.py:125-185) and flip_2d_joint before or after the noise
    j3d_processing    lib/aug_utils.py:67-83 on the lift target

The random stream is restated draw for draw (oracle/inputs_oracle.py's Philox), so the device agrees with this module
to rounding; tests/golden/samples.npz (the unmodified reference) pins the distributions and the geometry.
"""
from __future__ import annotations

import numpy as np

from oracle import inputs_oracle as io

AUG_SID = 1 << 31          # the augmentation's stream domain: 2^31 + purpose
COCO_FLIP_PAIRS = ((1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))
H36M_FLIP_PAIRS = ((1, 4), (2, 5), (3, 6), (14, 11), (15, 12), (16, 13))


def flip_perm(joint_set: str, J: int):
    """Row j of a flipped pose is row perm[j] of the pose."""
    perm = np.arange(J)
    for a, b in (COCO_FLIP_PAIRS if joint_set == "coco" else H36M_FLIP_PAIRS):
        perm[a], perm[b] = b, a
    return perm


def augm_params(B: int, flip: bool, rotate_factor: float, seed, sample_index=None):
    """-> (flip int32 [B], rot float32 [B] degrees)."""
    b = np.arange(B, dtype=np.uint64) if sample_index is None else np.asarray(sample_index, np.uint64)
    u_flip, u_keep = io.uniforms(seed, b, AUG_SID, 0)
    g0, g1 = io.uniforms(seed, b, AUG_SID + 1, 0)
    z = np.sqrt(-2.0 * np.log(1.0 - g0)) * np.cos(2 * np.pi * g1)
    rf = float(rotate_factor)
    rot = np.minimum(2 * rf, np.maximum(-2 * rf, z * rf))
    f = (bool(flip) & (u_flip <= 0.5)).astype(np.int32)
    return f, np.where(u_keep <= 0.5, 0.0, rot).astype(np.float32)


def rot_map(m, rot, input_shape=io.INPUT_SHAPE):
    """get_affine_transform(centre, (w, h), rot, (in_w, in_h)) per sample on inputs_oracle.crop_map's box:
    -> (s0 [B, 2], q0 [2], A [B, 2, 2]); a point maps to q0 + A (p - s0)."""
    in_h, in_w = input_shape
    f = np.float32
    rr = np.pi * np.asarray(rot, np.float64) / 180
    sn, cs = np.sin(rr), np.cos(rr)
    hw = (m["crop_w"].astype(np.float32) * f(-0.5)).astype(np.float64)
    s0 = np.stack([m["ccx"], m["ccy"]], -1).astype(np.float32)
    s1 = np.stack([s0[:, 0] + (0 * cs - hw * sn), s0[:, 1] + (0 * sn + hw * cs)], -1).astype(np.float32)
    s2 = s1 + np.stack([-(s0[:, 1] - s1[:, 1]), s0[:, 0] - s1[:, 0]], -1)
    q0 = np.array([in_w * 0.5, in_h * 0.5], np.float32)
    q1 = np.array([in_w * 0.5, in_h * 0.5 + np.float32(in_w * -0.5)], np.float32)
    q2 = q1 + np.array([-(q0[1] - q1[1]), q0[0] - q1[0]], np.float32)
    E = np.stack([s1 - s0, s2 - s0], -1).astype(np.float64)              # [B, 2 (x, y), 2 (e1, e2)]
    F = np.stack([q1 - q0, q2 - q0], -1).astype(np.float64)
    return s0.astype(np.float64), q0.astype(np.float64), F[None] @ np.linalg.inv(E)


def crop_points(m, joints_px, rot, input_shape=io.INPUT_SHAPE):
    """joints_px [B, J, 2] through each sample's map (the rot-0 closed form where rot == 0) -> float64 [B, J, 2],
    before rounding."""
    in_h, in_w = input_shape
    p = np.asarray(joints_px, np.float32).astype(np.float64)
    out = np.stack([(p[:, :, 0] - m["ccx"].astype(np.float64)[:, None]) * m["sc"][:, None] + in_w * 0.5,
                    (p[:, :, 1] - m["ccy"].astype(np.float64)[:, None]) * m["sc"][:, None] + in_h * 0.5], -1)
    rot = np.asarray(rot, np.float32)
    if (rot != 0).any():
        s0, q0, A = rot_map(m, rot, input_shape)
        r = q0 + np.einsum("bij,bkj->bki", A, p - s0[:, None])
        out = np.where((rot != 0)[:, None, None], r, out)
    return out


def flip_2d(crop, flip, joint_set: str, width: int):
    """flip_2d_joint on the flipped samples: x -> width - x - 1 in the array's dtype, the pairs swapped."""
    crop = crop.copy()
    fl = np.asarray(flip) != 0
    x = crop[fl, :, 0]
    crop[fl, :, 0] = (x.dtype.type(width) - x) - x.dtype.type(1)
    crop[fl] = crop[fl][:, flip_perm(joint_set, crop.shape[1])]
    return crop


def training_pose2d(joints_px, noise: str, joint_set: str, seed=None, table=None, area_box="tight", box_joints=None,
                    rot=None, flip=None, flip_before_noise=False, input_shape=io.INPUT_SHAPE):
    """The device's training_pose2d with augmentation.  -> (pose2d [B, J, 2] float64, crop [B, J, 2] float32 before
    the normalisation)."""
    joints_px = np.asarray(joints_px, np.float32)
    B = joints_px.shape[0]
    in_h, in_w = input_shape
    rot = np.zeros(B, np.float32) if rot is None else np.asarray(rot, np.float32)
    flip = np.zeros(B, np.int32) if flip is None else np.asarray(flip, np.int32)
    m = io.crop_map(joints_px if box_joints is None else box_joints, input_shape)
    crop = crop_points(m, joints_px, rot, input_shape)
    if flip_before_noise:
        crop = flip_2d(crop, flip, joint_set, in_w)                    # MuCo: in fp64 inside j2d_processing
    crop = crop.astype(np.float32)
    if noise == "coco":
        j17 = np.concatenate([crop[:, :17].astype(np.float64), np.ones((B, 17, 1))], axis=2)
        crop[:, :17] = io.synthesize_pose(j17, io.crop_area(m, area_box), seed)[:, :, :2].astype(np.float32)
    elif noise == "h36m":
        err = io.generate_syn_error(table, B, seed)
        crop = crop + (err / np.float32(256)) * np.array([in_w, in_h], np.float32)
    if not flip_before_noise:
        crop = flip_2d(crop, flip, joint_set, in_w)                    # float32, after the noise
    return io.normalize(crop, input_shape), crop


def j3d_processing(lift, rot, flip, joint_set: str):
    """lift [B, J, 3] float64 (the value the reference holds before its float32 cast) -> augmented, float64."""
    lift = np.asarray(lift, np.float64).copy()
    rot = np.asarray(rot, np.float32).astype(np.float64)
    rr = -rot * np.pi / 180
    sn, cs = np.sin(rr)[:, None], np.cos(rr)[:, None]
    x, y = lift[:, :, 0].copy(), lift[:, :, 1].copy()
    on = (rot != 0)[:, None]
    lift[:, :, 0] = np.where(on, cs * x - sn * y, x)
    lift[:, :, 1] = np.where(on, sn * x + cs * y, y)
    fl = np.asarray(flip) != 0
    lift[fl] = lift[fl][:, flip_perm(joint_set, lift.shape[1])]
    lift[fl, :, 0] = -lift[fl, :, 0]
    return lift


# --------------------------------------------------------------------------------------------- sample targets
# MuCo.get_fitting_error's permutation (data/MuCo/dataset.py:246-262): source row MUCO_SRC[k] of the Human3.6M-ordered
# joints lands in Human3.6M slot MUCO_DST[k] by MuCo's joint names; the root is row 14 (MuCo's pelvis index)
MUCO_DST = (0, 1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 14, 15, 16)
MUCO_SRC = (14, 8, 9, 10, 11, 12, 13, 16, 5, 6, 7, 2, 3, 4)
FITTING_THR = {"human36m": 25.0, "coco": 3.0, "muco": 45.0, "amass": 0.0}


def _project(dataset, p, f=None, c=None, s=None, t=None):
    """The dataset's projection of camera-frame points p [B, J, 3] (mm) -> [B, J, 2] float64."""
    if dataset == "coco":
        s = np.asarray(s, np.float64).reshape(len(p), -1)
        return p[..., :2] / 1000 * s[:, None, :] + np.asarray(t, np.float64)[:, None, :]
    f, c = np.asarray(f, np.float64), np.asarray(c, np.float64)
    if dataset == "amass":
        p = p / 1000
    return p[..., :2] / p[..., 2:3] * f[:, None, :] + c[:, None, :]


def sample_targets(dataset, mesh_cam, reg_h36m, reg_coco, joint_set="human36", fitting_thr=None, joint_cam=None,
                   f=None, c=None, s=None, t=None, keypoints=None, keypoints_valid=None):
    """p2m_sample_targets in float64 (unaugmented; j3d_processing augments lift_pose3d)."""
    mesh_cam = np.asarray(mesh_cam, np.float64)
    thr = FITTING_THR[dataset] if fitting_thr is None else fitting_thr
    B, V = mesh_cam.shape[:2]
    coco = np.einsum("jv,bvc->bjc", np.asarray(reg_coco, np.float64), mesh_cam)
    coco = np.concatenate([coco, ((coco[:, 11] + coco[:, 12]) * 0.5)[:, None], ((coco[:, 5] + coco[:, 6]) * 0.5)[:, None]],
                          1)
    h36m = np.asarray(joint_cam, np.float64) if dataset == "human36m" else \
        np.einsum("jv,bvc->bjc", np.asarray(reg_h36m, np.float64), mesh_cam)
    root = h36m[:, :1]
    mesh = mesh_cam - root
    reg = h36m - root
    if joint_set == "coco":
        inp, lift = coco, coco - coco[:, 17:18]
    else:
        inp, lift = h36m, (reg.astype(np.float32).astype(np.float64) if dataset == "human36m" else reg)
    img = _project(dataset, inp, f, c, s, t)
    ones = np.ones(B)
    if dataset == "human36m":
        sm = np.einsum("jv,bvc->bjc", np.asarray(reg_h36m, np.float64), mesh)
        sm = sm - sm.mean(1, keepdims=True) + reg.mean(1, keepdims=True)
        err = np.sqrt(((reg - sm) ** 2).sum(2)).mean(1)
    elif dataset == "muco":
        hj = (reg - reg[:, 14:15]).astype(np.float32).astype(np.float64)[:, list(MUCO_SRC)]
        sm = np.einsum("jv,bvc->bjc", np.asarray(reg_h36m, np.float64), mesh)[:, list(MUCO_DST)]
        sm = sm - sm.mean(1, keepdims=True) + hj.mean(1, keepdims=True)
        err = np.sqrt(((hj - sm) ** 2).sum(2)).mean(1)
    elif dataset == "coco":
        m = io.crop_map(img.astype(np.float32), (64, 64))
        r = io.crop_points(m, _project("coco", coco[:, :17], s=s, t=t).astype(np.float32), (64, 64))
        k = io.crop_points(m, np.asarray(keypoints, np.float32), (64, 64))
        d = np.sqrt(((k - r) ** 2).sum(2, dtype=np.float32)).astype(np.float64)
        vis = np.asarray(keypoints_valid) > 0
        with np.errstate(invalid="ignore"):
            err = (d * vis).sum(1) / vis.sum(1)
    else:
        err = np.zeros(B)
    valid = (~(err > thr)).astype(np.float64) if dataset != "amass" else ones
    zero_reg = dataset in ("coco", "muco")
    lift_valid = ones if (dataset == "human36m" and joint_set != "coco") else valid
    joint_valid = valid if (dataset == "coco" or (dataset == "human36m" and joint_set == "coco")) else ones
    J = lift.shape[1]
    col = lambda v, n: np.repeat(v[:, None, None], n, 1)  # noqa: E731
    return {"mesh": mesh / 1000, "lift_pose3d": lift, "reg_pose3d": reg, "joint_img": img, "fitting_error": err,
            "mesh_valid": col(valid, V), "lift_pose3d_valid": col(lift_valid, J),
            "reg_pose3d_valid": col(valid if zero_reg else ones, 17), "joint_valid": col(joint_valid, J)}
