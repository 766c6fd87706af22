"""Float64 CPU restatement of the datasets' target construction (pose2mesh_release_b200/targets.py):

    camera_frame   the seven get_smpl_coord / get_mano_coord bodies (data/{Human36M,AMASS,FreiHAND,MuCo,COCO,SURREAL,
                   PW3D}/dataset.py), one sample at a time as the datasets run them
    h36m_targets   the target / meta assembly of Human36M.__getitem__ (data/Human36M/dataset.py:301-333,344-418),
                   augmentation off

The body model is a callable forward(pose [B, 3J], betas [B, S], trans [B, 3] or None) -> (verts, joints) in float64
(tests/body_model_oracle.py's smpl_forward / mano_forward bound to a model).  The root rotation goes through scipy's
Rotation, independently of the kernel's log map, and is rounded to float32 where the reference stores it into its
float32 pose.  Everything else is float64.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial.transform import Rotation

FACE_KPS_VERTEX = (331, 2802, 6262, 3489, 3990)
COCO_LSH, COCO_RSH, COCO_LHIP, COCO_RHIP = 5, 6, 11, 12

# (rotate root, clamp betas, layer trans: None / "t" / "trans", after the layer: None / "h36m" / "t", to mm, extra)
PRESETS = {
    "human36m": (True, True, None, "h36m", True, ()),
    "amass": (True, False, None, "t", True, ()),
    "freihand": (True, False, "t", None, False, ()),
    "muco": (False, True, "trans", None, True, FACE_KPS_VERTEX),
    "coco": (False, True, None, None, True, ()),
    "surreal": (False, False, "trans", None, True, ()),
    "pw3d": (False, False, "trans", None, True, ()),
}


def rotate_root(root, R) -> np.ndarray:
    """float32 rotvec of R exp(root) for root [B, 3], R [B, 3, 3]; a zero root is the identity."""
    root = np.asarray(root, np.float64)
    M = np.asarray(R, np.float64) @ Rotation.from_rotvec(root).as_matrix()
    return Rotation.from_matrix(M).as_rotvec().astype(np.float32)


def resolve_betas(betas, model_betas, clamp: bool, zero_means_model: bool) -> np.ndarray:
    """The clamp (any |beta| > 3 -> zeros) and, for SMPL, the one-sample "all-zero betas -> model betas" rule."""
    b = np.array(betas, np.float64)
    if clamp:
        b[(np.abs(b) > 3).any(1)] = 0.0
    if zero_means_model:
        zero = (b == 0).all(1)
        b[zero] = np.asarray(model_betas, np.float64)[None]
    return b


def camera_frame(forward, model_betas, dataset, pose, betas, trans=None, R=None, t=None, mano=False, chunk=64):
    """-> (mesh, joints) float64 in the preset's units."""
    rot, clamp, layer_trans, after, to_mm, extra = PRESETS[dataset]
    pose = np.array(pose, np.float64)
    if rot:
        pose[:, :3] = rotate_root(pose[:, :3], R)
    b = resolve_betas(betas, model_betas, clamp, not mano)
    lt = {None: None, "t": t, "trans": trans}[layer_trans]
    meshes, joints = [], []
    for s in range(0, pose.shape[0], chunk):
        sl = slice(s, s + chunk)
        v, j = forward(pose[sl], b[sl], None if lt is None else np.asarray(lt, np.float64)[sl])
        if extra:
            j = np.concatenate([j, v[:, list(extra)]], 1)
        if after == "h36m":
            Rs = np.asarray(R, np.float64)[sl]
            j0 = j[:, :1]
            off = (np.einsum("brc,bc->br", Rs, np.asarray(trans, np.float64)[sl]) + np.asarray(t, np.float64)[sl] / 1000
                   )[:, None] - j0 + np.einsum("brc,bjc->bjr", Rs, j0)
            v, j = v + off, j + off
        elif after == "t":
            off = np.asarray(t, np.float64)[sl][:, None]
            v, j = v + off, j + off
        if to_mm:
            v, j = v * 1000, j * 1000
        meshes.append(v)
        joints.append(j)
    return np.concatenate(meshes), np.concatenate(joints)


def cam2pixel(p, f, c):
    """lib/coord_utils.py:104-109 on [B, J, 3] points, -> [B, J, 2]."""
    return np.stack([p[..., 0] / p[..., 2] * f[:, None, 0] + c[:, None, 0],
                     p[..., 1] / p[..., 2] * f[:, None, 1] + c[:, None, 1]], -1)


def fitting_error(h36m_joint, reg_h36m, mesh):
    """Human36M.get_fitting_error for a batch: h36m_joint [B, 17, 3], mesh [B, V, 3] (mm) -> [B]."""
    h = h36m_joint - h36m_joint[:, :1]
    s = np.einsum("jv,bvc->bjc", reg_h36m, mesh)
    s = s - s.mean(1, keepdims=True) + h.mean(1, keepdims=True)
    return np.sqrt(((h - s) ** 2).sum(2)).mean(1)


def h36m_targets(mesh_cam, joint_cam, f, c, reg_h36m, reg_coco, joint_set="human36", fitting_thr=25.0) -> dict:
    """Human36M.__getitem__'s targets and meta (pose2mesh_net; posenet's joint_valid = lift_pose3d_valid), float64."""
    mesh_cam, joint_cam = np.asarray(mesh_cam, np.float64), np.asarray(joint_cam, np.float64)
    f, c = np.asarray(f, np.float64), np.asarray(c, np.float64)
    reg_h36m, reg_coco = np.asarray(reg_h36m, np.float64), np.asarray(reg_coco, np.float64)
    B, V = mesh_cam.shape[:2]
    coco = np.einsum("jv,bvc->bjc", reg_coco, mesh_cam)
    pelvis = (coco[:, COCO_LHIP] + coco[:, COCO_RHIP]) * 0.5
    neck = (coco[:, COCO_LSH] + coco[:, COCO_RSH]) * 0.5
    coco = np.concatenate([coco, pelvis[:, None], neck[:, None]], 1)
    root = joint_cam[:, :1]
    mesh = mesh_cam - root
    h36m = joint_cam - root
    err = fitting_error(h36m, reg_h36m, mesh)
    valid = (~(err > fitting_thr)).astype(np.float64)
    if joint_set == "coco":
        lift, img, lift_valid = coco - coco[:, -2:-1], cam2pixel(coco, f, c), valid
    else:
        lift, img, lift_valid = h36m, cam2pixel(joint_cam, f, c), np.ones(B)
    J = lift.shape[1]
    return {"mesh": mesh / 1000, "lift_pose3d": lift, "reg_pose3d": h36m,
            "mesh_valid": np.repeat(valid[:, None, None], V, 1), "lift_pose3d_valid": np.repeat(
                lift_valid[:, None, None], J, 1), "reg_pose3d_valid": np.ones((B, 17, 1)), "joint_img": img,
            "fitting_error": err}
