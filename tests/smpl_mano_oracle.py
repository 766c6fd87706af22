"""Float64 CPU restatement of the SURREAL, FreiHAND and 3DPW samples on the device (pose2mesh_release_b200.inputs
training_pose2d with the 'smpl' / 'mano' joint sets, targets.SURREALTargets / FreiHANDTargets / PW3DTargets):

    training_pose2d   the noise-free crop (oracle/inputs_oracle.py's crop_map, oracle/samples_oracle.py's rotated map)
                      with SURREAL's flip pairs, flipped in float64 before the crop is rounded or in float32 after it
    surreal_targets   data/SURREAL/dataset.py:143-203: float32 rooting at SMPL joint 0, fp64 cam2pixel of the absolute
                      joints, j3d_processing on the lift target, reg_pose3d the same augmented array
    freihand_targets  data/FreiHAND/dataset.py:139-192: float32 rooting at MANO joint 0 (the wrist)
    pw3d_targets      data/PW3D/dataset.py:208-261: the Human3.6M and COCO regressors in fp64, rooted as the other
                      regressor datasets, cam2pixel of the COCO joints with pelvis and neck, every mask 1

The reference's own float32 steps (the rooting, the mesh / 1000) are float32 here too: they are the rule.
tests/golden/smpl_mano_samples.npz (the unmodified reference) pins the geometry.
"""
from __future__ import annotations

import numpy as np

from oracle import inputs_oracle as io
from oracle import samples_oracle as so

SMPL_FLIP_PAIRS = ((1, 2), (4, 5), (7, 8), (10, 11), (13, 14), (16, 17), (18, 19), (20, 21), (22, 23))
N_JOINTS = {"smpl": 24, "mano": 21}


def flip_perm(joint_set: str, J: int):
    """Row j of a flipped pose is row perm[j] of the pose ('smpl', or samples_oracle's 'coco' / 'human36')."""
    if joint_set != "smpl":
        return so.flip_perm(joint_set, J)
    perm = np.arange(J)
    for a, b in SMPL_FLIP_PAIRS:
        perm[a], perm[b] = b, a
    return perm


def flip_2d(crop, flip, joint_set: str, width: int):
    """flip_2d_joint on the flipped samples: x -> width - x - 1 in the array's dtype, the pairs swapped."""
    crop = crop.copy()
    fl = np.asarray(flip) != 0
    x = crop[fl, :, 0]
    crop[fl, :, 0] = (x.dtype.type(width) - x) - x.dtype.type(1)
    crop[fl] = crop[fl][:, flip_perm(joint_set, crop.shape[1])]
    return crop


def training_pose2d(joints_px, joint_set: str, rot=None, flip=None, flip_before=False, input_shape=io.INPUT_SHAPE):
    """The device's noise-free training_pose2d on the 'smpl' / 'mano' set.  -> (pose2d [B, J, 2] float64, crop
    [B, J, 2] float32 before the normalisation).  flip_before: j2d_processing on float64 joints flips before its
    result is rounded to float32 (SURREAL's ground-truth input); else float32 joints flip after it (detections)."""
    joints_px = np.asarray(joints_px, np.float32)
    B = joints_px.shape[0]
    rot = np.zeros(B, np.float32) if rot is None else np.asarray(rot, np.float32)
    flip = np.zeros(B, np.int32) if flip is None else np.asarray(flip, np.int32)
    m = io.crop_map(joints_px, input_shape)
    crop = so.crop_points(m, joints_px, rot, input_shape)
    if flip_before:
        crop = flip_2d(crop, flip, joint_set, input_shape[1])
    crop = crop.astype(np.float32)
    if not flip_before:
        crop = flip_2d(crop, flip, joint_set, input_shape[1])
    return io.normalize(crop, input_shape), crop


def cam2pixel(p, f, c):
    """lib/coord_utils.py:104-109 in fp64: p [B, J, 3] -> [B, J, 2]."""
    p = np.asarray(p, np.float64)
    return p[..., :2] / p[..., 2:3] * np.asarray(f, np.float64)[:, None, :] + np.asarray(c, np.float64)[:, None, :]


def _ones(B, n):
    return np.ones((B, n, 1))


def _rooted(mesh_cam, joints):
    """The reference's float32 rooting at joint 0 and mesh / 1000."""
    mesh_cam, joints = np.asarray(mesh_cam, np.float32), np.asarray(joints, np.float32)
    root = joints[:, :1]
    return (mesh_cam - root) / np.float32(1000), joints - root


def surreal_targets(mesh_cam, joints, f, c, rot=None, flip=None):
    """-> the SURREALTargets dict (float64 arrays; lift_pose3d and reg_pose3d the same augmented joints)."""
    B, V, J = len(mesh_cam), np.shape(mesh_cam)[1], np.shape(joints)[1]
    mesh, rooted = _rooted(mesh_cam, joints)
    rot = np.zeros(B, np.float32) if rot is None else rot
    flip = np.zeros(B, np.int32) if flip is None else flip
    lift = so.j3d_processing(rooted, rot, np.zeros(B, np.int32), "coco")    # the rotation alone
    fl = np.asarray(flip) != 0
    lift[fl] = lift[fl][:, flip_perm("smpl", J)]
    lift[fl, :, 0] = -lift[fl, :, 0]
    return {"mesh": mesh.astype(np.float64), "lift_pose3d": lift, "reg_pose3d": lift.copy(),
            "joint_img": cam2pixel(joints, f, c), "fitting_error": np.zeros(B), "mesh_valid": _ones(B, V),
            "lift_pose3d_valid": _ones(B, J), "reg_pose3d_valid": _ones(B, J), "joint_valid": _ones(B, J)}


def freihand_targets(mesh_cam, joints):
    """-> the FreiHANDTargets dict (no joint_img)."""
    B, V, J = len(mesh_cam), np.shape(mesh_cam)[1], np.shape(joints)[1]
    mesh, rooted = _rooted(mesh_cam, joints)
    return {"mesh": mesh.astype(np.float64), "lift_pose3d": rooted.astype(np.float64),
            "reg_pose3d": rooted.astype(np.float64), "fitting_error": np.zeros(B), "mesh_valid": _ones(B, V),
            "lift_pose3d_valid": _ones(B, J), "reg_pose3d_valid": _ones(B, J), "joint_valid": _ones(B, J)}


def pw3d_targets(mesh_cam, reg_h36m, reg_coco, f, c):
    """-> the PW3DTargets dict (the coco input set), regression in fp64."""
    mesh_cam = np.asarray(mesh_cam, np.float64)
    B, V = mesh_cam.shape[:2]
    coco = np.einsum("jv,bvc->bjc", np.asarray(reg_coco, np.float64), mesh_cam)
    coco = np.concatenate([coco, ((coco[:, 11] + coco[:, 12]) * 0.5)[:, None],
                           ((coco[:, 5] + coco[:, 6]) * 0.5)[:, None]], 1)
    h36m = np.einsum("jv,bvc->bjc", np.asarray(reg_h36m, np.float64), mesh_cam)
    root = h36m[:, :1]
    return {"mesh": (mesh_cam - root) / 1000, "lift_pose3d": coco - coco[:, 17:18], "reg_pose3d": h36m - root,
            "joint_img": cam2pixel(coco, f, c), "fitting_error": np.zeros(B), "mesh_valid": _ones(B, V),
            "lift_pose3d_valid": _ones(B, 19), "reg_pose3d_valid": _ones(B, 17), "joint_valid": _ones(B, 19)}
