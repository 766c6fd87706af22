#!/usr/bin/env python
"""Golden vectors of the datasets' target construction, produced from the UNMODIFIED reference:

    P2M_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_targets.py   ->  tests/golden/targets.npz

The layers are smplpytorch's SMPL_Layer and manopth's ManoLayer on the seeded synthetic models of tests/body_models.py,
built as make_golden_body_model.py builds them; coord_utils.cam2pixel / world2cam are the reference's, imported through
oracle/ref_shim.py; the regressors are the reference's J_regressor_h36m_correct.npy and J_regressor_coco.npy, stored in
the fixture as data.  The dataset modules themselves need pycocotools and transforms3d, so the bodies of their
get_smpl_coord / get_mano_coord and of Human36M.__getitem__'s target side (augmentation off) are restated below line for
line, with transforms3d's axangle2mat / mat2axangle restated too (RESTATEMENT markers).  Everything runs on CPU in the
reference's dtypes, one sample at a time as the datasets call it.

Keys: reg_h36m, reg_coco [17, 6890] float64; rows (a seeded 256 of SMPL's 6890 vertices; MANO keeps all 778); per
preset p: p__pose, p__betas, p__trans, p__R, p__t, p__mesh (on the rows), p__joints; per joint set s of the Human3.6M
assembly (inputs: the human36m preset's and h36m__f, h36m__c, h36m__joint_cam): h36m_s__mesh (rows), h36m_s__lift_pose3d,
h36m_s__reg_pose3d, h36m_s__mesh_valid (rows), h36m_s__lift_pose3d_valid, h36m_s__joint_img, h36m_s__fitting_error.
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import body_models as bm  # noqa: E402
from oracle import ref_shim  # noqa: E402

REF = os.environ.get("P2M_REFERENCE_ROOT", "")
PRESETS = ("human36m", "amass", "freihand", "muco", "coco", "surreal", "pw3d")
FACE_KPS_VERTEX = (331, 2802, 6262, 3489, 3990)
B = 4


# ---- RESTATEMENT of transforms3d.axangles (transforms3d 0.3.1) ----------------------------------------------------
def axangle2mat(axis, angle, is_normalized=False):
    x, y, z = axis
    if not is_normalized:
        n = math.sqrt(x * x + y * y + z * z)
        x = x / n
        y = y / n
        z = z / n
    c = math.cos(angle)
    s = math.sin(angle)
    C = 1 - c
    xs = x * s
    ys = y * s
    zs = z * s
    xC = x * C
    yC = y * C
    zC = z * C
    xyC = x * yC
    yzC = y * zC
    zxC = z * xC
    return np.array([[x * xC + c, xyC - zs, zxC + ys],
                     [xyC + zs, y * yC + c, yzC - xs],
                     [zxC - ys, yzC + xs, z * zC + c]])


def mat2axangle(mat, unit_thresh=1e-5):
    M = np.asarray(mat, dtype=np.float64)
    # direction: unit eigenvector of R33 corresponding to eigenvalue of 1
    L, W = np.linalg.eig(M.T)
    i = np.where(np.abs(L - 1.0) < unit_thresh)[0]
    if not len(i):
        raise ValueError("no unit eigenvector corresponding to eigenvalue 1")
    direction = np.real(W[:, i[-1]]).squeeze()
    # rotation angle depending on direction
    cosa = (np.trace(M) - 1.0) / 2.0
    if abs(direction[2]) > 1e-8:
        sina = (M[1, 0] + (cosa - 1.0) * direction[0] * direction[1]) / direction[2]
    elif abs(direction[1]) > 1e-8:
        sina = (M[0, 2] + (cosa - 1.0) * direction[0] * direction[2]) / direction[1]
    else:
        sina = (M[2, 1] + (cosa - 1.0) * direction[1] * direction[2]) / direction[0]
    angle = math.atan2(sina, cosa)
    return direction, angle


# ---- RESTATEMENT of the datasets' get_*_coord bodies (one sample) ---------------------------------------------------
def rotate_root(smpl_pose, R):
    root_pose = smpl_pose[0, :].numpy()
    angle = np.linalg.norm(root_pose)
    root_pose = axangle2mat(root_pose / angle, angle)
    root_pose = np.dot(R, root_pose)
    axis, angle = mat2axangle(root_pose)
    root_pose = axis * angle
    smpl_pose[0] = torch.from_numpy(root_pose)


def get_coord(preset, layer, pose, shape, trans, R, t):
    pose = np.array(pose)  # torch.FloatTensor shares a float32 array's memory (the dataset deep-copies its sample)
    smpl_pose = torch.FloatTensor(pose).view(-1, 3)
    smpl_shape = torch.FloatTensor(shape).view(1, -1)
    R, t = np.array(R, dtype=np.float32).reshape(3, 3), np.array(t, dtype=np.float32).reshape(3)
    if preset in ("human36m", "muco", "coco"):
        smpl_shape[(smpl_shape.abs() > 3).any(dim=1)] = 0.
    if preset in ("human36m", "amass", "freihand"):
        rotate_root(smpl_pose, R)
    smpl_pose = smpl_pose.view(1, -1)
    with torch.no_grad():
        if preset == "freihand":                                      # FreiHAND/dataset.py:110-134
            mano_trans = torch.from_numpy(t).view(-1, 3)
            m, j = layer(smpl_pose, smpl_shape, mano_trans)
            return m.numpy().reshape(-1, 3), j.numpy().reshape(-1, 3)
        if preset in ("muco", "surreal", "pw3d"):
            m, j = layer(smpl_pose, smpl_shape, torch.FloatTensor(trans).view(1, 3))
        else:
            m, j = layer(smpl_pose, smpl_shape)
    smpl_mesh_coord = m.numpy().astype(np.float32).reshape(-1, 3)
    smpl_joint_coord = j.numpy().astype(np.float32).reshape(-1, 3)
    if preset == "muco":                                              # MuCo/dataset.py:209-211
        smpl_face_kps_coord = smpl_mesh_coord[FACE_KPS_VERTEX, :].reshape(-1, 3)
        smpl_joint_coord = np.concatenate((smpl_joint_coord, smpl_face_kps_coord))
    if preset == "human36m":                                          # Human36M/dataset.py:286-294
        smpl_trans = np.array(trans, dtype=np.float32).reshape(3)
        smpl_trans = np.dot(R, smpl_trans[:, None]).reshape(1, 3) + t.reshape(1, 3) / 1000
        root_joint_coord = smpl_joint_coord[0].reshape(1, 3)
        smpl_trans = smpl_trans - root_joint_coord + np.dot(R, root_joint_coord.transpose(1, 0)).transpose(1, 0)
        smpl_mesh_coord += smpl_trans
        smpl_joint_coord += smpl_trans
    if preset == "amass":                                             # AMASS/dataset.py:206-208
        smpl_mesh_coord += t.reshape(-1, 3)
        smpl_joint_coord += t.reshape(-1, 3)
    smpl_mesh_coord *= 1000
    smpl_joint_coord *= 1000
    return smpl_mesh_coord, smpl_joint_coord


# ---- RESTATEMENT of Human36M's target side (dataset.py:301-333,344-405, augmentation off) -------------------------
def h36m_sample(cu, reg_h36m, reg_coco, mesh_cam, joint_cam_h36m, f, c, joint_set, fitting_thr=25):
    def add_pelvis_and_neck(joint_coord):
        pelvis = ((joint_coord[11, :] + joint_coord[12, :]) * 0.5).reshape((1, -1))
        neck = ((joint_coord[5, :] + joint_coord[6, :]) * 0.5).reshape((1, -1))
        return np.concatenate((joint_coord, pelvis, neck))

    joint_cam_coco = add_pelvis_and_neck(np.dot(reg_coco, mesh_cam))
    joint_img_coco = cu.cam2pixel(joint_cam_coco, f, c)
    joint_img_h36m = cu.cam2pixel(joint_cam_h36m, f, c)[:, :2]
    mesh_cam = mesh_cam - joint_cam_h36m[:1]
    joint_cam_coco = joint_cam_coco - joint_cam_coco[-2:-1]
    joint_cam_h36m = joint_cam_h36m - joint_cam_h36m[:1]
    if joint_set == "coco":
        joint_img, joint_cam = joint_img_coco[:, :2], joint_cam_coco
    else:
        joint_img, joint_cam = joint_img_h36m, joint_cam_h36m
    mesh_valid = np.ones((len(mesh_cam), 1), dtype=np.float32)
    lift_joint_valid = np.ones((len(joint_cam), 1), dtype=np.float32)
    h = joint_cam_h36m - joint_cam_h36m[0, None, :]
    s = np.dot(reg_h36m, mesh_cam)
    s = s - np.mean(s, 0)[None, :] + np.mean(h, 0)[None, :]
    error = np.sqrt(np.sum((h - s) ** 2, 1)).mean()
    if error > fitting_thr:
        mesh_valid[:] = 0
        if joint_set == "coco":
            lift_joint_valid[:] = 0
    return {"mesh": mesh_cam / 1000, "lift_pose3d": joint_cam, "reg_pose3d": joint_cam_h36m, "mesh_valid": mesh_valid,
            "lift_pose3d_valid": lift_joint_valid, "joint_img": joint_img, "fitting_error": np.array(error)}


# ---- seeded inputs (shared with the tests) ---------------------------------------------------------------------------
def rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                  2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                  2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1)
    return R.reshape(n, 3, 3).astype(np.float32)


def inputs(rng, n, n_pose, mano=False):
    """pose, betas (sample 1: one |beta| > 3; sample 2: all zero), trans (metres), R, t (mm for the H36M camera,
    metres elsewhere), as float32."""
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    pose = f32(rng.normal(0, 0.4, (n, n_pose)))
    pose[:, :3] = bm.random_axisang(rng, n, 0.2, 3.0)
    betas = f32(rng.normal(0, 1.0, (n, 10)))
    betas[:, 0] = np.clip(betas[:, 0], -2.5, 2.5)
    if n > 1:
        betas[1, 3] = 3.5
    if n > 2:
        betas[2] = 0
    trans = f32(rng.normal(0, 0.3, (n, 3)))
    R = rotations(rng, n)
    t = f32(rng.normal(0, 0.05 if mano else 0.3, (n, 3)) + ([0, 0, 0.5] if mano else [0, 0, 4.0]))
    return pose, betas, trans, R, t


def main():
    if not ref_shim.available():
        raise SystemExit("set P2M_REFERENCE_ROOT to a Pose2Mesh_RELEASE checkout")
    ref_shim.load()
    import coord_utils as cu  # reference module, lib/ on sys.path after ref_shim.load()
    sys.path[:0] = [os.path.join(REF, "smplpytorch"), os.path.join(REF, "manopth")]
    from manopth.manolayer import ManoLayer
    from smplpytorch.pytorch.smpl_layer import SMPL_Layer

    torch.set_num_threads(1)
    smpl, mano = bm.smpl_model(), bm.mano_model("right", False)
    smpl_layer = bm.smpl_reference_layer(SMPL_Layer, smpl)
    mano_layer = bm.mano_reference_layer(ManoLayer, mano)
    rng = np.random.RandomState(77)
    rows = np.sort(rng.choice(6890, 256, replace=False)).astype(np.int32)
    Z = {"rows": rows, "digest_smpl": np.array(bm.digest(smpl)), "digest_mano": np.array(bm.digest(mano)),
         "reg_h36m": np.load(os.path.join(REF, "data", "Human36M", "J_regressor_h36m_correct.npy")).astype(np.float64),
         "reg_coco": np.load(os.path.join(REF, "data", "COCO", "J_regressor_coco.npy")).astype(np.float64)}
    for p in PRESETS:
        mano_p = p == "freihand"
        pose, betas, trans, R, t = inputs(rng, B, 48 if mano_p else 72, mano_p)
        if p == "human36m":
            t = t * 1000  # the H36M camera's t is in millimetres
        out = [get_coord(p, mano_layer if mano_p else smpl_layer, pose[i], betas[i], trans[i], R[i], t[i])
               for i in range(B)]
        for k, v in (("pose", pose), ("betas", betas), ("trans", trans), ("R", R), ("t", t)):
            Z[f"{p}__{k}"] = v
        Z[f"{p}__mesh"] = np.stack([m if mano_p else m[rows] for m, _ in out])
        Z[f"{p}__joints"] = np.stack([j for _, j in out])
    # the Human3.6M assembly: joint_cam = world2cam(joints near the fitted mesh's H36M joints), two of the four samples
    # far enough off to fail the 25 mm fit test
    pose, betas, trans, R, t = (Z[f"human36m__{k}"] for k in ("pose", "betas", "trans", "R", "t"))
    f = np.asarray(rng.uniform(1100, 1200, (B, 2)), np.float32)
    c = np.asarray(rng.uniform(480, 540, (B, 2)), np.float32)
    joint_cam = []
    for i in range(B):
        mesh_cam, _ = get_coord("human36m", smpl_layer, pose[i], betas[i], trans[i], R[i], t[i])
        reg = np.dot(Z["reg_h36m"], mesh_cam)
        noise = rng.normal(0, 4.0 if i % 2 == 0 else 60.0, reg.shape)
        joint_world = np.dot(R[i].T.astype(np.float64), (reg + noise - t[i]).T).T
        joint_cam.append(cu.world2cam(joint_world, R[i], t[i]))
    joint_cam = np.asarray(joint_cam, np.float32)
    for k, v in (("f", f), ("c", c), ("joint_cam", joint_cam)):
        Z[f"h36m__{k}"] = v
    for s in ("human36", "coco"):
        outs = []
        for i in range(B):
            mesh_cam, _ = get_coord("human36m", smpl_layer, pose[i], betas[i], trans[i], R[i], t[i])
            outs.append(h36m_sample(cu, Z["reg_h36m"], Z["reg_coco"], mesh_cam, joint_cam[i].astype(np.float64), f[i],
                                    c[i], s))
        for k in outs[0]:
            v = np.stack([o[k] for o in outs])
            Z[f"h36m_{s}__{k}"] = v[:, rows] if k in ("mesh", "mesh_valid") else v
        print(s, "fitting errors", Z[f"h36m_{s}__fitting_error"])
    path = os.path.join(HERE, "targets.npz")
    np.savez_compressed(path, **Z)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
