#!/usr/bin/env python
"""Golden vectors of the SURREAL, FreiHAND and 3DPW samples, produced from the UNMODIFIED reference:

    P2M_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_smpl_mano_samples.py
        ->  tests/golden/smpl_mano_samples.npz

lib/coord_utils.py (get_bbox, process_bbox, cam2pixel) and lib/aug_utils.py (j2d_processing, j3d_processing,
flip_2d_joint) are the reference's, imported through oracle/ref_shim.py with a cfg.AUG stub.  The datasets' modules need
pycocotools, so their __getitem__ bodies are restated line by line (RESTATEMENT markers).

Inputs: the 'surreal' and 'freihand' camera-frame meshes and joints of tests/golden/targets.npz (SURREAL's mesh is its
256 golden rows, since the assembly is per vertex, moved 3-6 m along z in float32 so that it is in front of the
camera), and for 3DPW, whose regressors need whole meshes, the three synthetic SMPL
meshes fit__mesh of tests/golden/samples.npz with targets.npz's regressors.  Seeded f, c (float32 values, handed to the
reference as float64 arrays as its JSON gives them) and detections (float32; 3DPW's with pelvis and neck appended as
(a + b) * 0.5 in float32).

Keys (C cases, A = len(AUG_CASES)):
  aug_cases [A, 2] (flip, rot float32)
  surreal__mesh_in [C, 256, 3], surreal__joints_in [C, 24, 3], surreal__f, surreal__c [C, 2], surreal__det [C, 24, 2]
  float32; surreal__gt [C, 24, 2] float64 (cam2pixel, use_gt_input); surreal__mesh [C, 256, 3] float32;
  surreal__lift [C, A, 24, 3] float32 (also reg_pose3d); surreal__crop_{det,gt} [C, A, 24, 2] float32 (j2d_processing);
  surreal__pose2d_{det,gt} [C, A, 24, 2] (the normalised input)
  freihand__mesh_in [C, 778, 3], freihand__joints_in [C, 21, 3], freihand__det [C, 21, 2]; freihand__mesh [C, 778, 3],
  freihand__joints [C, 21, 3] float32 (lift_pose3d = reg_pose3d); freihand__crop, freihand__pose2d [C, 21, 2]
  pw3d__mesh_index [C], pw3d__f, pw3d__c [C, 2], pw3d__det [C, 19, 2]; pw3d__rows [256]; pw3d__mesh [C, 256, 3]
  (those rows), pw3d__reg [C, 17, 3], pw3d__lift [C, 19, 3] float32; pw3d__joint_img [C, 19, 2] float64 (gt input);
  pw3d__crop, pw3d__pose2d [C, 19, 2]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

INPUT_SHAPE = (384, 288)
SMPL_FLIP_PAIRS = ((1, 2), (4, 5), (7, 8), (10, 11), (13, 14), (16, 17), (18, 19), (20, 21), (22, 23))
AUG_CASES = ((0, 0.0), (1, 0.0), (0, 17.3), (1, -40.0))
COCO_JOINTS = ('Nose', 'L_Eye', 'R_Eye', 'L_Ear', 'R_Ear', 'L_Shoulder', 'R_Shoulder', 'L_Elbow', 'R_Elbow', 'L_Wrist',
               'R_Wrist', 'L_Hip', 'R_Hip', 'L_Knee', 'R_Knee', 'L_Ankle', 'R_Ankle')


class _Aug:
    flip = False
    rotate_factor = 0.0


def camera(rng, C):
    f = rng.uniform(900, 1600, (C, 2)).astype(np.float32)
    c = rng.uniform(200, 600, (C, 2)).astype(np.float32)
    return f, c


def main():
    ref_shim.load()
    ref_shim._Cfg.AUG = _Aug
    import aug_utils  # noqa: E402  (reference module)
    import coord_utils  # noqa: E402

    tg = np.load(os.path.join(HERE, "targets.npz"))
    sm = np.load(os.path.join(HERE, "samples.npz"))
    rng = np.random.default_rng(20261018)
    res = (INPUT_SHAPE[1], INPUT_SHAPE[0])
    out = {"aug_cases": np.array(AUG_CASES, np.float64)}

    def normalise(joint_coord_img):
        # the shared tail of the three __getitem__: -> 0~1, then loc / scale
        joint_coord_img = joint_coord_img[:, :2]
        joint_coord_img /= np.array([[INPUT_SHAPE[1], INPUT_SHAPE[0]]])
        mean, std = np.mean(joint_coord_img, axis=0), np.std(joint_coord_img, axis=0)
        return (joint_coord_img.copy() - mean) / std

    # ------------------------------------------------------------------------------------------------- SURREAL
    # the preset's bodies sit at the origin: moved 3-6 m in front of the camera so cam2pixel sees them
    C, V = tg["surreal__mesh"].shape[:2]
    depth = np.zeros((C, 1, 3), np.float32)
    depth[:, 0, 2] = rng.uniform(3000, 6000, C).astype(np.float32)
    mesh_in, joints_in = tg["surreal__mesh"] + depth, tg["surreal__joints"] + depth
    f, c = camera(rng, C)
    A = len(AUG_CASES)
    det = np.zeros((C, 24, 2), np.float32)
    gt = np.zeros((C, 24, 2), np.float64)
    mesh_t = np.zeros((C, V, 3), np.float32)
    lift = np.zeros((C, A, 24, 3), np.float32)
    crops = {k: np.zeros((C, A, 24, 2), np.float32) for k in ("det", "gt")}
    pose2d = {k: np.zeros((C, A, 24, 2), np.float64) for k in ("det", "gt")}
    for i in range(C):
        cam_param = {"focal": f[i].astype(np.float64), "princpt": c[i].astype(np.float64)}
        for a, (fl, rot) in enumerate(AUG_CASES):
            rot = float(np.float32(rot))
            for kind in ("det", "gt"):
                # ---- RESTATEMENT of SURREAL.__getitem__ (data/SURREAL/dataset.py:143-203) ----------------------
                smpl_mesh_coord_cam, smpl_joint_coord_cam = mesh_in[i].copy(), joints_in[i].copy()
                smpl_coord_cam = np.concatenate((smpl_mesh_coord_cam, smpl_joint_coord_cam))
                smpl_coord_img = coord_utils.cam2pixel(smpl_coord_cam, cam_param['focal'], cam_param['princpt'])
                joint_coord_img = smpl_coord_img[V:][:, :2]
                smpl_coord_cam = smpl_coord_cam - smpl_coord_cam[V + 0]
                mesh_coord_cam = smpl_coord_cam[:V]
                joint_coord_cam = smpl_coord_cam[V:]
                if kind == "det":
                    if a == 0:
                        det[i] = (joint_coord_img + rng.normal(0, 6.0, (24, 2))).astype(np.float32)
                    joint_coord_img = det[i].copy()
                else:
                    gt[i] = joint_coord_img
                bbox = coord_utils.get_bbox(joint_coord_img)
                bbox = coord_utils.process_bbox(bbox.copy())
                joint_coord_img, trans = aug_utils.j2d_processing(joint_coord_img.copy(), res, bbox, rot, fl,
                                                                  SMPL_FLIP_PAIRS)
                joint_coord_cam = aug_utils.j3d_processing(joint_coord_cam, rot, fl, SMPL_FLIP_PAIRS)
                crops[kind][i, a] = joint_coord_img[:, :2]
                pose2d[kind][i, a] = normalise(joint_coord_img)
                targets = {'mesh': mesh_coord_cam / 1000, 'lift_pose3d': joint_coord_cam,
                           'reg_pose3d': joint_coord_cam}
                # ---- end RESTATEMENT ---------------------------------------------------------------------------
                assert targets['reg_pose3d'] is targets['lift_pose3d']
                mesh_t[i], lift[i, a] = targets['mesh'], targets['lift_pose3d']
    out.update({"surreal__mesh_in": mesh_in, "surreal__joints_in": joints_in, "surreal__f": f, "surreal__c": c,
                "surreal__det": det, "surreal__gt": gt, "surreal__mesh": mesh_t, "surreal__lift": lift,
                "surreal__crop_det": crops["det"], "surreal__crop_gt": crops["gt"],
                "surreal__pose2d_det": pose2d["det"], "surreal__pose2d_gt": pose2d["gt"]})

    # ------------------------------------------------------------------------------------------------ FreiHAND
    mesh_in, joints_in = tg["freihand__mesh"], tg["freihand__joints"]
    C, V = mesh_in.shape[:2]
    det = np.zeros((C, 21, 2), np.float32)
    mesh_t = np.zeros((C, V, 3), np.float32)
    joints_t = np.zeros((C, 21, 3), np.float32)
    crop = np.zeros((C, 21, 2), np.float32)
    p2d = np.zeros((C, 21, 2), np.float64)
    for i in range(C):
        centre, size = rng.uniform([200, 150], [500, 400]), rng.uniform(60, 250)
        det[i] = (centre + rng.uniform(-1, 1, (21, 2)) * [size * (1.4 if i % 2 else 0.5), size]).astype(np.float32)
        # ---- RESTATEMENT of FreiHAND.__getitem__ (data/FreiHAND/dataset.py:139-192) --------------------------------
        rot, flip = 0, 0
        mano_mesh_cam, mano_joint_cam = mesh_in[i].copy(), joints_in[i].copy()
        mano_coord_cam = np.concatenate((mano_mesh_cam, mano_joint_cam))
        mano_coord_cam = mano_coord_cam - mano_joint_cam[:1]
        mesh_coord_cam = mano_coord_cam[:V]
        joint_coord_cam = mano_coord_cam[V:]
        joint_coord_img = det[i].copy()
        bbox = coord_utils.get_bbox(joint_coord_img)
        bbox = coord_utils.process_bbox(bbox.copy())
        joint_coord_img, trans = aug_utils.j2d_processing(joint_coord_img.copy(), res, bbox, rot, flip, None)
        crop[i] = joint_coord_img[:, :2]
        p2d[i] = normalise(joint_coord_img)
        targets = {'mesh': mesh_coord_cam / 1000, 'lift_pose3d': joint_coord_cam, 'reg_pose3d': joint_coord_cam}
        # ---- end RESTATEMENT -------------------------------------------------------------------------------------
        mesh_t[i], joints_t[i] = targets['mesh'], targets['reg_pose3d']
    out.update({"freihand__mesh_in": mesh_in, "freihand__joints_in": joints_in, "freihand__det": det,
                "freihand__mesh": mesh_t, "freihand__joints": joints_t, "freihand__crop": crop,
                "freihand__pose2d": p2d})

    # ---------------------------------------------------------------------------------------------------- 3DPW
    meshes = sm["fit__mesh"]
    reg_h36m, reg_coco = torch.Tensor(tg["reg_h36m"]), torch.Tensor(tg["reg_coco"])
    rows = tg["rows"]
    C = 4
    mi = np.arange(C) % len(meshes)
    f, c = camera(rng, C)
    keys = ("mesh", "reg", "lift", "joint_img", "crop", "pose2d", "det")
    pw = {k: [] for k in keys}

    def add_pelvis_and_neck(joint_coord, joints_name):  # PW3D.add_pelvis_and_neck (:168-183), only_pelvis=False
        lhip_idx, rhip_idx = joints_name.index('L_Hip'), joints_name.index('R_Hip')
        pelvis = ((joint_coord[lhip_idx, :] + joint_coord[rhip_idx, :]) * 0.5).reshape((1, -1))
        lsh_idx, rsh_idx = joints_name.index('L_Shoulder'), joints_name.index('R_Shoulder')
        neck = ((joint_coord[lsh_idx, :] + joint_coord[rsh_idx, :]) * 0.5).reshape((1, -1))
        return np.concatenate((joint_coord, pelvis, neck))

    for i in range(C):
        cam_param = {"focal": f[i].astype(np.float64), "princpt": c[i].astype(np.float64)}
        # ---- RESTATEMENT of PW3D.__getitem__ (data/PW3D/dataset.py:208-261) and its helpers (:185-206) --------------
        rot, flip = 0, 0
        mesh_cam = meshes[mi[i]].copy()
        joint_cam_coco = torch.matmul(reg_coco, torch.Tensor(mesh_cam)).numpy()
        joint_cam_coco = add_pelvis_and_neck(joint_cam_coco, COCO_JOINTS)
        gt_joint_img_coco = coord_utils.cam2pixel(joint_cam_coco, cam_param['focal'], cam_param['princpt'])
        gt_joint_img_coco[:, 2] = 1
        joint_cam_h36m = torch.matmul(reg_h36m, torch.Tensor(mesh_cam)).numpy()
        mesh_cam = mesh_cam - joint_cam_h36m[:1]
        joint_cam_coco = joint_cam_coco - joint_cam_coco[-2:-1]
        joint_cam_h36m = joint_cam_h36m - joint_cam_h36m[:1]
        det17 = (gt_joint_img_coco[:17, :2] + rng.normal(0, 4.0, (17, 2))).astype(np.float32)
        joint_img_coco = add_pelvis_and_neck(det17, COCO_JOINTS)           # the detections' pelvis and neck
        bbox = coord_utils.get_bbox(joint_img_coco)
        bbox = coord_utils.process_bbox(bbox.copy())
        joint_img_coco, trans = aug_utils.j2d_processing(joint_img_coco.copy(), res, bbox, rot, flip, None)
        pw["crop"].append(joint_img_coco[:, :2].copy())
        pw["pose2d"].append(normalise(joint_img_coco))
        targets = {'mesh': mesh_cam / 1000, 'reg_pose3d': joint_cam_h36m}
        # ---- end RESTATEMENT -------------------------------------------------------------------------------------
        pw["det"].append(add_pelvis_and_neck(det17, COCO_JOINTS))
        pw["mesh"].append(targets['mesh'][rows])
        pw["reg"].append(targets['reg_pose3d'])
        pw["lift"].append(joint_cam_coco)                                   # posenet's target
        pw["joint_img"].append(gt_joint_img_coco[:, :2])
    out.update({f"pw3d__{k}": np.stack(v) for k, v in pw.items()})
    out.update({"pw3d__mesh_index": mi, "pw3d__f": f, "pw3d__c": c, "pw3d__rows": rows})

    path = os.path.join(HERE, "smpl_mano_samples.npz")
    np.savez_compressed(path, **out)
    print(path, {k: (v.shape, v.dtype.name) for k, v in out.items()})


if __name__ == "__main__":
    main()
