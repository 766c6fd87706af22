#!/usr/bin/env python
"""Golden vectors of the training sample's augmentation, produced from the UNMODIFIED reference:

    P2M_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_samples.py   ->  tests/golden/samples.npz

lib/aug_utils.py (augm_params, j2d_processing, flip_2d_joint, j3d_processing) and lib/coord_utils.py (get_bbox,
process_bbox) are the reference's, imported through oracle/ref_shim.py with a cfg.AUG stub.  The datasets' modules
need pycocotools, so the order in which their __getitem__ applies these steps is restated (RESTATEMENT markers):
Human36M / COCO / AMASS crop with rot and no flip, then flip_2d_joint in float32 (data/Human36M/dataset.py:365-372);
MuCo flips inside j2d_processing (data/MuCo/dataset.py:290-296).  No noise: the noise's order is tested on the device
against the oracle, which restates the same rule.

Keys:
  augm_settings [4, 2] (flip, rotate_factor); augm_M; augm_flips [4], augm_zero [4] (rot == 0), augm_clip [4]
  (|rot| == 2 rf), augm_hist [4, N_BINS] (the nonzero rot in N_BINS equal bins of [-2 rf, 2 rf]); augm_bins
  geometry: for s in (coco, human36): s__joints [C, J, 2] float32 image pixels, s__lift [C, J, 3] float64
  (human36: float32 values), aug_cases [A, 2] (flip, rot float32), s__crop_after [C, A, J, 2] float32 (flip after),
  s__crop_before [C, A, J, 2] float32 (MuCo's flip inside j2d_processing), s__lift_aug [C, A, J, 3] float32
  fitting tests of COCO and MuCo: see fitting_cases
"""
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

INPUT_SHAPE = (384, 288)
COCO_FLIP_PAIRS = ((1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))
H36M_FLIP_PAIRS = ((1, 4), (2, 5), (3, 6), (14, 11), (15, 12), (16, 13))
AUG_CASES = ((0, 0.0), (1, 0.0), (0, 17.3), (1, -40.0))
AUGM_SETTINGS = ((0, 0.0), (1, 0.0), (0, 30.0), (1, 30.0))
AUGM_M = 40000
N_BINS = 16
N_CASES = 6


class _Aug:
    flip = False
    rotate_factor = 0.0


MUCO_JOINTS = ('Head_top', 'Thorax', 'R_Shoulder', 'R_Elbow', 'R_Wrist', 'L_Shoulder', 'L_Elbow', 'L_Wrist', 'R_Hip',
               'R_Knee', 'R_Ankle', 'L_Hip', 'L_Knee', 'L_Ankle', 'Pelvis', 'Spine', 'Head', 'R_Hand', 'L_Hand',
               'R_Toe', 'L_Toe')
H36M_JOINTS = ('Pelvis', 'R_Hip', 'R_Knee', 'R_Ankle', 'L_Hip', 'L_Knee', 'L_Ankle', 'Torso', 'Neck', 'Nose', 'Head',
               'L_Shoulder', 'L_Elbow', 'L_Wrist', 'R_Shoulder', 'R_Elbow', 'R_Wrist')


def fitting_cases(rng, coord_utils, aug_utils):
    """The fitting tests of COCO and MuCo on the synthetic SMPL template (tests/body_models.py) with the fixture's
    H36M / COCO regressors (tests/golden/targets.npz).  Keys: fit__mesh [3, V, 3] float32 (mm, camera frame);
    coco_fit__s [4], coco_fit__t [4, 2], coco_fit__kps [4, 17, 2], coco_fit__valid [4, 17], coco_fit__mesh_index [4],
    coco_fit__set [4] (1: the coco input set), coco_fit__error [4]; muco_fit__error [3]."""
    sys.path.insert(0, os.path.dirname(HERE))
    import body_models as bm  # noqa: E402
    tg = np.load(os.path.join(HERE, "targets.npz"))
    reg_h36m, reg_coco = tg["reg_h36m"], tg["reg_coco"]
    tmpl = bm.smpl_model()["v_template"].astype(np.float64)
    meshes = np.stack([((tmpl + rng.normal(0, 0.01, tmpl.shape)) * 1000 + [0, 0, 5000 + 500 * k]).astype(np.float32)
                       for k in range(3)])
    out = {"fit__mesh": meshes}

    # ---- RESTATEMENT of MuCo.get_fitting_error (data/MuCo/dataset.py:246-262), called as __getitem__ does (:317)
    def muco_fitting_error(muco_joint, smpl_mesh):
        muco_joint = muco_joint.copy()
        muco_joint = muco_joint - muco_joint[MUCO_JOINTS.index('Pelvis'), None, :]
        muco_joint_valid = np.ones((21, 3), dtype=np.float32)
        h36m_joint = aug_utils.transform_joint_to_other_db(muco_joint, MUCO_JOINTS, H36M_JOINTS)
        h36m_joint_valid = aug_utils.transform_joint_to_other_db(muco_joint_valid, MUCO_JOINTS, H36M_JOINTS)
        h36m_joint = h36m_joint[h36m_joint_valid == 1].reshape(-1, 3)
        h36m_from_smpl = np.dot(reg_h36m, smpl_mesh)
        h36m_from_smpl = h36m_from_smpl[h36m_joint_valid == 1].reshape(-1, 3)
        h36m_from_smpl = h36m_from_smpl - np.mean(h36m_from_smpl, 0)[None, :] + np.mean(h36m_joint, 0)[None, :]
        return np.sqrt(np.sum((h36m_joint - h36m_from_smpl) ** 2, 1)).mean()

    errs = []
    for mesh_cam in meshes:
        joint_cam_h36m = np.dot(reg_h36m, mesh_cam)
        mesh_rooted = mesh_cam - joint_cam_h36m[:1]
        errs.append(muco_fitting_error(joint_cam_h36m - joint_cam_h36m[:1], mesh_rooted))
    out["muco_fit__error"] = np.array(errs)

    # ---- RESTATEMENT of COCO.get_fitting_error (data/COCO/dataset.py:196-214) and its call (:227-258, 272)
    def coco_fitting_error(bbox, coco_from_dataset, coco_from_smpl, coco_joint_valid):
        bbox = coord_utils.process_bbox(bbox.copy(), aspect_ratio=1.0)
        coco_from_smpl_xy1 = np.concatenate((coco_from_smpl[:, :2], np.ones_like(coco_from_smpl[:, 0:1])), 1)
        coco_from_smpl, _ = aug_utils.j2d_processing(coco_from_smpl_xy1, (64, 64), bbox, 0, 0, None)
        coco_from_dataset_xy1 = np.concatenate((coco_from_dataset[:, :2], np.ones_like(coco_from_smpl[:, 0:1])), 1)
        coco_from_dataset, trans = aug_utils.j2d_processing(coco_from_dataset_xy1, (64, 64), bbox, 0, 0, None)
        coco_joint = coco_from_dataset[:, :2][np.tile(coco_joint_valid, (1, 2)) == 1].reshape(-1, 2)
        coco_from_smpl = coco_from_smpl[:, :2][np.tile(coco_joint_valid, (1, 2)) == 1].reshape(-1, 2)
        return np.sqrt(np.sum((coco_joint - coco_from_smpl) ** 2, 1)).mean()

    def project(joint_coord_cam, s, t):  # get_joints_from_mesh's projection (:200-210)
        return (joint_coord_cam[:, :2] / 1000) * s + t.reshape(-1, 2)

    cs, ct, ck, cv, cm, cset, ce = [], [], [], [], [], [], []
    for k, (noise_px, n_vis, coco_set) in enumerate(((0.5, 17, 1), (40.0, 12, 0), (0.3, 9, 0), (1.0, 0, 1))):
        mi = k % 3
        s_ = np.float32(rng.uniform(180, 260))
        t_ = rng.uniform(300, 500, 2).astype(np.float32)
        coco = np.dot(reg_coco, meshes[mi])
        coco19 = np.concatenate([coco, (coco[11:12] + coco[12:13]) * 0.5, (coco[5:6] + coco[6:7]) * 0.5])
        h36m = np.dot(reg_h36m, meshes[mi])
        joint_img = project(coco19 if coco_set else h36m, s_, t_)
        joint_img_coco = project(coco19, s_, t_)
        kps = (joint_img_coco[:17] + rng.normal(0, noise_px, (17, 2))).astype(np.float32)
        valid = np.zeros((17, 1), np.float32)
        valid[rng.permutation(17)[:n_vis]] = 1
        tight_bbox = coord_utils.get_bbox(joint_img)
        with np.errstate(invalid="ignore"):
            err = coco_fitting_error(tight_bbox, np.concatenate([kps, np.zeros((17, 1), np.float32)], 1),
                                     joint_img_coco[:17], valid)
        cs.append(s_), ct.append(t_), ck.append(kps), cv.append(valid[:, 0]), cm.append(mi), cset.append(coco_set)
        ce.append(err)
    # ---- end RESTATEMENT
    out.update({"coco_fit__s": np.array(cs), "coco_fit__t": np.array(ct), "coco_fit__kps": np.array(ck),
                "coco_fit__valid": np.array(cv), "coco_fit__mesh_index": np.array(cm),
                "coco_fit__set": np.array(cset), "coco_fit__error": np.array(ce)})
    return out


def main():
    ref_shim.load()
    ref_shim._Cfg.AUG = _Aug
    import aug_utils  # noqa: E402  (reference module)
    import coord_utils  # noqa: E402

    out = {"augm_settings": np.array(AUGM_SETTINGS, np.float64), "augm_M": np.int64(AUGM_M),
           "augm_bins": np.int64(N_BINS), "aug_cases": np.array(AUG_CASES, np.float64)}
    flips, zeros, clips, hists = [], [], [], []
    for k, (fl, rf) in enumerate(AUGM_SETTINGS):
        _Aug.flip, _Aug.rotate_factor = bool(fl), rf
        random.seed(1000 + k)
        np.random.seed(2000 + k)
        draws = np.array([aug_utils.augm_params(True) for _ in range(AUGM_M)], np.float64)
        f, r = draws[:, 0], draws[:, 1]
        flips.append(int((f == 1).sum()))
        zeros.append(int((r == 0).sum()))
        clips.append(int((np.abs(r) == 2 * rf).sum()) if rf > 0 else 0)
        nz = r[r != 0]
        hists.append(np.histogram(nz, bins=N_BINS, range=(-2 * rf, 2 * rf))[0] if rf > 0 else np.zeros(N_BINS, int))
    out.update(augm_flips=np.array(flips), augm_zero=np.array(zeros), augm_clip=np.array(clips),
               augm_hist=np.array(hists))

    rng = np.random.default_rng(20261017)
    res = (INPUT_SHAPE[1], INPUT_SHAPE[0])
    for name, J, pairs in (("coco", 19, COCO_FLIP_PAIRS), ("human36", 17, H36M_FLIP_PAIRS)):
        joints = np.zeros((N_CASES, J, 2), np.float32)
        lift = np.zeros((N_CASES, J, 3), np.float64)
        after = np.zeros((N_CASES, len(AUG_CASES), J, 2), np.float32)
        before = np.zeros_like(after)
        lift_aug = np.zeros((N_CASES, len(AUG_CASES), J, 3), np.float32)
        for c in range(N_CASES):
            centre = rng.uniform([200, 200], [1000, 800])
            size = rng.uniform(80, 500) * (1.0 if c % 2 else 0.4)      # wide and tall boxes
            joints[c] = (centre + rng.uniform(-1, 1, (J, 2)) * [size * (1.6 if c % 3 == 0 else 0.5), size]
                         ).astype(np.float32)
            lift[c] = rng.uniform(-900, 900, (J, 3))
            if name == "human36":
                lift[c] = lift[c].astype(np.float32)                     # the annotation's float32 joint_cam
            for a, (fl, rot) in enumerate(AUG_CASES):
                rot = float(np.float32(rot))
                # ---- RESTATEMENT of the datasets' __getitem__ (crop box and augmentation order) ----------------
                kp = joints[c].astype(np.float64)
                tight = coord_utils.get_bbox(kp)
                bbox = coord_utils.process_bbox(tight.copy())
                img, _ = aug_utils.j2d_processing(kp.copy(), res, bbox, rot, 0, None)
                if fl:
                    img = aug_utils.flip_2d_joint(img, INPUT_SHAPE[1], pairs)
                after[c, a] = img
                img, _ = aug_utils.j2d_processing(kp.copy(), res, bbox, rot, fl, pairs)
                before[c, a] = img
                lift_aug[c, a] = aug_utils.j3d_processing(lift[c].copy(), rot, fl, pairs)
                # ---- end RESTATEMENT ---------------------------------------------------------------------------
        out.update({f"{name}__joints": joints, f"{name}__lift": lift, f"{name}__crop_after": after,
                    f"{name}__crop_before": before, f"{name}__lift_aug": lift_aug})
    out.update(fitting_cases(rng, coord_utils, aug_utils))
    path = os.path.join(HERE, "samples.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
