"""The SURREAL, FreiHAND and 3DPW sample rules (tests/smpl_mano_oracle.py) against the unmodified reference
(tests/golden/smpl_mano_samples.npz): the 'smpl' crop with rotation and flip in both flip orders, the 'mano' crop, and
the three datasets' targets.

Bounds.  The crops: one float32 ulp, and for rot = 0 the closed-form scale's difference that test_samples_cpu.py
derives.  The reference's float32 steps (rooting, mesh / 1000) are the rule, so SURREAL's and FreiHAND's meshes and
FreiHAND's joints match bit for bit.  SURREAL's joint_img: the reference divides x / z in float32 before its float64
product with f, half a float32 ulp of x / z times f.  3DPW: the reference regresses in float32 (torch.matmul), the
oracle in fp64; pw3d_bounds gives the float32 dot product's worst case, (n + 1) 2^-24 sum |r| |m| for a row of n
non-zeros (the + 1 is the regressor's own float32 cast), carried through the rooting, the pelvis / neck means and the
projection.
"""
import os

import numpy as np
import pytest

import smpl_mano_oracle as smo
from oracle import inputs_oracle as io

HERE = os.path.dirname(__file__)
GOLDEN = np.load(os.path.join(HERE, "golden", "smpl_mano_samples.npz"))
TARGETS = np.load(os.path.join(HERE, "golden", "targets.npz"))
SAMPLES = np.load(os.path.join(HERE, "golden", "samples.npz"))
U = 2.0 ** -24


def aug_case(a):
    fl, rot = GOLDEN["aug_cases"][a]
    return int(fl), np.float32(rot)


def crop_ok(crop, want, joints, rot, fl, extra=0.0):
    """One float32 ulp (the flipped x's pre-flip value counts too), or for rot = 0 the closed form's scale.  With
    float32 joints, NumPy 2 computes get_bbox's centre and size in float32 where the library (like NumPy 1, which the
    reference was written for) takes them in float64: that moves the box by up to two float32 ulps of the largest
    coordinate, and every crop point by that times the crop's scale."""
    got, want = np.asarray(crop, np.float64), np.asarray(want, np.float64)
    mag = np.maximum(np.abs(got), np.abs(want))
    if fl:
        mag[..., 0] = np.maximum(mag[..., 0], np.abs(287 - want[..., 0]))
    m = io.crop_map(joints)
    box = 2 * m["sc"] * np.spacing(np.abs(np.asarray(joints, np.float32)).max(axis=(1, 2)))
    tol = np.spacing(mag.astype(np.float32)).astype(np.float64) + extra + box[:, None, None]
    if rot == 0:
        rel = np.spacing(np.abs(m["ccx"]).astype(np.float32) + m["crop_w"].astype(np.float32)) / (m["crop_w"] / 2)
        tol = tol + rel[:, None, None] * np.abs(want - [144.0, 192.0]) + 1e-5
    return np.abs(got - want) <= tol


@pytest.mark.parametrize("kind", ["det", "gt"])
def test_smpl_crop_matches_reference(kind):
    """det: float32 detections, flipped in float32 after the crop; gt: float64 cam2pixel joints, flipped in fp64 before
    the crop is rounded.  The oracle takes the gt joints rounded to float32, as the device does: that moves a joint by
    half an ulp of its pixel value, times the crop's scale (below 4 crop pixels per image pixel here)."""
    joints = GOLDEN[f"surreal__{kind}"].astype(np.float32)
    extra = 0.0 if kind == "det" else 4 * 0.5 * np.spacing(np.float32(1024.0))
    C = joints.shape[0]
    for a in range(len(GOLDEN["aug_cases"])):
        fl, rot = aug_case(a)
        p2d, crop = smo.training_pose2d(joints, "smpl", rot=np.full(C, rot), flip=np.full(C, fl),
                                        flip_before=kind == "gt")
        want = GOLDEN[f"surreal__crop_{kind}"][:, a]
        ok = crop_ok(crop, want, joints, rot, fl, extra)
        assert ok.all(), (a, np.abs(crop - want).max())
        assert np.abs(p2d - GOLDEN[f"surreal__pose2d_{kind}"][:, a]).max() <= 1e-5


def test_flip_orders_differ_only_by_rounding():
    """The two flip orders are different arithmetic: they agree to a float32 ulp, not bit for bit in general."""
    joints = GOLDEN["surreal__det"]
    C = joints.shape[0]
    _, after = smo.training_pose2d(joints, "smpl", rot=np.zeros(C), flip=np.ones(C), flip_before=False)
    _, before = smo.training_pose2d(joints, "smpl", rot=np.zeros(C), flip=np.ones(C), flip_before=True)
    assert np.abs(after - before).max() <= np.spacing(np.float32(288.0))


def test_smpl_flip_pairs_are_an_involution():
    perm = smo.flip_perm("smpl", 24)
    assert np.array_equal(perm[perm], np.arange(24))
    assert sorted({tuple(sorted((j, int(perm[j])))) for j in range(24) if perm[j] != j}) == list(smo.SMPL_FLIP_PAIRS)


def test_mano_crop_matches_reference():
    joints = GOLDEN["freihand__det"]
    p2d, crop = smo.training_pose2d(joints, "mano")
    assert crop_ok(crop, GOLDEN["freihand__crop"], joints, 0.0, 0).all()
    assert np.abs(p2d - GOLDEN["freihand__pose2d"]).max() <= 1e-5


def test_pw3d_crop_matches_reference():
    joints = GOLDEN["pw3d__det"]
    p2d, crop = smo.training_pose2d(joints, "coco")
    assert crop_ok(crop, GOLDEN["pw3d__crop"], joints, 0.0, 0).all()
    assert np.abs(p2d - GOLDEN["pw3d__pose2d"]).max() <= 1e-5


def surreal_img_tol(joints, f):
    """Half a float32 ulp of the reference's float32 x / z, times f, plus the float32 output's half ulp."""
    q = np.abs(joints[..., :2] / joints[..., 2:3])
    return 0.5 * np.spacing(q.astype(np.float32)) * f[:, None, :] + np.spacing(np.float32(1024.0))


def test_surreal_targets_match_reference():
    mesh, joints, f, c = (GOLDEN[f"surreal__{k}"] for k in ("mesh_in", "joints_in", "f", "c"))
    C = len(mesh)
    for a in range(len(GOLDEN["aug_cases"])):
        fl, rot = aug_case(a)
        o = smo.surreal_targets(mesh, joints, f, c, np.full(C, rot), np.full(C, fl))
        assert np.array_equal(o["mesh"].astype(np.float32), GOLDEN["surreal__mesh"])
        want = GOLDEN["surreal__lift"][:, a].astype(np.float64)
        tol = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        assert (np.abs(o["lift_pose3d"].astype(np.float32) - want) <= tol).all()
        assert np.array_equal(o["reg_pose3d"], o["lift_pose3d"])          # the same augmented array
        assert (np.abs(o["joint_img"] - GOLDEN["surreal__gt"]) <= surreal_img_tol(joints, f)).all()
        for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid", "joint_valid"):
            assert (o[k] == 1).all()
        assert (o["fitting_error"] == 0).all()


def test_freihand_targets_match_reference_bitwise():
    o = smo.freihand_targets(GOLDEN["freihand__mesh_in"], GOLDEN["freihand__joints_in"])
    assert np.array_equal(o["mesh"].astype(np.float32), GOLDEN["freihand__mesh"])
    assert np.array_equal(o["lift_pose3d"].astype(np.float32), GOLDEN["freihand__joints"])
    assert np.array_equal(o["reg_pose3d"], o["lift_pose3d"])
    assert "joint_img" not in o


def pw3d_mesh():
    return SAMPLES["fit__mesh"][GOLDEN["pw3d__mesh_index"]]


def pw3d_bounds(mesh, reg_h36m, reg_coco, out, f):
    """The reference's float32 regression error, worst case, for each 3DPW output (mesh on every row)."""
    mesh = np.asarray(mesh, np.float64)

    def rows_err(reg):
        A = np.abs(np.asarray(reg, np.float64))
        n = (A != 0).sum(1)
        return (n + 1)[None, :, None] * U * np.einsum("jv,bvc->bjc", A, np.abs(mesh))

    eh, ec = rows_err(reg_h36m), rows_err(reg_coco)
    ep = (ec[:, 11] + ec[:, 12]) * 0.5
    en = (ec[:, 5] + ec[:, 6]) * 0.5
    ec19 = np.concatenate([ec, ep[:, None], en[:, None]], 1)
    reg_b = eh + eh[:, :1] + U * np.abs(out["reg_pose3d"])
    lift_b = ec19 + ep[:, None] + U * np.abs(out["lift_pose3d"])
    mesh_b = (eh[:, :1] + U * np.abs(out["mesh"] * 1000)) / 1000 + U * np.abs(out["mesh"])
    # cam2pixel of the absolute COCO joints p: d(x / z) <= (|dx| + |x / z| |dz|) / |z|, the float32 quotient's rounding,
    # then times f
    absc = np.einsum("jv,bvc->bjc", np.asarray(reg_coco, np.float64), mesh)
    absc = np.concatenate([absc, ((absc[:, 11] + absc[:, 12]) * 0.5)[:, None], ((absc[:, 5] + absc[:, 6]) * 0.5)[:, None]],
                          1)
    q = absc[..., :2] / absc[..., 2:3]
    img_b = ((ec19[..., :2] + np.abs(q) * ec19[..., 2:3]) / np.abs(absc[..., 2:3]) + U * np.abs(q)) * f[:, None, :] + \
        U * np.abs(out["joint_img"])
    return {"reg_pose3d": reg_b, "lift_pose3d": lift_b, "mesh": mesh_b, "joint_img": img_b}


def test_pw3d_targets_match_reference_within_float32_regression():
    mesh, f, c = pw3d_mesh(), GOLDEN["pw3d__f"], GOLDEN["pw3d__c"]
    o = smo.pw3d_targets(mesh, TARGETS["reg_h36m"], TARGETS["reg_coco"], f, c)
    b = pw3d_bounds(mesh, TARGETS["reg_h36m"], TARGETS["reg_coco"], o, f)
    rows = GOLDEN["pw3d__rows"]
    for key, gkey, sl in (("reg_pose3d", "reg", slice(None)), ("lift_pose3d", "lift", slice(None)),
                          ("mesh", "mesh", rows), ("joint_img", "joint_img", slice(None))):
        err = np.abs(o[key][:, sl] - GOLDEN[f"pw3d__{gkey}"])
        assert (err <= b[key][:, sl]).all(), (key, err.max(), b[key][:, sl].min())
    for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid", "joint_valid"):
        assert (o[k] == 1).all()
