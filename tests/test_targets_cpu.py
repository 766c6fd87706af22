"""oracle/targets_oracle.py against the unmodified reference's outputs in tests/golden/targets.npz (CPU only).

The reference runs its layers in float32, so the bounds are float32 ones: the body-model fixture's 5e-6 of each
sample's largest |coordinate| plus a few float32 roundings of the translation terms (1e-5 in all); the Human3.6M
assembly's fp64 steps add nothing beyond the mesh's own error.
"""
import os

import numpy as np
import pytest

import body_model_oracle as bo
import body_models as bm
from oracle import targets_oracle as to

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "targets.npz"))
SMPL, MANO = bm.smpl_model(), bm.mano_model("right", False)
PRESETS = ("human36m", "amass", "freihand", "muco", "coco", "surreal", "pw3d")
REL = 1e-5


def preset_inputs(p):
    return [GOLDEN[f"{p}__{k}"] for k in ("pose", "betas", "trans", "R", "t")]


def oracle_frame(p, pose, betas, trans, R, t):
    mano = p == "freihand"
    model = MANO if mano else SMPL
    fwd = (lambda q, b, tr: bo.mano_forward(model, q, b, tr)) if mano else \
        (lambda q, b, tr: bo.smpl_forward(model, q, b, tr))
    return to.camera_frame(fwd, model["betas"], p, pose, betas, trans, R, t, mano=mano)


def close(got, want, scale):
    err = np.abs(np.asarray(got, np.float64) - want).max()
    assert err <= REL * scale, (err, REL * scale)


def test_fixture_models():
    assert str(GOLDEN["digest_smpl"]) == bm.digest(SMPL)
    assert str(GOLDEN["digest_mano"]) == bm.digest(MANO)


@pytest.mark.parametrize("preset", PRESETS)
def test_camera_frame_matches_reference(preset):
    mesh, joints = oracle_frame(preset, *preset_inputs(preset))
    rows = slice(None) if preset == "freihand" else GOLDEN["rows"]
    for b in range(mesh.shape[0]):
        scale = max(np.abs(mesh[b]).max(), np.abs(joints[b]).max())
        close(GOLDEN[f"{preset}__mesh"][b], mesh[b, rows], scale)
        close(GOLDEN[f"{preset}__joints"][b], joints[b], scale)


def test_betas_rules_are_per_sample():
    b = np.array([[0.5] * 10, [0.0] * 10, [4.0] + [0.1] * 9], np.float32)
    r = to.resolve_betas(b, SMPL["betas"], clamp=True, zero_means_model=True)
    assert np.array_equal(r[0], b[0].astype(np.float64))
    assert np.array_equal(r[1], SMPL["betas"].astype(np.float64))
    assert np.array_equal(r[2], SMPL["betas"].astype(np.float64))  # clamped to zero, then the model's betas
    r = to.resolve_betas(b, MANO["betas"], clamp=False, zero_means_model=False)
    assert np.array_equal(r, b.astype(np.float64))


@pytest.mark.parametrize("joint_set", ["human36", "coco"])
def test_h36m_targets_match_reference(joint_set):
    pose, betas, trans, R, t = preset_inputs("human36m")
    mesh_cam, _ = oracle_frame("human36m", pose, betas, trans, R, t)
    out = to.h36m_targets(mesh_cam, GOLDEN["h36m__joint_cam"], GOLDEN["h36m__f"], GOLDEN["h36m__c"],
                          GOLDEN["reg_h36m"], GOLDEN["reg_coco"], joint_set)
    rows = GOLDEN["rows"]
    for b in range(pose.shape[0]):
        scale = np.abs(mesh_cam[b]).max()
        close(GOLDEN[f"h36m_{joint_set}__mesh"][b], out["mesh"][b, rows], scale / 1000)
        close(GOLDEN[f"h36m_{joint_set}__lift_pose3d"][b], out["lift_pose3d"][b], scale)
        close(GOLDEN[f"h36m_{joint_set}__reg_pose3d"][b], out["reg_pose3d"][b], scale)
        # pixels: a relative error e of the camera-frame point moves the projection by about 2 e f
        close(GOLDEN[f"h36m_{joint_set}__joint_img"][b], out["joint_img"][b], 2 * 1200 + scale)
        assert abs(GOLDEN[f"h36m_{joint_set}__fitting_error"][b] - out["fitting_error"][b]) <= REL * scale
    assert np.array_equal(GOLDEN[f"h36m_{joint_set}__mesh_valid"], out["mesh_valid"][:, rows])
    assert np.array_equal(GOLDEN[f"h36m_{joint_set}__lift_pose3d_valid"], out["lift_pose3d_valid"])
    # the fixture has samples on both sides of the 25 mm threshold, each well away from it
    err = GOLDEN[f"h36m_{joint_set}__fitting_error"]
    assert (err < 20).any() and (err > 30).any() and not ((err > 20) & (err < 30)).any()
