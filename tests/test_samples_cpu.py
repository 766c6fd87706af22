"""The training sample's augmentation rule (oracle/samples_oracle.py) against the unmodified reference
(tests/golden/samples.npz): the rotated and flipped crop in both noise orders and the augmented lift target to a
float32 ulp, and the augmentation parameters' distribution against the reference's augm_params counts."""
import os

import numpy as np
import pytest
from scipy import stats

from oracle import samples_oracle as so
from inputs_cases import P_FAIL, chi2_p
from oracle import inputs_oracle as io

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "samples.npz"))
SEED = (0x5EED_0001_2345_6789, 0x0000_00AB_CDEF_0123)
SETS = ("coco", "human36")


def within_ulp(got, want, ulps=1, flipped=False, width=288):
    """|got - want| within `ulps` float32 ulps; for flipped x the ulp of the pre-flip value width - 1 - x counts too,
    since the flip subtracts it from the width in float32."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    mag = np.maximum(np.abs(got), np.abs(want))
    if flipped:
        mag[..., 0] = np.maximum(mag[..., 0], np.abs(width - 1 - want[..., 0]))
    tol = ulps * np.spacing(mag.astype(np.float32)).astype(np.float64)
    return np.abs(got - want) <= tol


def aug_case(a):
    fl, rot = GOLDEN["aug_cases"][a]
    return int(fl), np.float32(rot)


@pytest.mark.parametrize("joint_set", SETS)
@pytest.mark.parametrize("flip_before_noise", [False, True])
def test_oracle_crop_matches_reference(joint_set, flip_before_noise):
    joints = GOLDEN[f"{joint_set}__joints"]
    want = GOLDEN[f"{joint_set}__crop_{'before' if flip_before_noise else 'after'}"]
    C = joints.shape[0]
    m = io.crop_map(joints)
    for a in range(want.shape[1]):
        fl, rot = aug_case(a)
        _, crop = so.training_pose2d(joints, "none", joint_set, rot=np.full(C, rot), flip=np.full(C, fl),
                                     flip_before_noise=flip_before_noise)
        ok = within_ulp(crop, want[:, a], flipped=bool(fl))
        if rot == 0:
            # rot = 0 keeps the library's closed form (one scale from the box height), while the reference's x scale
            # comes from a third point rounded to float32: a relative scale difference of up to one float32 ulp of
            # that point's x (about |centre| + w) over the half-width w / 2, times the distance from the crop's centre
            rel = np.spacing(np.abs(m["ccx"]).astype(np.float32) + m["crop_w"].astype(np.float32)) / (m["crop_w"] / 2)
            ok |= np.abs(crop - want[:, a]) <= rel[:, None, None] * np.abs(want[:, a] - [144.0, 192.0]) + 1e-5
        assert ok.all(), (a, np.argwhere(~ok)[:4], crop[~ok][:4], want[:, a][~ok][:4])


@pytest.mark.parametrize("joint_set", SETS)
def test_oracle_lift_matches_reference(joint_set):
    lift = GOLDEN[f"{joint_set}__lift"]
    want = GOLDEN[f"{joint_set}__lift_aug"]
    C = lift.shape[0]
    for a in range(want.shape[1]):
        fl, rot = aug_case(a)
        got = so.j3d_processing(lift, np.full(C, rot), np.full(C, fl), joint_set).astype(np.float32)
        ok = within_ulp(got, want[:, a])
        assert ok.all(), (a, np.argwhere(~ok)[:4])


def test_unaugmented_crop_is_inputs_oracle():
    joints = GOLDEN["coco__joints"]
    m = io.crop_map(joints)
    C = joints.shape[0]
    want = io.crop_points(m, joints)
    got = so.crop_points(m, joints, np.zeros(C, np.float32)).astype(np.float32)
    np.testing.assert_array_equal(got, want)
    _, crop = so.training_pose2d(joints, "none", "coco", rot=np.zeros(C), flip=np.zeros(C))
    np.testing.assert_array_equal(crop, want)


def test_flip_perm_is_an_involution():
    for s, J in (("coco", 19), ("human36", 17)):
        p = so.flip_perm(s, J)
        np.testing.assert_array_equal(p[p], np.arange(J))
    assert list(so.flip_perm("coco", 19)[17:]) == [17, 18]


@pytest.mark.parametrize("k", range(4))
def test_oracle_augm_params_match_reference_counts(k):
    fl, rf = GOLDEN["augm_settings"][k]
    M, nb = int(GOLDEN["augm_M"]), int(GOLDEN["augm_bins"])
    f, r = so.augm_params(M, bool(fl), rf, SEED)
    ref_flip, ref_zero = int(GOLDEN["augm_flips"][k]), int(GOLDEN["augm_zero"][k])
    ps = [chi2_p(np.array([ref_flip, M - ref_flip]), np.array([f.sum(), M - f.sum()])),
          chi2_p(np.array([ref_zero, M - ref_zero]), np.array([(r == 0).sum(), M - (r == 0).sum()]))]
    if not fl:
        assert f.sum() == 0
    if rf == 0:
        assert (r == 0).all()
    else:
        nz = r[r != 0].astype(np.float64)
        hist = np.histogram(nz, bins=nb, range=(-2 * rf, 2 * rf))[0]
        ps.append(chi2_p(GOLDEN["augm_hist"][k], hist))
        ref_clip = int(GOLDEN["augm_clip"][k])
        clip = int((np.abs(nz) == np.float32(2 * rf)).sum())
        ps.append(chi2_p(np.array([ref_clip, M - ref_clip]), np.array([clip, M - clip])))
        # the nonzero rotations are the clipped normal: KS against its CDF inside the clip
        inside = nz[np.abs(nz) < 2 * rf] / rf
        cdf = lambda x: (stats.norm.cdf(x) - stats.norm.cdf(-2)) / (stats.norm.cdf(2) - stats.norm.cdf(-2))  # noqa: E731
        ps.append(stats.kstest(inside, cdf).pvalue)
    assert min(ps) > P_FAIL, ps


def test_augm_params_streams_are_per_sample():
    f, r = so.augm_params(64, True, 30.0, SEED)
    f2, r2 = so.augm_params(8, True, 30.0, SEED, sample_index=np.arange(40, 48))
    np.testing.assert_array_equal(f[40:48], f2)
    np.testing.assert_array_equal(r[40:48], r2)


TGOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "targets.npz"))


def test_oracle_muco_fitting_quirk_matches_reference():
    m = GOLDEN["fit__mesh"]
    B = m.shape[0]
    got = so.sample_targets("muco", m, TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"], f=np.full((B, 2), 1000.0),
                            c=np.full((B, 2), 500.0))
    np.testing.assert_allclose(got["fitting_error"], GOLDEN["muco_fit__error"], rtol=1e-6)
    assert (got["fitting_error"] > 300).all() and (got["mesh_valid"] == 0).all()   # the quirk rejects every sample


def test_oracle_coco_fitting_matches_reference():
    m, mi = GOLDEN["fit__mesh"], GOLDEN["coco_fit__mesh_index"]
    want = GOLDEN["coco_fit__error"]
    assert (want[:3] < 3).sum() == 2 and want[1] > 3 and np.isnan(want[3])          # both sides of 3 px, none visible
    for k in range(len(want)):
        got = so.sample_targets("coco", m[mi[k]][None], TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"],
                                "coco" if GOLDEN["coco_fit__set"][k] else "human36", s=GOLDEN["coco_fit__s"][k:k + 1],
                                t=GOLDEN["coco_fit__t"][k:k + 1], keypoints=GOLDEN["coco_fit__kps"][k:k + 1],
                                keypoints_valid=GOLDEN["coco_fit__valid"][k:k + 1])
        np.testing.assert_allclose(got["fitting_error"], want[k:k + 1], rtol=1e-4, atol=1e-5)
        assert got["mesh_valid"][0, 0, 0] == (0.0 if want[k] > 3 else 1.0)             # NaN keeps the sample
