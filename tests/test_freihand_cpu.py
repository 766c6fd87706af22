"""The FreiHAND oracle (oracle/freihand_oracle.py) and the evaluation regressor on the CPU: brute-force distances
against a KD-tree, align_w_scale on exact similarities (reflections included), the F-score's symmetry, and
mano_eval_regressor against the regressor the unmodified lib/_mano.py builds (tests/golden/freihand_regressor.npz)."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import body_models as bm
from helpers import load_npz
from oracle import freihand_oracle as fo
from oracle import metrics_oracle as mo
from pose2mesh_release_b200 import freihand


def random_rotation(rng):
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


@pytest.mark.parametrize("n,m", [(1, 1), (31, 2), (778, 778), (1000, 331)])
def test_brute_force_distances_equal_kdtree(n, m):
    rng = np.random.default_rng(n + 7 * m)
    P = rng.normal(0, 0.05, (n, 3)).astype(np.float32)
    Q = rng.normal(0, 0.05, (m, 3)).astype(np.float32)
    Q[: m // 3] = P[: m // 3]  # some exact duplicates: distance 0
    d_p, d_q = fo.nearest(P, Q, chunk=97)
    assert np.array_equal(d_p, cKDTree(Q.astype(np.float64)).query(P.astype(np.float64))[0])
    assert np.array_equal(d_q, cKDTree(P.astype(np.float64)).query(Q.astype(np.float64))[0])


def test_nearest_isolates_non_finite_samples():
    P = np.zeros((4, 3))
    P[1, 2] = np.nan
    d_p, d_q = fo.nearest(P, np.ones((3, 3)))
    assert np.isnan(d_p).all() and np.isnan(d_q).all()
    f, a, b = fo.fscore(P, np.ones((3, 3)), 0.01)
    assert np.isnan(f) and np.isnan(a) and np.isnan(b)


@pytest.mark.parametrize("reflect", [False, True])
def test_align_w_scale_recovers_similar_copies(reflect):
    rng = np.random.default_rng(3 + reflect)
    gt = rng.normal(0, 0.05, (778, 3)) + [0.1, -0.2, 0.6]
    R = random_rotation(rng)
    if reflect:
        R = R @ np.diag([1.0, 1.0, -1.0])
    pred = 1.7 * gt @ R.T + [0.3, 0.1, -0.4]
    aligned = fo.align_w_scale(gt, pred)
    # the script's + 1e-8 on both norms scales the recovered copy about the centroid by exactly (|P| / (|P| + 1e-8))^2
    t1, nP = gt.mean(0), np.linalg.norm(pred - pred.mean(0))
    expect = t1 + (gt - t1) * (nP / (nP + 1e-8)) ** 2
    assert np.abs(aligned - expect).max() <= 1e-12 * np.abs(gt).max()
    assert np.abs(aligned - gt).max() <= 1e-8 * np.abs(gt).max()
    if reflect:  # Pose2Mesh's rigid_align forces det R = +1 and cannot undo a mirror image
        assert np.abs(mo.rigid_align(pred, gt) - gt).max() > 1e-3


def test_fscore_is_symmetric_and_strict():
    rng = np.random.default_rng(11)
    gt = rng.normal(0, 0.02, (300, 3))
    pred = gt[:200] + rng.normal(0, 0.004, (200, 3))
    for th in (0.001, 0.005, 0.015):
        f1, a1, b1 = fo.fscore(gt, pred, th)
        f2, a2, b2 = fo.fscore(pred, gt, th)
        assert f1 == f2 and (a1, b1) == (b2, a2)
    # a point exactly at the threshold does not count
    f, a, b = fo.fscore(np.zeros((1, 3)), np.array([[0.0, 0.0, 0.015625]]), 0.015625)
    assert (f, a, b) == (0.0, 0.0, 0.0)
    f, a, b = fo.fscore(np.zeros((1, 3)), np.array([[0.0, 0.0, 0.015625]]), np.nextafter(0.015625, 1))
    assert (f, a, b) == (1.0, 1.0, 1.0)


def test_mano_eval_regressor_matches_reference():
    z = load_npz("freihand_regressor.npz")
    assert str(z["model_digest"]) == bm.digest(bm.mano_model("right"))
    J = freihand.mano_eval_regressor(z["J_regressor"]).numpy()
    assert J.dtype == np.float32 and np.array_equal(J, z["joint_regressor"])
    assert np.flatnonzero(J[12]).tolist() == [445] and J[12, 445] == 1.0
    assert [int(np.flatnonzero(J[k])[0]) for k in (4, 8, 12, 16, 20)] == [745, 317, 445, 556, 673]


def test_mano_eval_regressor_rejects_wrong_shape():
    with pytest.raises(ValueError):
        freihand.mano_eval_regressor(np.zeros((21, 778), np.float32))


def test_evaluator_rejects_bad_thresholds_before_any_launch():
    for bad in ((0.015, 0.005), (-0.001, 0.005), (np.nan,), ()):
        with pytest.raises(ValueError):
            freihand._thresholds(bad, 16)
