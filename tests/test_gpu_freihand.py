"""The FreiHAND scores on the GPU (SURVEY.md §8 row f9, pose2mesh_release_b200.freihand) against the float64 restatement
of the FreiHAND evaluation script (oracle/freihand_oracle.py): nearest distances, counts and F-scores bit for bit,
align_w_scale within 1e-9 of max |gt|, and the evaluator over a FreiHAND-sized set."""
import numpy as np
import pytest
import torch

import body_models as bm
from oracle import freihand_oracle as fo
from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200 import freihand as F
from pose2mesh_release_b200.body_model import ManoLayer
from pose2mesh_release_b200.postprocess import regress_joints

pytestmark = pytest.mark.gpu
TH = (0.005, 0.015)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def host(t):
    return t.cpu().numpy()


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def cloud(rng, B, n, scale=0.05):
    return (rng.normal(0, scale, (B, n, 3)) + rng.normal(0, 0.2, (B, 1, 3))).astype(np.float32)


def check_nearest(P, Q, samples=None):
    dp, dq = F.nearest_distances(cuda(P), cuda(Q))
    fs, fa, fb = F.f_scores(cuda(P), cuda(Q), TH)
    _, _, cnt, _, _ = F._nearest(cuda(P), cuda(Q), F._thresholds(TH, 16)[0], 2, dist=False, counts=True)
    dp, dq, fs, fa, fb, cnt = map(host, (dp, dq, fs, fa, fb, cnt))
    for b in (range(len(P)) if samples is None else samples):
        op, oq = fo.nearest(P[b], Q[b])
        assert same(dp[b], op) and same(dq[b], oq), b
        for j, th in enumerate(TH):
            f, a, bb = fo.fscore_from_distances(op, oq, th)
            assert same(np.array([fs[b, j], fa[b, j], fb[b, j]]), np.array([f, a, bb])), (b, j)
            assert cnt[b, 0, j] == np.sum(op < th) and cnt[b, 1, j] == np.sum(oq < th), (b, j)


@pytest.mark.parametrize("n,m", [(1, 1), (2, 31), (31, 2), (778, 778), (1000, 778), (778, 6890), (6890, 1000)])
@pytest.mark.parametrize("B", [1, 7])
def test_nearest_distances_bitwise(n, m, B):
    rng = np.random.default_rng(n * 13 + m + B)
    P, Q = cloud(rng, B, n), cloud(rng, B, m, 0.02)
    Q[:, : min(n, m) // 2] = P[:, : min(n, m) // 2]  # duplicates across the sets
    check_nearest(P, Q)


def test_nearest_distances_smpl_size_b256_subset():
    rng = np.random.default_rng(256)
    P, Q = cloud(rng, 256, 6890, 0.3), cloud(rng, 256, 6890, 0.3)
    check_nearest(P, Q, samples=(0, 1, 127, 200, 255))


def test_identical_sets_duplicates_and_points_at_the_threshold():
    rng = np.random.default_rng(5)
    P = cloud(rng, 3, 778)
    Q = P.copy()
    Q[1] = np.repeat(P[1, :10], 78, axis=0)[:778]  # many duplicate points
    # sample 2: exact power-of-two offsets of 2^-6 = 0.015625 and 2^-8 = 0.00390625 from grid points
    g = (np.arange(778 * 3).reshape(778, 3) % 7).astype(np.float32) * 0.25
    P[2], Q[2] = g, g + np.array([0, 0, 0.015625], np.float32)
    Q[2, ::2] = g[::2] + np.array([0.00390625, 0, 0], np.float32)
    check_nearest(P, Q)
    ths = (0.00390625, 0.015625)
    fs, fa, fb = (host(x) for x in F.f_scores(cuda(P[2]), cuda(Q[2]), ths))
    # every gt point is exactly 2^-8 from a prediction; half the predictions 2^-8, half 2^-6: the strict `<`
    # excludes every point exactly at t
    assert fa[0] == fb[0] == 0 and fa[1] == 1 and fb[1] == 0.5
    assert np.array_equal(fs, [fo.fscore(P[2], Q[2], t)[0] for t in ths])
    dp, dq = F.nearest_distances(cuda(P[0]), cuda(Q[0]))
    assert (host(dp) == 0).all() and (host(dq) == 0).all()


def test_nan_sample_is_isolated():
    rng = np.random.default_rng(9)
    P, Q = cloud(rng, 5, 778), cloud(rng, 5, 778)
    ref = [host(t) for t in F.f_scores(cuda(P), cuda(Q))]
    P[2, 100, 1] = np.nan
    Q[3, 5, 0] = np.inf
    got = [host(t) for t in F.f_scores(cuda(P), cuda(Q))]
    for g, r in zip(got, ref):
        assert np.isnan(g[2:4]).all()
        assert same(g[[0, 1, 4]], r[[0, 1, 4]])
    dp, dq = (host(t) for t in F.nearest_distances(cuda(P), cuda(Q)))
    assert np.isnan(dp[2]).all() and np.isnan(dq[3]).all() and not np.isnan(dp[[0, 1, 4]]).any()


def test_float64_inputs_and_split_invariance():
    rng = np.random.default_rng(17)
    P, Q = rng.normal(0, 0.05, (7, 1000, 3)), rng.normal(0, 0.05, (7, 700, 3))
    dp, dq = (host(t) for t in F.nearest_distances(cuda(P), cuda(Q)))
    for b in range(7):
        op, oq = fo.nearest(P[b], Q[b])
        assert same(dp[b], op) and same(dq[b], oq)
    one = host(F.nearest_distances(cuda(P[3]), cuda(Q[3]))[0])  # B=1 splits each sample over many CTAs
    assert same(one, dp[3])


def _similar(rng, X, reflect):
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    R = q * np.sign(np.diag(r))
    if (np.linalg.det(R) < 0) != reflect:
        R[:, 2] = -R[:, 2]
    return (rng.uniform(0.5, 2.0) * X @ R.T + rng.normal(0, 0.1, 3)).astype(np.float32)


def test_align_w_scale_matches_oracle():
    rng = np.random.default_rng(21)
    gt = cloud(rng, 12, 778)
    pred = np.stack([_similar(rng, gt[b] + rng.normal(0, 0.003, (778, 3)), reflect=b % 2 == 1) for b in range(12)])
    pred[10] = np.linspace(0, 1, 778)[:, None] * np.array([1, 2, 3], np.float32)  # collinear: rank-1 A^T P
    pred[11] = pred[11, :1]  # all points equal: P = 0
    got, Y, E = host(F.align_w_scale(cuda(gt), cuda(pred))), *F._align(cuda(gt), cuda(pred), torch.float64, err=True)
    Y, E = host(Y), host(E)
    for b in range(12):
        o = fo.align_w_scale(gt[b], pred[b])
        tol = 1e-9 * np.abs(gt[b]).max()
        res_o = fo.point_dist(o, gt[b])
        assert np.abs(E[b] - res_o).max() <= tol, b
        if b < 10:  # unique R: the points themselves
            assert np.abs(Y[b] - o).max() <= tol, b
            assert np.abs(got[b] - o.astype(np.float32)).max() <= 2 ** -22 * np.abs(o).max() + tol, b
        else:  # rank-deficient: R is not unique, the residual is
            assert abs(np.sum(E[b] ** 2) - np.sum(res_o ** 2)) <= 1e-9 * np.sum(res_o ** 2), b
    assert E[1].mean() < 0.007  # a mirror image is aligned (det R = -1 kept) down to its 3 mm noise


def test_align_w_scale_nan_isolated():
    rng = np.random.default_rng(2)
    gt, pred = cloud(rng, 3, 21), cloud(rng, 3, 21)
    pred[1, 4, 0] = np.nan
    Y = host(F.align_w_scale(cuda(gt), cuda(pred)))
    assert np.isnan(Y[1]).all() and not np.isnan(Y[[0, 2]]).any()


# ------------------------------------------------------------------------------------------------ evaluator
N_EVAL = 3960


def _freihand_set():
    """Seeded MANO hands of the repository's ManoLayer (metres) and perturbed predictions: noise on every sample,
    a random similarity on every third, a mirrored similarity on every seventh."""
    m = bm.mano_model("right")
    layer = ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                      m["hands_mean"], flat_hand_mean=False, side="right")
    rng = np.random.default_rng(3960)
    pose = torch.from_numpy(rng.normal(0, 0.6, (N_EVAL, 48)).astype(np.float32)).cuda()
    betas = torch.from_numpy(rng.normal(0, 1.0, (N_EVAL, 10)).astype(np.float32)).cuda()
    trans = torch.from_numpy(rng.normal(0, 0.1, (N_EVAL, 3)).astype(np.float32)).cuda()
    with torch.no_grad():
        verts, joints = layer(pose, betas, trans)
    gt_v, gt_x = host(verts) / 1000, host(joints) / 1000
    pred_v = gt_v + rng.normal(0, 0.004, gt_v.shape)
    for i in range(N_EVAL):
        if i % 3 == 0 or i % 7 == 0:
            pred_v[i] = _similar(rng, pred_v[i], reflect=i % 7 == 0)
    pred_v = pred_v.astype(np.float32)
    reg = F.mano_eval_regressor(m["J_regressor"]).cuda()
    pred_x = host(regress_joints(cuda(pred_v), reg))
    return gt_x.astype(np.float32), gt_v.astype(np.float32), pred_x, pred_v


@pytest.fixture(scope="module")
def freihand_set():
    data = _freihand_set()
    return data, fo.evaluate(*data, thresholds=TH)


def _run(data, splits):
    gx, gv, px, pv = (cuda(a) for a in data)
    ev = F.FreiHANDEvaluator(TH)
    for a, b in zip(splits[:-1], splits[1:]):
        ev.update(px[a:b], pv[a:b], gx[a:b], gv[a:b])
    return ev.compute()


def test_evaluator_matches_script_loop(freihand_set):
    data, ref = freihand_set
    got = _run(data, [0, 1000, 2000, 3000, N_EVAL])
    assert got["n_samples"] == N_EVAL
    for k in F.FreiHANDEvaluator.KINDS:
        assert np.array_equal(got[f"{k}_counts"], ref[f"{k}_counts"]), k
        for key in (f"{k}_mean3d", f"{k}_auc3d"):
            assert abs(got[key] - ref[key]) <= 1e-12 * abs(ref[key]), key
        assert np.abs(got[f"{k}_pck"] - ref[f"{k}_pck"]).max() <= 1e-12
    for key in ("f_score", "f_score_aligned"):
        assert np.abs(got[key] - ref[key]).max() <= 1e-12 * np.abs(ref[key]).max(), key
    assert 0.0 < ref["f_score"][0] < ref["f_score_aligned"][0] < 1.0  # alignment matters on these predictions


def test_evaluator_batch_split_invariant_and_deterministic(freihand_set):
    data, _ = freihand_set
    a = _run(data, [0, 1000, 2000, 3000, N_EVAL])
    b = _run(data, [0, 1, 8, 777, 1500, 3959, N_EVAL])
    c = _run(data, [0, 1000, 2000, 3000, N_EVAL])
    for k, v in a.items():
        assert np.array_equal(np.asarray(v), np.asarray(b[k])), k
        assert np.array_equal(np.asarray(v), np.asarray(c[k])), k


def test_evaluator_update_is_sync_free_with_fixed_launches(freihand_set):
    (gx, gv, px, pv), _ = freihand_set
    gx, gv, px, pv = (cuda(a[:64]) for a in (gx, gv, px, pv))
    ev = F.FreiHANDEvaluator(TH)
    ev.update(px, pv, gx, gv)
    counts = []
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for B in (64, 5):
            _lib.load().p2m_launch_count_reset()
            ev.update(px[:B], pv[:B], gx[:B], gv[:B])
            counts.append(_lib.load().p2m_launch_count())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert counts == [12, 12]
    assert ev.compute()["n_samples"] == 133


def test_argument_errors():
    P = torch.zeros((2, 10, 3), device="cuda")
    with pytest.raises(RuntimeError):
        F.nearest_distances(P.cpu(), P.cpu())
    with pytest.raises(ValueError):
        F.nearest_distances(P, torch.zeros((3, 10, 3), device="cuda"))
    with pytest.raises(ValueError):
        F.nearest_distances(P, torch.zeros((2, 10, 2), device="cuda"))
    with pytest.raises(ValueError):
        F.nearest_distances(P, P.double())
    with pytest.raises(ValueError):
        F.f_scores(P, P, (0.015, 0.005))
    with pytest.raises(ValueError):
        F.f_scores(P, P, (-0.001,))
    with pytest.raises(ValueError):
        F.align_w_scale(P, torch.zeros((2, 11, 3), device="cuda"))
    with pytest.raises(ValueError):
        F.FreiHANDEvaluator((0.01, 0.005))
    with pytest.raises(ValueError):
        F.FreiHANDEvaluator(pck=(0.05, 0.0, 100))
    ev = F.FreiHANDEvaluator()
    with pytest.raises(ValueError):
        ev.update(P, P, P[:, :5], P)
    with pytest.raises(ValueError):
        ev.compute()
    # the C ABI checks again on the host, before any launch
    bad = (F.C.c_double * 2)(0.015, 0.005)
    with torch.cuda.device(0):
        st = _lib.load().p2m_nearest_distances(0, P.data_ptr(), P.data_ptr(), 2, 10, 10, bad, 2, None, None, None,
                                               None, torch.empty((2, 2), device="cuda", dtype=torch.float64).data_ptr(),
                                               None)
    assert st != 0 and b"sorted" in _lib.load().p2m_last_error()
