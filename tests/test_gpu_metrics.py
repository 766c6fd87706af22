"""The evaluation metrics on the GPU (pose2mesh_release_b200/metrics.py; run on an H100 with -m gpu) against the
reference's golden values (tests/golden/eval_metrics.npz) and the float64 oracle (oracle/metrics_oracle.py).

Tolerances: compute_*_err means 1e-6 relative (the reference's are float32); per-point errors of point_errors bit for
bit; Procrustes c, R, t 1e-9 relative where the singular-value gaps exceed 1e-6 s1 (elsewhere R is ill-determined),
aligned points and their errors 2^-22 max|B| (float32 output rounding); evaluate_meshes 1e-6 of the sample's largest
coordinate (fp32 accumulation of the joint regression)."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from helpers import load_npz
from oracle import metrics_oracle as mo

pytestmark = pytest.mark.gpu

Z = load_npz("eval_metrics.npz")
NAMES = [str(s) for s in Z["rt_names"]]
H36M_EVAL = (1, 2, 3, 4, 5, 6, 8, 10, 11, 12, 13, 14, 15, 16)


def dev():
    return torch.device("cuda:0")


def cu(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float32)).to(dev())


def _gaps_ok(A, B):
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    s = np.linalg.svd((A - A.mean(0)).T @ (B - B.mean(0)) / len(A), compute_uv=False)
    return s[0] > 0 and s[0] - s[1] > 1e-6 * s[0] and s[1] - s[2] > 1e-6 * s[0]


def _check_sample(A, B, c, R, t, Y, E, label):
    """One sample of the GPU Procrustes (c, R, t, aligned Y, errors E) against the oracle."""
    A64, B64 = np.asarray(A, np.float64), np.asarray(B, np.float64)
    c0, R0, t0 = mo.rigid_transform_3D(A64, B64)
    Y0 = mo.rigid_align(A64, B64)
    E0 = np.sqrt(((Y0 - B64) ** 2).sum(1))
    if np.isnan(c0):
        assert np.isnan(c) and np.isnan(t).all() and np.isnan(Y).all() and np.isnan(E).all(), label
        return
    tol_pts = 2.0 ** -22 * max(np.abs(B64).max(), 1e-30)
    assert np.abs(Y - Y0).max() <= tol_pts, (label, np.abs(Y - Y0).max(), tol_pts)
    assert np.abs(E - E0).max() <= tol_pts, (label, np.abs(E - E0).max(), tol_pts)
    assert abs(np.linalg.det(R) - 1.0) < 1e-12, label
    assert abs(c - c0) <= 1e-9 * abs(c0), (label, c, c0)
    if _gaps_ok(A64, B64):
        assert np.abs(R - R0).max() <= 1e-9, (label, np.abs(R - R0).max())
        scale = max(np.abs(t0).max(), np.abs(B64).max())
        assert np.abs(t - t0).max() <= 1e-9 * scale, (label, np.abs(t - t0).max(), scale)


def _run_align(A, B, subset=None):
    """(transform [B, 13] f64, aligned, err, sums [B + 1]) through the metrics module's single library call."""
    from pose2mesh_release_b200 import metrics

    A, B = cu(A), cu(B)
    sums = torch.empty(A.shape[0] + 1, device=dev(), dtype=torch.float64)
    T, Y, E = metrics._align(A, B, subset, transform=True, aligned=True, err=True, sums=sums)
    return T.cpu().numpy(), Y.cpu().numpy(), E.cpu().numpy(), sums.cpu().numpy()


# ------------------------------------------------------------------------------------------------ against the golden
@pytest.mark.parametrize("tag", ["h36m", "pw3d", "surreal"])
def test_compute_err_against_reference(tag):
    from pose2mesh_release_b200 import metrics

    sub = lambda key: (Z[key].tolist() or None)  # noqa: E731
    pj, gj = cu(Z[f"{tag}_pred_joint"]), cu(Z[f"{tag}_gt_joint"])
    pm, gm = cu(Z[f"{tag}_pred_mesh"]), cu(Z[f"{tag}_gt_mesh"])
    root = int(Z[f"{tag}_joint_root"])
    je = metrics.compute_joint_err(pj, gj, root=root, eval_joint=sub(f"{tag}_joint_subset"))
    assert isinstance(je, float) and abs(je - Z[f"{tag}_joint_err"]) <= 1e-6 * Z[f"{tag}_joint_err"]
    bj, bm = metrics.compute_both_err(pm, gm, pj, gj, eval_joint=sub(f"{tag}_both_subset"))
    assert abs(bj - Z[f"{tag}_both_joint_err"]) <= 1e-6 * Z[f"{tag}_both_joint_err"]
    assert abs(bm - Z[f"{tag}_both_mesh_err"]) <= 1e-6 * Z[f"{tag}_both_mesh_err"]
    # per-point values: the reference's float32 bits
    pp = metrics.point_errors(pj, gj, root=root, subset=sub(f"{tag}_joint_subset")).cpu().numpy()
    assert np.array_equal(pp.view(np.uint32), Z[f"{tag}_joint_pp"].view(np.uint32))
    pp = metrics.point_errors(pj, gj, root=0, subset=sub(f"{tag}_both_subset")).cpu().numpy()
    assert np.array_equal(pp.view(np.uint32), Z[f"{tag}_both_joint_pp"].view(np.uint32))
    pp = metrics.point_errors(pm, gm, pred_root=pj[:, 0], gt_root=gj[:, 0]).cpu().numpy()
    assert np.array_equal(pp.view(np.uint32), Z[f"{tag}_mesh_pp"].view(np.uint32))


@pytest.mark.parametrize("i", range(len(NAMES)), ids=NAMES)
def test_procrustes_against_reference_cases(i):
    from pose2mesh_release_b200 import metrics

    A, B = Z[f"rt{i}_A"], Z[f"rt{i}_B"]
    T, Y, E, _ = _run_align(A[None], B[None])
    c, R, t = T[0, 0], T[0, 1:10].reshape(3, 3), T[0, 10:]
    _check_sample(A, B, c, R, t, Y[0], E[0], NAMES[i])
    if NAMES[i] == "all_equal":
        return
    # the golden values of the unmodified reference: c always, aligned rows always, R / t where R is determined
    assert abs(c - Z[f"rt{i}_c"]) <= 1e-9 * abs(Z[f"rt{i}_c"])
    rows = Z[f"rt{i}_rows"]
    assert np.abs(Y[0][rows] - Z[f"rt{i}_aligned"]).max() <= 2.0 ** -22 * np.abs(B).max()
    if _gaps_ok(A, B):
        assert np.abs(R - Z[f"rt{i}_R"]).max() <= 1e-9
    # the public wrappers agree with the single call
    c2, R2, t2 = metrics.rigid_transform(cu(A), cu(B))
    assert c2.shape == () and R2.shape == (3, 3) and t2.shape == (3,)
    assert np.array_equal(R2.cpu().numpy(), R) and np.array_equal(t2.cpu().numpy(), t)
    assert np.array_equal(metrics.rigid_align(cu(A), cu(B)).cpu().numpy(), Y[0])


def test_mirrored_target_gets_the_reference_flipped_answer():
    i = NAMES.index("mirrored")
    A, B = Z[f"rt{i}_A"], Z[f"rt{i}_B"]
    T, _, _, _ = _run_align(A[None], B[None])
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    H = (A64 - A64.mean(0)).T @ (B64 - B64.mean(0)) / len(A)
    s = np.linalg.svd(H, compute_uv=False)
    var_p = np.var(A64, axis=0).sum()
    assert abs(T[0, 0] - (s[0] + s[1] - s[2]) / var_p) <= 1e-9 * T[0, 0]  # s[-1] negated
    assert abs(T[0, 0] - Z[f"rt{i}_c"]) <= 1e-9 * T[0, 0]
    assert np.abs(T[0, 1:10] - Z[f"rt{i}_R"].reshape(-1)).max() <= 1e-9


# ------------------------------------------------------------------------------------------------ seeded sweep
def _sweep_data(batch, n, seed):
    rng = np.random.default_rng(seed)
    scale = np.where(rng.random(batch) < 0.5, 1000.0, 1.0)[:, None, None]
    A = rng.standard_normal((batch, n, 3)) * 0.3 + rng.standard_normal((batch, 1, 3))
    Q, Rr = np.linalg.qr(rng.standard_normal((batch, 3, 3)))
    Q = Q * np.sign(np.diagonal(Rr, axis1=1, axis2=2))[:, None, :]
    Q[np.linalg.det(Q) < 0] *= -1
    s = rng.uniform(0.7, 1.4, (batch, 1, 1))
    B = s * A @ Q.transpose(0, 2, 1) + rng.standard_normal((batch, 1, 3)) + 0.02 * rng.standard_normal((batch, n, 3))
    return (A * scale).astype(np.float32), (B * scale).astype(np.float32)


@pytest.mark.parametrize("n", [1, 3, 14, 17, 255, 256, 257, 778, 6890])
@pytest.mark.parametrize("batch", [1, 7, 256, 1000])
def test_procrustes_sweep_against_oracle(batch, n):
    A, B = _sweep_data(batch, n, seed=batch * 10007 + n)
    T, Y, E, sums = _run_align(A, B)
    check = range(batch) if batch * n <= 256 * 6890 else np.random.default_rng(n).choice(batch, 64, replace=False)
    for b in check:
        _check_sample(A[b], B[b], T[b, 0], T[b, 1:10].reshape(3, 3), T[b, 10:], Y[b], E[b], f"b={b}")
    if n == 1:  # varP = 0 everywhere
        assert np.isnan(T).all() and np.isnan(sums).all()
    else:
        E0 = E.astype(np.float64).sum(1)
        assert np.allclose(sums[:batch], E0, rtol=1e-6) and np.isclose(sums[batch], sums[:batch].sum(), rtol=1e-12)


def test_bad_samples_are_nan_and_leave_their_neighbours_alone():
    A, B = _sweep_data(7, 17, seed=5)
    ref = _run_align(A, B)
    A2, B2 = A.copy(), B.copy()
    A2[2] = A2[2, :1]          # all points equal: varP = 0
    A2[4, 3, 1] = np.nan
    B2[5, 0, 2] = np.inf
    got = _run_align(A2, B2)
    for b in (2, 4, 5):
        assert np.isnan(got[0][b]).all() and np.isnan(got[1][b]).all() and np.isnan(got[2][b]).all()
        assert np.isnan(got[3][b])
    for b in (0, 1, 3, 6):
        for x, y in zip(got[:3], ref[:3]):
            assert np.array_equal(x[b], y[b])
        assert np.array_equal(got[3][b], ref[3][b])


# ------------------------------------------------------------------------------------------------ determinism
def test_results_are_bitwise_reproducible_and_position_independent():
    from pose2mesh_release_b200 import metrics

    A, B = _sweep_data(1000, 778, seed=9)
    r1, r2 = _run_align(A, B), _run_align(A, B)
    for x, y in zip(r1, r2):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    one = _run_align(A[17:18], B[17:18])
    A256, B256 = A[:256].copy(), B[:256].copy()
    A256[0], B256[0] = A[17], B[17]
    A256[255], B256[255] = A[17], B[17]
    mid = _run_align(A256, B256)
    for k in range(3):
        for got in (mid[k][0], mid[k][255], r1[k][17]):
            assert np.array_equal(got.view(np.uint8), one[k][0].view(np.uint8))
    for got in (mid[3][0], mid[3][255], r1[3][17]):
        assert got == one[3][0]
    # point errors: same bits at any batch position
    e_all = metrics.point_errors(cu(A), cu(B), root=0, subset=[1, 5, 700]).cpu().numpy()
    e_one = metrics.point_errors(cu(A[17:18]), cu(B[17:18]), root=0, subset=[1, 5, 700]).cpu().numpy()
    assert np.array_equal(e_all[17], e_one[0])


# ------------------------------------------------------------------------------------------------ end to end
@functools.lru_cache(maxsize=None)
def _hierarchy(name):
    """The seeded sphere hierarchies of test_gpu_at_size (smpl_like: 6890 vertices, mano_like: 778)."""
    import test_gpu_at_size

    graph_L, perm_rev, _, _ = test_gpu_at_size._hierarchy(name)
    return graph_L, perm_rev


def _seeded_regressor(n_joint, n_vertex, per_row, seed, sum_jitter=0.0):
    rng = np.random.default_rng(seed)
    J = np.zeros((n_joint, n_vertex))
    for j in range(n_joint):
        cols = rng.choice(n_vertex, per_row, replace=False)
        w = rng.random(per_row)
        J[j, cols] = w / w.sum() * (1.0 + rng.uniform(-sum_jitter, sum_jitter))
    return J


def _check_evaluate(pred, gt, Jm, Jh, eval_joint, gt_joints, pa_mesh=True):
    from pose2mesh_release_b200 import metrics

    got = metrics.evaluate_meshes(pred, gt, torch.as_tensor(Jm, dtype=torch.float32), 0,
                                  torch.as_tensor(Jh, dtype=torch.float32), 0, eval_joint=eval_joint,
                                  gt_joints=gt_joints, pa_mesh=pa_mesh)
    got = {k: v.cpu().numpy() for k, v in got.items()}
    P, G = pred.cpu().double().numpy(), gt.cpu().double().numpy()
    GJ = None if gt_joints is None else gt_joints.cpu().double().numpy()
    keys = {"mpjpe", "pa_mpjpe", "mpjpe_mesh_joints", "mpvpe"} | ({"pa_mpvpe"} if pa_mesh else set())
    assert set(got) == keys
    worst = 0.0
    for b in range(len(P)):
        ref = mo.evaluate_sample(P[b], G[b], Jm, 0, Jh, 0, eval_joint, None if GJ is None else GJ[b], pa_mesh)
        scale = max(np.abs(P[b]).max(), np.abs(G[b]).max())
        for k in keys:
            assert got[k][b].shape == ref[k].shape, k
            d = np.abs(got[k][b] - ref[k]).max() / scale
            worst = max(worst, d)
            assert d <= 1e-6, (k, b, d)
    return worst


@pytest.mark.parametrize("gt_source", ["gt_joints", "regressed"])
def test_evaluate_meshes_smpl_b256_against_oracle(gt_source):
    from pose2mesh_release_b200 import pose2mesh_net

    graph_L, perm_rev = _hierarchy("smpl_like")
    torch.manual_seed(123)
    flat = pose2mesh_net.get_model(17, graph_L).to(dev()).eval()
    Jh = Z["J_regressor_h36m"]
    pose2d = torch.randn(256, 17, 2, generator=torch.Generator().manual_seed(4)).to(dev())
    verts, joints, _ = flat.predict_vertices_and_joints(pose2d, perm_rev, 6890, torch.as_tensor(Jh).float())
    pred = verts * 1000.0
    g = torch.Generator().manual_seed(8)
    gt = pred + 30.0 * torch.randn(pred.shape, generator=g).to(dev())
    Jm = _seeded_regressor(24, 6890, 30, seed=11)
    gt_joints = (joints * 1000.0 + 20.0 * torch.randn(joints.shape, generator=g).to(dev())) \
        if gt_source == "gt_joints" else None
    assert float(pred.std()) > 1e-3
    _check_evaluate(pred, gt, Jm, Jh, H36M_EVAL, gt_joints)


@pytest.mark.parametrize("gt_source", ["gt_joints", "regressed"])
def test_evaluate_meshes_mano_b1024_against_oracle(gt_source):
    from pose2mesh_release_b200 import postprocess
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    graph_L, perm_rev = _hierarchy("mano_like")
    torch.manual_seed(123)
    model = Pose2Mesh(5, 3, graph_L, joint_set="mano").to(dev()).eval()
    x = torch.randn(1024, 21, 5, generator=torch.Generator().manual_seed(2)).to(dev())
    g = torch.Generator().manual_seed(3)
    # the untrained network's vertices barely spread, so a seeded hand-sized shape (80 mm) keeps every sample's
    # Procrustes well conditioned: near-coincident joints would amplify the fp32 rounding of the regression by c
    shape = 80.0 * torch.randn(778, 3, generator=g).to(dev())
    with torch.no_grad():
        pred = model.forward_vertices(x, perm_rev, 778) * 100.0 + shape
    gt = pred + 5.0 * torch.randn(pred.shape, generator=g).to(dev())
    J = _seeded_regressor(21, 778, 12, seed=13, sum_jitter=1e-3)
    assert np.abs(J.sum(1) - 1.0).max() <= 1e-3
    gt_joints = None
    if gt_source == "gt_joints":
        gt_joints = postprocess.regress_joints(gt, torch.as_tensor(J).float()) + \
            2.0 * torch.randn(1024, 21, 3, generator=g).to(dev())
    _check_evaluate(pred, gt, J, J, None, gt_joints)


# ------------------------------------------------------------------------------------------------ errors
def test_bad_arguments_raise_and_leave_no_pending_error():
    from pose2mesh_release_b200 import _lib, metrics

    a = torch.randn(4, 17, 3, device=dev())
    with pytest.raises(RuntimeError):
        metrics.rigid_align(a.cpu(), a.cpu())
    with pytest.raises(RuntimeError):
        metrics.point_errors(a, a.cpu())
    with pytest.raises(RuntimeError):
        metrics.compute_joint_err(a.cpu(), a.cpu())
    with pytest.raises(ValueError):
        metrics.rigid_transform(a, a[:, :16])
    with pytest.raises(ValueError):
        metrics.point_errors(a, a[:3])
    with pytest.raises(ValueError):
        metrics.compute_both_err(a, a, a[:2], a[:2])
    with pytest.raises(ValueError):
        metrics.point_errors(a, a, subset=[0, 17])
    with pytest.raises(ValueError):
        metrics.compute_joint_err(a, a, root=17)
    # the library checks the subset itself (host side, before any launch)
    lib = _lib.load()
    err = torch.empty(4, 2, device=dev())
    bad = (C.c_int32 * 2)(3, 17)
    stream = torch.cuda.current_stream().cuda_stream
    assert lib.p2m_point_errors(a.data_ptr(), a.data_ptr(), None, None, 4, 17, bad, 2, 0, err.data_ptr(), None,
                                stream) == 1
    assert b"subset[1] = 17" in lib.p2m_last_error()
    neg = (C.c_int32 * 1)(-1)
    assert lib.p2m_rigid_align(a.data_ptr(), a.data_ptr(), 4, 17, neg, 1, None, None, err.data_ptr(), None,
                               stream) == 1
    assert lib.p2m_rigid_align(a.data_ptr(), a.data_ptr(), 4, 17, None, 0, None, None, None, None, stream) == 1
    assert lib.p2m_rigid_align(a.cpu().data_ptr(), a.data_ptr(), 4, 17, None, 0, None, None, err.data_ptr(), None,
                               stream) == 1
    assert lib.p2m_point_errors(a.data_ptr(), a.data_ptr(), None, None, 1 << 25, 17, None, 0, 0, err.data_ptr(), None,
                                stream) == 1
    torch.cuda.synchronize()
    # the device is healthy: a fresh call works
    assert metrics.compute_joint_err(a, a) == 0.0
    torch.cuda.synchronize()
