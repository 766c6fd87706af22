"""The float64 oracle of the evaluation metrics (oracle/metrics_oracle.py) against golden vectors of the unmodified
reference functions (tests/golden/eval_metrics.npz, made by tests/golden/make_golden_metrics.py)."""
import numpy as np
import pytest

from helpers import load_npz
from oracle import metrics_oracle as mo

Z = load_npz("eval_metrics.npz")
NAMES = [str(s) for s in Z["rt_names"]]


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


@pytest.mark.parametrize("i", range(len(NAMES)), ids=NAMES)
def test_rigid_transform_matches_reference(i):
    A, B = Z[f"rt{i}_A"].astype(np.float64), Z[f"rt{i}_B"].astype(np.float64)
    c, R, t = mo.rigid_transform_3D(A, B)
    aligned = mo.rigid_align(A, B)[Z[f"rt{i}_rows"]]
    if NAMES[i] == "all_equal":
        assert np.isnan(c) and np.isnan(t).all() and np.isnan(aligned).all()
        assert np.isnan(Z[f"rt{i}_c"]) and np.isnan(Z[f"rt{i}_aligned"]).all()
        return
    assert abs(c - Z[f"rt{i}_c"]) <= 1e-12 * abs(Z[f"rt{i}_c"])
    assert _rel(t, Z[f"rt{i}_t"]) <= 1e-12
    assert _rel(aligned, Z[f"rt{i}_aligned"]) <= 1e-12
    if NAMES[i] != "collinear":  # rank-1 H: R is not unique (the aligned points are)
        assert _rel(R, Z[f"rt{i}_R"]) <= 1e-12
    assert abs(np.linalg.det(R) - 1.0) < 1e-12


def test_mirrored_case_takes_the_det_branch():
    i = NAMES.index("mirrored")
    A, B = Z[f"rt{i}_A"].astype(np.float64), Z[f"rt{i}_B"].astype(np.float64)
    H = (A - A.mean(0)).T @ (B - B.mean(0))
    U, _, Vh = np.linalg.svd(H)
    assert np.linalg.det(Vh.T @ U.T) < 0
    c, R, _ = mo.rigid_transform_3D(A, B)
    assert np.linalg.det(R) > 0 and c < np.linalg.svd(H, compute_uv=False).sum() / len(A) / np.var(A, 0).sum()


@pytest.mark.parametrize("tag", ["h36m", "pw3d", "surreal"])
def test_compute_err_matches_reference(tag):
    sub = lambda key: (Z[key].tolist() or None)  # noqa: E731
    pj, gj = Z[f"{tag}_pred_joint"], Z[f"{tag}_gt_joint"]
    pm, gm = Z[f"{tag}_pred_mesh"], Z[f"{tag}_gt_mesh"]
    je = mo.joint_err(pj, gj, root=int(Z[f"{tag}_joint_root"]), eval_joint=sub(f"{tag}_joint_subset"))
    assert abs(je - Z[f"{tag}_joint_err"]) <= 1e-6 * Z[f"{tag}_joint_err"]
    bj, bm = mo.both_err(pm, gm, pj, gj, eval_joint=sub(f"{tag}_both_subset"))
    assert abs(bj - Z[f"{tag}_both_joint_err"]) <= 1e-6 * Z[f"{tag}_both_joint_err"]
    assert abs(bm - Z[f"{tag}_both_mesh_err"]) <= 1e-6 * Z[f"{tag}_both_mesh_err"]
    pp = mo.point_errors(pm, gm, pred_root=pj[:, 0], gt_root=gj[:, 0])
    assert _rel(pp, Z[f"{tag}_mesh_pp"]) <= 1e-6


def test_h36m_regressor_rows_do_not_sum_to_one():
    """Why evaluate_sample regresses the eval joints from the ROOTED mesh: the order changes the joints."""
    J = Z["J_regressor_h36m"]
    assert J.shape == (17, 6890)
    s = J.sum(1)
    assert s.min() < 0.9997 and s.max() > 1.00004
