"""TEST INFRASTRUCTURE ONLY — float64 numpy restatement of the reference's evaluation metrics.

    rigid_transform_3D(A, B), rigid_align(A, B)   lib/coord_utils.py:127-149
    joint_err(...), both_err(...)                 compute_joint_err / compute_both_err of data/Human36M/dataset.py:454-477,
                                                  data/PW3D/dataset.py:263-286, data/SURREAL/dataset.py:205-226
    evaluate_sample(...)                          the per-sample body of Human36M.evaluate (data/Human36M/dataset.py:
                                                  540-568) and PW3D.evaluate (data/PW3D/dataset.py:342-375)

The reference computes compute_*_err in float32 (torch root subtraction, numpy distances and mean); here everything is
float64, which agrees with it to the float32 rounding of those means.  evaluate_sample keeps the reference's order of
operations: the eval joints are regressed from the ROOTED mesh, which matters because the H36M regressor's rows do not
sum to exactly 1.
"""
import numpy as np


def rigid_transform_3D(A, B):
    """c, R, t with B ~ c R A + t (coord_utils.py:127-143): R = Vh^T U^T, det R < 0 -> negate s[-1] and Vh[2]."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    n = A.shape[0]
    mu_a, mu_b = A.mean(axis=0), B.mean(axis=0)
    H = (A - mu_a).T @ (B - mu_b) / n
    U, s, Vh = np.linalg.svd(H)
    R = Vh.T @ U.T
    if np.linalg.det(R) < 0:
        s[-1] = -s[-1]
        Vh[2] = -Vh[2]
        R = Vh.T @ U.T
    var_p = np.var(A, axis=0).sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        c = 1.0 / var_p * np.sum(s)
        t = -(c * R) @ mu_a + mu_b
    return c, R, t


def rigid_align(A, B):
    """A mapped by its similarity Procrustes onto B (coord_utils.py:146-149)."""
    c, R, t = rigid_transform_3D(A, B)
    with np.errstate(invalid="ignore"):
        return (c * R @ np.asarray(A, dtype=np.float64).T).T + t


def point_errors(pred, gt, root=None, subset=None, pred_root=None, gt_root=None):
    """[B, k] root-aligned distances |(pred_i - pred_root) - (gt_i - gt_root)|, roots taken before the subset."""
    pred = np.asarray(pred, dtype=np.float64)
    gt = np.asarray(gt, dtype=np.float64)
    if root is not None:
        pred_root, gt_root = pred[:, root], gt[:, root]
    if pred_root is not None:
        pred = pred - np.asarray(pred_root, dtype=np.float64).reshape(-1, 1, 3)
        gt = gt - np.asarray(gt_root, dtype=np.float64).reshape(-1, 1, 3)
    if subset is not None:
        pred, gt = pred[:, list(subset)], gt[:, list(subset)]
    return np.sqrt(((pred - gt) ** 2).sum(axis=2))


def joint_err(pred_joint, target_joint, root=0, eval_joint=None):
    """compute_joint_err: H36M root 0 + eval subset, PW3D root -2, SURREAL root 0."""
    return point_errors(pred_joint, target_joint, root=root, subset=eval_joint).mean()


def both_err(pred_mesh, target_mesh, pred_joint, target_joint, eval_joint=None):
    """compute_both_err -> (joint_mean_error, mesh_mean_error); meshes rooted at joint 0."""
    pj = np.asarray(pred_joint, dtype=np.float64)
    gj = np.asarray(target_joint, dtype=np.float64)
    mesh = point_errors(pred_mesh, target_mesh, pred_root=pj[:, 0], gt_root=gj[:, 0]).mean()
    joint = point_errors(pj, gj, root=0, subset=eval_joint).mean()
    return joint, mesh


def evaluate_sample(mesh_out, mesh_gt, mesh_regressor, mesh_root, joint_regressor, joint_root, eval_joint=None,
                    joint_gt=None, pa_mesh=True):
    """One sample of Human36M.evaluate / PW3D.evaluate in float64 -> dict of per-point error arrays:
    mpjpe_mesh_joints, mpvpe, pa_mpvpe (pa_mesh), mpjpe and pa_mpjpe (eval joints).  joint_gt: the target eval joints
    (H36M annot['joint_cam']); None regresses them from the rooted target mesh (PW3D)."""
    mesh_out = np.asarray(mesh_out, dtype=np.float64)
    mesh_gt = np.asarray(mesh_gt, dtype=np.float64)
    Jm = np.asarray(mesh_regressor, dtype=np.float64)
    Jh = np.asarray(joint_regressor, dtype=np.float64)
    sub = list(range(Jh.shape[0])) if eval_joint is None else list(eval_joint)
    # dataset.py:540-545 — regress the mesh joints, root mesh and joints at the mesh root joint
    j_out, j_gt = Jm @ mesh_out, Jm @ mesh_gt
    mesh_out = mesh_out - j_out[mesh_root:mesh_root + 1]
    mesh_gt = mesh_gt - j_gt[mesh_root:mesh_root + 1]
    pose_out = j_out - j_out[mesh_root:mesh_root + 1]
    pose_gt = j_gt - j_gt[mesh_root:mesh_root + 1]
    res = {"mpjpe_mesh_joints": np.sqrt(np.sum((pose_out - pose_gt) ** 2, 1)),
           "mpvpe": np.sqrt(np.sum((mesh_out - mesh_gt) ** 2, 1))}
    if pa_mesh:  # PW3D/dataset.py:360-361 (commented out there)
        res["pa_mpvpe"] = np.sqrt(np.sum((rigid_align(mesh_out, mesh_gt) - mesh_gt) ** 2, 1))
    # dataset.py:559-567 — eval joints from the rooted mesh, re-rooted at the joint root, eval subset
    h_out = Jh @ mesh_out
    h_out = (h_out - h_out[joint_root])[sub]
    h_gt = Jh @ mesh_gt if joint_gt is None else np.asarray(joint_gt, dtype=np.float64)
    h_gt = (h_gt - h_gt[joint_root])[sub]
    res["mpjpe"] = np.sqrt(np.sum((h_out - h_gt) ** 2, 1))
    res["pa_mpjpe"] = np.sqrt(np.sum((rigid_align(h_out, h_gt) - h_gt) ** 2, 1))
    return res
