"""The evaluation step of the reference's test loop, on the GPU (SURVEY.md §8 row f5):

    rigid_transform(A, B) / rigid_align(A, B)   lib/coord_utils.py:127-149        similarity Procrustes, batched
    point_errors(pred, gt, ...)                 the root-aligned distances of the datasets' compute_*_err
    compute_joint_err / compute_both_err        data/Human36M/dataset.py:454-477, data/PW3D/dataset.py:263-286,
                                                data/SURREAL/dataset.py:205-226  (Tester.test, lib/core/base.py:196-214)
    evaluate_meshes(...)                        the per-sample body of Human36M.evaluate (data/Human36M/dataset.py:
                                                540-568) and PW3D.evaluate (data/PW3D/dataset.py:342-375)

Everything runs in libp2m_b200.so (p2m_rigid_align, p2m_point_errors, p2m_regress_joints); CUDA tensors only.  Point
sets are [B, n, 3] or [n, 3] (a single sample).  Subsets and root indices are host-side indices (tuples, lists, numpy
arrays); an index outside the point set raises.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .postprocess import regress_joints

H36M_EVAL_JOINT = (1, 2, 3, 4, 5, 6, 8, 10, 11, 12, 13, 14, 15, 16)  # data/Human36M/dataset.py:62


def _points(x: torch.Tensor, what: str) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.dim() == 2:
        x = x.unsqueeze(0)
    if x.dim() != 3 or x.shape[-1] != 3 or x.shape[0] == 0 or x.shape[1] == 0:
        raise ValueError(f"{what} must be [B, n, 3] or [n, 3] with B, n > 0; got {tuple(x.shape)}")
    return x.contiguous().float()


def _pair(a: torch.Tensor, b: torch.Tensor, names=("A", "B")):
    squeeze = a.dim() == 2
    a, b = _points(a, names[0]), _points(b, names[1])
    if a.shape != b.shape:
        raise ValueError(f"{names[0]} {tuple(a.shape)} and {names[1]} {tuple(b.shape)} differ in shape")
    if a.device != b.device:
        raise ValueError(f"{names[0]} is on {a.device}, {names[1]} on {b.device}")
    return a, b, squeeze


def _subset(subset, n: int):
    """-> (ctypes int32 array or None, k).  Indices are checked against n by the library as well."""
    if subset is None:
        return None, n
    idx = np.asarray(subset.cpu() if isinstance(subset, torch.Tensor) else subset, dtype=np.int64).reshape(-1)
    if idx.size == 0:
        raise ValueError("empty subset")
    if idx.min() < 0 or idx.max() >= n:
        raise ValueError(f"subset index out of range [0, {n}): {idx.tolist()}")
    return (C.c_int32 * idx.size)(*idx.tolist()), int(idx.size)


def _root_index(root: int, n: int) -> int:
    if not -n <= int(root) < n:
        raise ValueError(f"root index {root} out of range for {n} points")
    return int(root) % n


def _align(A, B, subset=None, transform=False, aligned=False, err=False, sums=None):
    """One p2m_rigid_align call on [B, n, 3] float32 CUDA tensors; returns the requested outputs."""
    batch, n = A.shape[0], A.shape[1]
    sub, k = _subset(subset, n)
    T = torch.empty((batch, 13), device=A.device, dtype=torch.float64) if transform else None
    Y = torch.empty((batch, k, 3), device=A.device, dtype=torch.float32) if aligned else None
    E = torch.empty((batch, k), device=A.device, dtype=torch.float32) if err else None
    _lib.call("p2m_rigid_align", A.device, A, B, batch, n, sub, k if sub is not None else 0, T, Y, E, sums)
    return T, Y, E


def _errors(pred, gt, pred_root=None, gt_root=None, subset=None, fp64=False, err=True, sums=None):
    """One p2m_point_errors call; roots are [B, 3] float32 contiguous (or None)."""
    batch, n = pred.shape[0], pred.shape[1]
    sub, k = _subset(subset, n)
    E = torch.empty((batch, k), device=pred.device, dtype=torch.float32) if err else None
    _lib.call("p2m_point_errors", pred.device, pred, gt, pred_root, gt_root, batch, n, sub, k if sub is not None else 0,
              int(fp64), E, sums)
    return E


def _root_rows(x: torch.Tensor, root, what: str, batch: int, device) -> torch.Tensor:
    """A per-sample root point: an index into x ([B, n, 3]) or an explicit [B, 3] / [B, 1, 3] / [3] tensor."""
    if isinstance(root, torch.Tensor):
        r = _lib.cuda_tensor(root, what).reshape(-1, 3)
        if r.shape[0] == 1 and batch > 1:
            r = r.expand(batch, 3)
        if r.shape[0] != batch or r.device != device:
            raise ValueError(f"{what} must hold one point per sample ({batch}) on {device}; got {tuple(root.shape)}")
        return r.contiguous().float()
    return x[:, _root_index(root, x.shape[1])].contiguous()


# ---------------------------------------------------------------------------------------------- public functions
def rigid_transform(A: torch.Tensor, B: torch.Tensor):
    """Batched coord_utils.rigid_transform_3D: the similarity (c, R, t) minimising |c R A + t - B| per sample, with the
    reference's conventions (R = Vh^T U^T, det R < 0 corrected by negating s[-1] and Vh[2], c = sum(s) / var(A)).
    A, B [B, n, 3] or [n, 3] -> c [B], R [B, 3, 3], t [B, 3] in float64 (no batch dimension for [n, 3] inputs).
    Samples whose A points are all equal, or that hold a non-finite value, get NaN."""
    A, B, squeeze = _pair(A, B)
    T, _, _ = _align(A, B, transform=True)
    c, R, t = T[:, 0], T[:, 1:10].reshape(-1, 3, 3), T[:, 10:13]
    return (c[0], R[0], t[0]) if squeeze else (c, R, t)


def rigid_align(A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """Batched coord_utils.rigid_align: A mapped by its Procrustes similarity onto B (float32, A's shape)."""
    A, B, squeeze = _pair(A, B)
    _, Y, _ = _align(A, B, aligned=True)
    return Y[0] if squeeze else Y


def point_errors(pred: torch.Tensor, gt: torch.Tensor, root=None, subset=None, pred_root=None, gt_root=None):
    """Root-aligned per-point distances |(pred_i - pred_root) - (gt_i - gt_root)| -> [B, k] float32 (k = len(subset)
    or n), bit for bit what the reference's float32 numpy computes.  `root` is an index into the same point set
    (0 for H36M / SURREAL, -2 for PW3D joints); `pred_root` / `gt_root` ([B, 3]) give the root points explicitly, e.g.
    the joint root a mesh is aligned at.  The roots are taken before the subset, as the reference does."""
    squeeze = pred.dim() == 2
    pred, gt, _ = _pair(pred, gt, ("pred", "gt"))
    if root is not None and (pred_root is not None or gt_root is not None):
        raise ValueError("give either root or pred_root / gt_root")
    if (pred_root is None) != (gt_root is None):
        raise ValueError("give both pred_root and gt_root")
    pr = gr = None
    if root is not None:
        pr, gr = (_root_rows(x, root, "root", pred.shape[0], pred.device) for x in (pred, gt))
    elif pred_root is not None:
        pr = _root_rows(pred, pred_root, "pred_root", pred.shape[0], pred.device)
        gr = _root_rows(gt, gt_root, "gt_root", pred.shape[0], pred.device)
    E = _errors(pred, gt, pr, gr, subset)
    return E[0] if squeeze else E


def _means(sums: torch.Tensor, counts):
    """The only host synchronisation of the compute_*_err functions: one read of the batch totals."""
    totals = sums[:, -1].tolist()
    return [s / n for s, n in zip(totals, counts)]


def compute_joint_err(pred_joint: torch.Tensor, target_joint: torch.Tensor, root: int = 0, eval_joint=None) -> float:
    """The datasets' compute_joint_err: mean root-aligned joint error over the batch (and the eval joints).
    H36M: root=0, eval_joint=H36M_EVAL_JOINT; PW3D: root=-2; SURREAL: root=0."""
    pred, gt, _ = _pair(pred_joint, target_joint, ("pred_joint", "target_joint"))
    batch = pred.shape[0]
    r = _root_index(root, pred.shape[1])
    sums = torch.empty((1, batch + 1), device=pred.device, dtype=torch.float64)
    k = _subset(eval_joint, pred.shape[1])[1]
    _errors(pred, gt, pred[:, r].contiguous(), gt[:, r].contiguous(), eval_joint, err=False, sums=sums[0])
    return _means(sums, [batch * k])[0]


def compute_both_err(pred_mesh: torch.Tensor, target_mesh: torch.Tensor, pred_joint: torch.Tensor,
                     target_joint: torch.Tensor, eval_joint=None):
    """The datasets' compute_both_err -> (joint_mean_error, mesh_mean_error): meshes and joints root-aligned at joint 0,
    joint errors over eval_joint (H36M and PW3D: H36M_EVAL_JOINT; SURREAL: None = all joints)."""
    pm, gm, _ = _pair(pred_mesh, target_mesh, ("pred_mesh", "target_mesh"))
    pj, gj, _ = _pair(pred_joint, target_joint, ("pred_joint", "target_joint"))
    if pm.shape[0] != pj.shape[0] or pm.device != pj.device:
        raise ValueError(f"meshes {tuple(pm.shape)} and joints {tuple(pj.shape)} differ in batch size or device")
    batch = pm.shape[0]
    pr, gr = pj[:, 0].contiguous(), gj[:, 0].contiguous()
    k = _subset(eval_joint, pj.shape[1])[1]
    sums = torch.empty((2, batch + 1), device=pm.device, dtype=torch.float64)
    _errors(pj, gj, pr, gr, eval_joint, err=False, sums=sums[0])
    _errors(pm, gm, pr, gr, None, err=False, sums=sums[1])
    joint, mesh = _means(sums, [batch * k, batch * pm.shape[1]])
    return joint, mesh


def evaluate_meshes(pred_verts: torch.Tensor, gt_verts: torch.Tensor, mesh_regressor: torch.Tensor, mesh_root: int,
                    joint_regressor: torch.Tensor, joint_root: int, eval_joint=None, gt_joints: torch.Tensor = None,
                    pa_mesh: bool = True):
    """Per-sample errors of the datasets' final evaluation for a batch of meshes [B, V, 3], in the reference's order:

      1. mesh joints = mesh_regressor @ mesh (SMPL: the model's J_regressor, mesh_root = its root joint);
      2. meshes and mesh joints rooted at the mesh joint `mesh_root`;
      3. eval joints = joint_regressor @ the ROOTED mesh (H36M regressor; its rows do not sum to exactly 1, so the
         order matters), or `gt_joints` [B, J, 3] for the target when given (H36M's annot['joint_cam']);
      4. eval joints rooted at `joint_root` and restricted to `eval_joint`.

    Returns a dict of [B, k] float32 device tensors: ``mpjpe`` / ``pa_mpjpe`` (eval joints, after Procrustes for the
    latter), ``mpjpe_mesh_joints`` (joints of mesh_regressor), ``mpvpe`` and, with pa_mesh, ``pa_mpvpe``.  The
    regressions accumulate in fp32 (p2m_regress_joints); rooting, distances and Procrustes run in fp64.  Nothing is
    read back to the host."""
    pv, gv, _ = _pair(pred_verts, gt_verts, ("pred_verts", "gt_verts"))
    mr = _root_index(mesh_root, mesh_regressor.shape[0])
    jr = _root_index(joint_root, joint_regressor.shape[0])
    # 1-2: mesh joints, rooted distances of the mesh joints and of the mesh
    jm_out, jm_gt = regress_joints(pv, mesh_regressor), regress_joints(gv, mesh_regressor)
    r_out, r_gt = jm_out[:, mr].contiguous(), jm_gt[:, mr].contiguous()
    out = {"mpjpe_mesh_joints": _errors(jm_out, jm_gt, r_out, r_gt, fp64=True),
           "mpvpe": _errors(pv, gv, r_out, r_gt, fp64=True)}
    if pa_mesh:  # Procrustes is translation invariant: rooting the meshes first changes nothing
        out["pa_mpvpe"] = _align(pv, gv, err=True)[2]
    # 3: eval joints from the rooted meshes
    jh_out = regress_joints(pv - r_out[:, None], joint_regressor)
    if gt_joints is not None:
        jh_gt = _points(gt_joints, "gt_joints")
        if jh_gt.shape != jh_out.shape or jh_gt.device != pv.device:
            raise ValueError(f"gt_joints {tuple(jh_gt.shape)} must match the regressed joints {tuple(jh_out.shape)}")
    else:
        jh_gt = regress_joints(gv - r_gt[:, None], joint_regressor)
    # 4: rooted at joint_root, restricted to the eval joints
    out["mpjpe"] = _errors(jh_out, jh_gt, jh_out[:, jr].contiguous(), jh_gt[:, jr].contiguous(), eval_joint, fp64=True)
    out["pa_mpjpe"] = _align(jh_out, jh_gt, eval_joint, err=True)[2]
    return out
