"""The steps either side of the model in the reference's callers, on the GPU (SURVEY.md §8 row f2):

    regress_joints(verts, J)      lib/core/base.py:131,204; demo/run.py:171   joints = J_regressor @ vertices
    normalize_pose2d(joints_px)   demo/run.py:150-158                          pixels -> network input coordinates

Both run in libp2m_b200.so (p2m_regress_joints and its backward, p2m_normalize_pose2d); CUDA tensors only.
"""
from __future__ import annotations

import torch

from . import _lib

INPUT_SHAPE = (384, 288)  # cfg.MODEL.input_shape (height, width), lib/core/config.py:52


def _regress(v: torch.Tensor, jr: torch.Tensor) -> torch.Tensor:
    B, nv, ch = v.shape
    out = torch.empty((B, jr.shape[0], ch), device=v.device, dtype=torch.float32)
    _lib.call("p2m_regress_joints", v.device, jr, v, out, B, jr.shape[0], nv, ch)
    return out


class _RegressJointsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vertices, jr):
        v = vertices.contiguous().float()
        ctx.save_for_backward(jr)
        ctx.shape = tuple(v.shape)
        return _regress(v, jr)

    @staticmethod
    def backward(ctx, g):
        (jr,) = ctx.saved_tensors
        B, nv, ch = ctx.shape
        g = g.contiguous().float()
        dv = torch.empty((B, nv, ch), device=g.device, dtype=torch.float32)
        _lib.call("p2m_regress_joints_backward", g.device, jr, g, dv, B, jr.shape[0], nv, ch)
        return dv, None


def regress_joints(vertices: torch.Tensor, joint_regressor: torch.Tensor) -> torch.Tensor:
    """vertices [B, n_vertex, C] (C <= 4), joint_regressor [n_joint, n_vertex] -> joints [B, n_joint, C].
    Differentiable in ``vertices`` (d vertices = joint_regressor^T d joints, p2m_regress_joints_backward); the
    regressor is a constant and may not require grad."""
    _lib.cuda_tensor(vertices, "vertices")
    jr = joint_regressor.to(vertices.device).contiguous().float()
    if vertices.dim() != 3 or jr.shape[1] != vertices.shape[1]:
        raise ValueError(f"joint_regressor has {jr.shape[1]} columns, vertices has shape {tuple(vertices.shape)}")
    if torch.is_grad_enabled() and joint_regressor.requires_grad:
        raise ValueError("regress_joints: no gradient with respect to joint_regressor")
    if torch.is_grad_enabled() and vertices.requires_grad:
        return _RegressJointsFn.apply(vertices, jr)
    return _regress(vertices.contiguous().float(), jr)


def normalize_pose2d(joints_px: torch.Tensor, input_shape=INPUT_SHAPE) -> torch.Tensor:
    """joints_px [B, J, 2] (or [J, 2]) image pixels on a CUDA device -> pose2d [B, J, 2] as demo/run.py:150-158
    computes it.  Integer tensors are treated like the reference treats integer arrays (its in-place affine transform
    truncates the transformed coordinates, aug_utils.py:57-59)."""
    _lib.cuda_tensor(joints_px, "joints_px")
    truncate = int(not joints_px.is_floating_point())
    x = joints_px.reshape(-1, joints_px.shape[-2], 2).contiguous().float()
    out = torch.empty_like(x)
    _lib.call("p2m_normalize_pose2d", x.device, x, out, x.shape[0], x.shape[1], int(input_shape[0]),
              int(input_shape[1]), truncate)
    return out
