"""The steps either side of the model in the reference's callers, on the GPU (SURVEY.md §8 row f2):

    regress_joints(verts, J)      lib/core/base.py:131,204; demo/run.py:171   joints = J_regressor @ vertices
    normalize_pose2d(joints_px)   demo/run.py:150-158                          pixels -> network input coordinates

Both run in libp2m_b200.so (p2m_regress_joints, p2m_normalize_pose2d); CUDA tensors only.
"""
from __future__ import annotations

import torch

from . import _lib

INPUT_SHAPE = (384, 288)  # cfg.MODEL.input_shape (height, width), lib/core/config.py:52


def regress_joints(vertices: torch.Tensor, joint_regressor: torch.Tensor) -> torch.Tensor:
    """vertices [B, n_vertex, C] (C <= 4), joint_regressor [n_joint, n_vertex] -> joints [B, n_joint, C]."""
    v = _lib.cuda_tensor(vertices, "vertices").contiguous().float()
    jr = joint_regressor.to(v.device).contiguous().float()
    B, nv, ch = v.shape
    if jr.shape[1] != nv:
        raise ValueError(f"joint_regressor has {jr.shape[1]} columns, vertices has {nv} rows")
    out = torch.empty((B, jr.shape[0], ch), device=v.device, dtype=torch.float32)
    _lib.call("p2m_regress_joints", v.device, jr, v, out, B, jr.shape[0], nv, ch)
    return out


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
