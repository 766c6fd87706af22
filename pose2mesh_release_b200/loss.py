"""Mesh losses on the GPU: drop-ins for ``core.loss.CoordLoss / NormalVectorLoss / EdgeLengthLoss``
(lib/core/loss.py:10-23,62-114) — SURVEY.md §8 row f3.

Same constructors and ``forward`` signatures.  The face-indexed gathers, normalisations and reductions of one call
run as ONE kernel over (mesh, face) in libp2m_b200.so (``p2m_mesh_losses``), forward and — recomputed with the
upstream gradients — backward; the face table is uploaded once per device instead of once per call
(the reference builds ``torch.LongTensor(self.face).cuda()`` in every forward, loss.py:68,97).
``MeshLosses(face)`` returns both face losses from a single pass.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import _lib


class _FaceTable:
    def __init__(self, face):
        self.face = np.ascontiguousarray(np.asarray(face), dtype=np.int32).reshape(-1, 3)
        self._dev = {}

    def on(self, device: torch.device) -> torch.Tensor:
        t = self._dev.get(device)
        if t is None:
            t = torch.from_numpy(self.face).to(device)
            self._dev[device] = t
        return t


class _MeshLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, coord_out, coord_gt, faces):
        _lib.cuda_tensor(coord_out, "coord_out")
        out, gt = coord_out.contiguous().float(), coord_gt.contiguous().float()
        B, nv, _ = out.shape
        nf = faces.shape[0]
        sums = torch.empty(2, device=out.device, dtype=torch.float64)
        _lib.call("p2m_mesh_losses", out.device, out, gt, faces, B, nv, nf, None, sums, None)
        ctx.save_for_backward(out, gt, faces)
        losses = (sums / (3.0 * B * nf)).float()
        return losses[0], losses[1]

    @staticmethod
    def backward(ctx, g_normal, g_edge):
        out, gt, faces = ctx.saved_tensors
        B, nv, _ = out.shape
        nf = faces.shape[0]
        scale = (torch.stack([g_normal, g_edge]).float() / (3.0 * B * nf)).contiguous()
        grad = torch.empty_like(out)
        sums = torch.empty(2, device=out.device, dtype=torch.float64)
        _lib.call("p2m_mesh_losses", out.device, out, gt, faces, B, nv, nf, scale, sums, grad)
        return grad, None, None


class MeshLosses(nn.Module):
    """(normal_vector_loss, edge_length_loss) of lib/core/loss.py:62-114 from one pass over the faces."""

    def __init__(self, face):
        super().__init__()
        self.face = face
        self._table = _FaceTable(face)

    def forward(self, coord_out, coord_gt):
        return _MeshLossFn.apply(coord_out, coord_gt, self._table.on(coord_out.device))


class NormalVectorLoss(MeshLosses):
    """lib/core/loss.py:62-87."""

    def forward(self, coord_out, coord_gt):
        return super().forward(coord_out, coord_gt)[0]


class EdgeLengthLoss(MeshLosses):
    """lib/core/loss.py:90-114."""

    def forward(self, coord_out, coord_gt):
        return super().forward(coord_out, coord_gt)[1]


class _CoordLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, valid):
        _lib.cuda_tensor(pred, "pred")
        p, t = pred.contiguous().float(), target.contiguous().float()
        v = None if valid is None else valid.expand_as(p).contiguous().float()
        s = torch.empty(1, device=p.device, dtype=torch.float64)
        _lib.call("p2m_coord_loss", p.device, p, t, v, p.numel(), None, s, None)
        ctx.save_for_backward(p, t, v if v is not None else torch.empty(0, device=p.device))
        return (s / p.numel()).float()[0]

    @staticmethod
    def backward(ctx, g):
        p, t, v = ctx.saved_tensors
        scale = (g.float() / p.numel()).reshape(1).contiguous()
        grad = torch.empty_like(p)
        s = torch.empty(1, device=p.device, dtype=torch.float64)
        _lib.call("p2m_coord_loss", p.device, p, t, v if v.numel() else None, p.numel(), scale, s, grad)
        return grad, None, None


class CoordLoss(nn.Module):
    """lib/core/loss.py:10-23: L1 between (optionally validity-masked) coordinates."""

    def __init__(self, has_valid=False):
        super().__init__()
        self.has_valid = has_valid

    def forward(self, pred, target, target_valid=None):
        return _CoordLossFn.apply(pred, target, target_valid if self.has_valid else None)


def get_loss(faces):
    """lib/core/loss.py:117-120."""
    return (CoordLoss(has_valid=True), NormalVectorLoss(faces), EdgeLengthLoss(faces), CoordLoss(has_valid=True),
            CoordLoss(has_valid=True))
