"""Mesh losses on the GPU: drop-ins for ``core.loss.CoordLoss / NormalVectorLoss / EdgeLengthLoss``
(lib/core/loss.py:10-23,62-114) — SURVEY.md §8 row f3.

Same constructors and ``forward`` signatures.  The face-indexed gathers, normalisations and reductions of one call
run as ONE kernel over (mesh, face) in libp2m_b200.so (``p2m_mesh_losses``), forward and — recomputed with the
upstream gradients — backward; the face table is uploaded once per device instead of once per call
(the reference builds ``torch.LongTensor(self.face).cuda()`` in every forward, loss.py:68,97).
``MeshLosses(face)`` returns both face losses from a single pass.

``Pose2MeshLoss`` is the Trainer's whole objective (lib/core/base.py:129-143) as one autograd op: the gather of the real
rows out of the model's padded output, the joint regression and the five weighted terms, forward and backward, in
``p2m_pose2mesh_loss`` / ``p2m_pose2mesh_loss_backward``.
"""
from __future__ import annotations

import ctypes as C

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


class _Pose2MeshLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cam_mesh, lift_pose, gt_mesh, gt_reg3dpose, gt_lift3dpose, mesh_valid, reg3dpose_valid,
                lift3dpose_valid, faces, jr, perm, weights, edge):
        x, lp = cam_mesh.contiguous().float(), lift_pose.contiguous().float()
        B = x.shape[0]
        pred_pose = torch.empty((B, jr.shape[0], 3), device=x.device, dtype=torch.float32)
        loss = torch.empty((), device=x.device, dtype=torch.float32)
        terms = torch.empty(5, device=x.device, dtype=torch.float32)
        saved = (x, lp, gt_mesh, gt_reg3dpose, gt_lift3dpose, mesh_valid, reg3dpose_valid, lift3dpose_valid, faces, jr,
                 perm, weights, edge, pred_pose)
        a = _pose2mesh_args(*saved, scratch=_scratch(x), loss=loss, terms=terms)
        _lib.call("p2m_pose2mesh_loss", x.device, C.byref(a))
        ctx.save_for_backward(*saved)
        ctx.mark_non_differentiable(terms)
        return loss, terms

    @staticmethod
    def backward(ctx, g_loss, g_terms):
        saved = ctx.saved_tensors
        x, lp = saved[0], saved[1]
        d_x, d_lp = torch.empty_like(x), torch.empty_like(lp)
        a = _pose2mesh_args(*saved, scratch=_scratch(x), grad_loss=g_loss.contiguous().float(), d_cam_mesh=d_x,
                            d_lift_pose=d_lp)
        _lib.call("p2m_pose2mesh_loss_backward", x.device, C.byref(a))
        return (d_x, d_lp) + (None,) * 11


def _scratch(x):
    return torch.empty(32 * (x.shape[0] + 1), device=x.device, dtype=torch.uint8)


def _pose2mesh_args(x, lp, gt_mesh, gt_reg, gt_lift, mesh_valid, reg_valid, lift_valid, faces, jr, perm, weights, edge,
                    pred_pose, **out):
    a = _lib.Pose2MeshLossArgs(x.shape[0], x.shape[1], gt_mesh.shape[1], faces.shape[0], jr.shape[0], lp.shape[1])
    for name, t in (("cam_mesh", x), ("lift_pose", lp), ("gt_mesh", gt_mesh), ("gt_reg3dpose", gt_reg),
                    ("gt_lift3dpose", gt_lift), ("mesh_valid", mesh_valid), ("reg3dpose_valid", reg_valid),
                    ("lift3dpose_valid", lift_valid), ("faces", faces), ("joint_regressor", jr),
                    ("perm_reverse", perm), ("weights", weights), ("edge", edge), ("pred_pose", pred_pose),
                    *out.items()):
        setattr(a, name, t.data_ptr())
    return a


class Pose2MeshLoss(nn.Module):
    """The Trainer's objective, lib/core/base.py:129-143, as one autograd op:

        pred_mesh = cam_mesh[:, perm_reverse[:n_vertex]]            n_vertex = face.max() + 1
        pred_pose = joint_regressor @ (pred_mesh * 1000)
        loss1 = CoordLoss(pred_mesh, gt_mesh, mesh_valid)
        loss2 = normal_weight * NormalVectorLoss(pred_mesh, gt_mesh)
        loss3 = edge_weight * EdgeLengthLoss(pred_mesh, gt_mesh) if edge else 0
        loss4 = joint_weight * CoordLoss(pred_pose, gt_reg3dpose, reg3dpose_valid)
        loss5 = joint_weight * CoordLoss(lift_pose, gt_lift3dpose, lift3dpose_valid)

    ``forward`` returns ``(loss, terms)``: the differentiable float32 sum of the five and a detached float32 [5] holding
    loss1 .. loss5 as the Trainer logs them.  ``cam_mesh`` is the padded [B, V0, 3] output of the model; its gradient
    comes back in that layout with the padding rows exactly zero.  Masks broadcast like the reference's
    ``pred * valid`` from [B, n, 1].  ``edge`` is a bool or a one-element CUDA tensor read on the device (nonzero:
    on), so a captured graph switches the edge term on at ``epoch > edge_loss_start`` (the reference's strict test)
    without being captured again.  Nothing synchronises with the host.

    The vertex, joint and lift terms are reduced in a fixed order and are bitwise reproducible; the normal and edge
    terms are those of ``MeshLosses`` (fp64 atomics across CTAs in the forward, fp32 atomics in the gradient).
    """

    def __init__(self, face, joint_regressor, perm_reverse, normal_weight=0.1, edge_weight=20.0, joint_weight=1e-3):
        super().__init__()
        self._table = _FaceTable(face)
        self.n_vertex = int(self._table.face.max()) + 1
        jr = torch.as_tensor(np.asarray(joint_regressor.detach().cpu() if isinstance(joint_regressor, torch.Tensor)
                                        else joint_regressor), dtype=torch.float32).contiguous()
        if jr.dim() != 2 or jr.shape[1] != self.n_vertex or not 1 <= jr.shape[0] <= _lib.P2M_POSE2MESH_MAX_REG_JOINT:
            raise ValueError(f"joint_regressor must be [J <= {_lib.P2M_POSE2MESH_MAX_REG_JOINT}, {self.n_vertex}], "
                             f"got {tuple(jr.shape)}")
        perm = np.asarray(perm_reverse).reshape(-1)[: self.n_vertex].astype(np.int64)
        if len(perm) != self.n_vertex or perm.min() < 0 or len(np.unique(perm)) != self.n_vertex:
            raise ValueError(f"perm_reverse must hold {self.n_vertex} distinct non-negative rows")
        self.n_rows_min = int(perm.max()) + 1
        self._jr, self._perm = jr, torch.from_numpy(perm.astype(np.int32))
        self._weights = torch.tensor([normal_weight, edge_weight, joint_weight], dtype=torch.float32)
        self.normal_weight, self.edge_weight, self.joint_weight = normal_weight, edge_weight, joint_weight
        self._dev = {}

    def _on(self, device):
        t = self._dev.get(device)
        if t is None:
            t = (self._table.on(device), self._jr.to(device), self._perm.to(device), self._weights.to(device),
                 {flag: torch.full((1,), float(flag), device=device) for flag in (False, True)})
            self._dev[device] = t
        return t

    def forward(self, cam_mesh, lift_pose, gt_mesh, gt_reg3dpose, gt_lift3dpose, mesh_valid, reg3dpose_valid,
                lift3dpose_valid, edge=True):
        _lib.cuda_tensor(cam_mesh, "cam_mesh")
        _lib.cuda_tensor(lift_pose, "lift_pose")
        dev = cam_mesh.device
        faces, jr, perm, weights, flags = self._on(dev)
        B, nj = cam_mesh.shape[0], jr.shape[0]
        if cam_mesh.dim() != 3 or cam_mesh.shape[2] != 3 or cam_mesh.shape[1] < self.n_rows_min:
            raise ValueError(f"cam_mesh must be [B, V0 >= {self.n_rows_min}, 3], got {tuple(cam_mesh.shape)}")
        if lift_pose.dim() != 3 or lift_pose.shape[0] != B or lift_pose.shape[2] != 3:
            raise ValueError(f"lift_pose must be [{B}, J, 3], got {tuple(lift_pose.shape)}")
        nl = lift_pose.shape[1]

        def target(t, n, what):
            if tuple(t.shape) != (B, n, 3):
                raise ValueError(f"{what} must be [{B}, {n}, 3], got {tuple(t.shape)}")
            return _lib.cuda_tensor(t, what).contiguous().float()

        def mask(t, n, what):
            _lib.cuda_tensor(t, what)
            return t.expand(B, n, 1).reshape(B, n).contiguous().float()

        if isinstance(edge, torch.Tensor):
            if edge.numel() != 1 or edge.device != dev:
                raise ValueError("edge must be a bool or a one-element tensor on cam_mesh's device")
            edge = edge.reshape(1).float()
        else:
            edge = flags[bool(edge)]
        return _Pose2MeshLossFn.apply(
            cam_mesh, lift_pose, target(gt_mesh, self.n_vertex, "gt_mesh"), target(gt_reg3dpose, nj, "gt_reg3dpose"),
            target(gt_lift3dpose, nl, "gt_lift3dpose"), mask(mesh_valid, self.n_vertex, "mesh_valid"),
            mask(reg3dpose_valid, nj, "reg3dpose_valid"), mask(lift3dpose_valid, nl, "lift3dpose_valid"), faces, jr,
            perm, weights, edge)
