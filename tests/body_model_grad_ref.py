"""Float64 torch restatement of the two body-model forwards, differentiated by autograd: the gradients the reference
layers (smplpytorch SMPL_Layer.forward, manopth ManoLayer.forward) give with respect to pose, betas and trans.

tests/body_model_oracle.py restates the same maths in numpy; this copy exists so that autograd can take the
derivative of exactly that sequence of operations (batch_rodrigues with its 1e-8 offset and quat2mat's
renormalisation, subtract_flat_id, the chain in parent order, A_j = G_j - pack(G_j [J_j; 0]), skinning, centring).

`vjp` returns numpy gradients with the library's conventions: None for absent (or single-element) betas and absent
trans; zeros for given betas or trans that the forward does not use (an all-zero SMPL betas batch, an all-zero trans).
Its keyword switches mutate the gradient (never the forward) for the tests that show the GPU bound has teeth; the
public calls never set them.
"""
from __future__ import annotations

import numpy as np
import torch

from body_models import MANO_PARENTS, MANO_REORDER, MANO_TIPS


def rodrigues(theta: torch.Tensor, *, renorm: bool = True) -> torch.Tensor:
    """batch_rodrigues: [N, 3] -> [N, 3, 3]."""
    angle = torch.norm(theta + 1e-8, dim=1, keepdim=True)
    axis = theta / angle
    half = angle * 0.5
    q = torch.cat([torch.cos(half), torch.sin(half) * axis], 1)
    if renorm:
        q = q / q.norm(dim=1, keepdim=True)
    else:  # the mutation: the renormalisation's value, without its derivative
        q = q / q.norm(dim=1, keepdim=True).detach()
    w, x, y, z = q.unbind(1)
    return torch.stack([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z,
                        2 * w * z + 2 * x * y, w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x,
                        2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z, w * w - x * x - y * y + z * z], 1).view(-1, 3, 3)


def _t(a):
    return torch.as_tensor(np.asarray(a, np.float64))


def forward(model, pose, betas_used, parents, trans, center_idx, joint_map, scale, *, pose_blend=True, centre_grad=True,
            joints_path=True, transpose_dx=True, renorm=True):
    """The shared body of both layers on float64 tensors (pose, betas_used, trans may require grad).  trans None =
    not added."""
    B, J = pose.shape[0], len(parents)
    shapedirs, posedirs = _t(model["shapedirs"]), _t(model["posedirs"])
    V = shapedirs.shape[0]
    R = rodrigues(pose.reshape(-1, 3), renorm=renorm).reshape(B, J, 3, 3)
    pose_map = (R[:, 1:] - torch.eye(3, dtype=R.dtype)).reshape(B, -1)
    v_shaped = _t(model["v_template"])[None] + (shapedirs.reshape(3 * V, -1) @ betas_used.T).T.reshape(B, V, 3)
    jts = _t(model["J_regressor"])[None] @ v_shaped
    blend = (posedirs.reshape(3 * V, -1) @ pose_map.T).T.reshape(B, V, 3)
    v_posed = v_shaped + (blend if pose_blend else blend.detach())
    G = []
    bottom = torch.zeros(B, 1, 4, dtype=R.dtype)
    bottom[:, 0, 3] = 1.0
    for j in range(J):
        p = parents[j]
        t = jts[:, j] - (jts[:, p] if p >= 0 else 0.0)
        rel = torch.cat([torch.cat([R[:, j], t[:, :, None]], 2), bottom], 1)
        G.append(rel if p < 0 else G[p] @ rel)
    G = torch.stack(G, 1)
    tcol = G[:, :, :3, 3] - torch.einsum("bjrc,bjc->bjr", G[:, :, :3, :3], jts)
    A = torch.cat([G[:, :, :3, :3], tcol[..., None]], 3)                    # the top three rows of A_j
    T = torch.einsum("vj,bjrc->bvrc", _t(model["weights"]), A)
    T3 = T[..., :3]
    if transpose_dx:
        lin = torch.einsum("bvrc,bvc->bvr", T3, v_posed)
    else:  # the mutation: the same value, but d/dx is T g instead of T^T g
        tt = T3.detach().transpose(2, 3)
        lin = (torch.einsum("bvrc,bvc->bvr", T3, v_posed.detach()) + torch.einsum("bvrc,bvc->bvr", tt, v_posed)
               - torch.einsum("bvrc,bvc->bvr", tt, v_posed).detach())
    verts = lin + T[..., 3]
    jk = G[:, :, :3, 3]
    if not joints_path:
        jk = jk.detach()
    joints = torch.stack([jk[:, e] if e >= 0 else verts[:, -1 - e] for e in joint_map], 1)
    if trans is None:
        if center_idx is not None:
            c = joints[:, center_idx][:, None]
            if not centre_grad:
                c = c.detach()
            joints, verts = joints - c, verts - c
    else:
        joints, verts = joints + trans[:, None], verts + trans[:, None]
    return verts * scale, joints * scale


def _is_zero(a) -> bool:
    return a is None or bool(np.linalg.norm(np.asarray(a, np.float64)) == 0)


def outputs(kind, model, pose_t, betas_t, trans_t, center_idx, *, leak_betas=False, **mut):
    """The layer's outputs on float64 tensors, with its batch-wide rules decided from the values: kind 'smpl' or
    'mano' (model carries side / hands_mean); betas_t / trans_t None = absent."""
    B = pose_t.shape[0]
    mb = _t(model["betas"])[None].expand(B, -1)
    if kind == "smpl":
        unused = betas_t is None or _is_zero(betas_t.detach().numpy())
        parents, joint_map, scale, p = list(model["parents"]), list(range(len(model["parents"]))), 1.0, pose_t
    else:
        unused = betas_t is None
        parents, scale = list(MANO_PARENTS), 1000.0
        jm = list(range(16)) + [-1 - t for t in MANO_TIPS[model["side"]]]
        joint_map = [jm[i] for i in MANO_REORDER]
        p = torch.cat([pose_t[:, :3], _t(model["hands_mean"])[None] + pose_t[:, 3:]], 1)
    if unused:
        b = mb + (betas_t - betas_t.detach()) if (leak_betas and betas_t is not None) else mb
    else:
        b = betas_t
    tr = None if trans_t is None or _is_zero(trans_t.detach().numpy()) else trans_t
    return forward(model, p, b, parents, tr, center_idx, joint_map, scale, **mut)


def vjp(kind, model, pose, betas, trans, center_idx, grad_verts, grad_joints, **mut):
    """pose, betas, trans, cotangents: numpy (None = absent; a None cotangent is zero).
    -> (verts, joints, grad_pose, grad_betas, grad_trans), float64 numpy."""
    pose_t = _t(pose).requires_grad_(True)
    betas_t = None if betas is None or np.asarray(betas).size == 1 else _t(betas).requires_grad_(True)
    trans_t = None if trans is None else _t(trans).requires_grad_(True)
    verts, joints = outputs(kind, model, pose_t, betas_t, trans_t, center_idx, **mut)
    loss = 0.0
    if grad_verts is not None:
        loss = loss + (verts * _t(grad_verts)).sum()
    if grad_joints is not None:
        loss = loss + (joints * _t(grad_joints)).sum()
    inputs = [x for x in (pose_t, betas_t, trans_t) if x is not None]
    grads = list(torch.autograd.grad(loss, inputs, allow_unused=True))
    out = []
    for x in (pose_t, betas_t, trans_t):
        if x is None:
            out.append(None)
            continue
        g = grads.pop(0)
        out.append(np.zeros(tuple(x.shape)) if g is None else g.numpy())
    return (verts.detach().numpy(), joints.detach().numpy(), *out)
