"""Float64 numpy restatement of the two body-model forwards Pose2Mesh builds its target meshes with:

    smpl_forward   smplpytorch/smplpytorch/pytorch/smpl_layer.py:65-158  (SMPL_Layer.forward)
    mano_forward   manopth/manopth/manolayer.py  (ManoLayer.forward, use_pca=False, axis-angle root and joints)

Models are dicts of tests/body_models.py.  The keyword switches of `_forward` exist for the tests that show the
error bound has teeth (a mutated oracle must fail it); the public functions never set them.
"""
from __future__ import annotations

import numpy as np

from body_models import MANO_PARENTS, MANO_REORDER, MANO_TIPS


def rodrigues(theta: np.ndarray) -> np.ndarray:
    """rodrigues_layer.batch_rodrigues: [N, 3] -> [N, 3, 3].  angle = |theta + 1e-8|, axis = theta / angle, half-angle
    quaternion, quat2mat (which renormalises the quaternion)."""
    theta = np.asarray(theta, np.float64)
    angle = np.linalg.norm(theta + 1e-8, axis=1, keepdims=True)
    axis = theta / angle
    half = angle * 0.5
    q = np.concatenate([np.cos(half), np.sin(half) * axis], 1)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z,
                     2 * w * z + 2 * x * y, w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x,
                     2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z, w * w - x * x - y * y + z * z], 1).reshape(-1, 3, 3)


def _forward(model, pose, betas_used, parents, trans, center_idx, joint_map, scale, *, pose_blend=True,
             basis_round=None):
    """The shared body of both layers: v_shaped, v_posed, the kinematic chain, A_j, skinning, output joints
    (joint_map: entry >= 0 a kinematic joint, < 0 vertex -1 - e), translation / centring, scale."""
    pose = np.asarray(pose, np.float64)
    B, J = pose.shape[0], len(parents)
    f64 = lambda k: np.asarray(model[k], np.float64)  # noqa: E731
    shapedirs, posedirs = f64("shapedirs"), f64("posedirs")
    if basis_round is not None:
        shapedirs, posedirs = basis_round(shapedirs), basis_round(posedirs)
    R = rodrigues(pose.reshape(-1, 3)).reshape(B, J, 3, 3)
    pose_map = (R[:, 1:] - np.eye(3)).reshape(B, -1)                       # subtract_flat_id
    V = shapedirs.shape[0]
    v_shaped = f64("v_template")[None] + (shapedirs.reshape(3 * V, -1) @ betas_used.T).T.reshape(B, V, 3)
    jts = f64("J_regressor")[None] @ v_shaped
    v_posed = v_shaped + ((posedirs.reshape(3 * V, -1) @ pose_map.T).T.reshape(B, V, 3) if pose_blend else 0.0)
    G = np.zeros((B, J, 4, 4))
    G[:, :, 3, 3] = 1.0
    for j in range(J):                                                     # th_with_zeros / matmul in parent order
        rel = np.zeros((B, 4, 4))
        rel[:, :3, :3], rel[:, 3, 3] = R[:, j], 1.0
        p = parents[j]
        rel[:, :3, 3] = jts[:, j] - (jts[:, p] if p >= 0 else 0.0)
        G[:, j] = rel if p < 0 else G[:, p] @ rel
    A = G.copy()
    A[:, :, :3, 3] -= np.einsum("bjrc,bjc->bjr", G[:, :, :3, :3], jts)     # G - pack(G [J; 0])
    T = (f64("weights")[None] @ A.reshape(B, J, 16)).reshape(B, V, 4, 4)
    verts = np.einsum("bvrc,bvc->bvr", T[:, :, :3, :3], v_posed) + T[:, :, :3, 3]
    jk = G[:, :, :3, 3]
    joints = np.stack([jk[:, e] if e >= 0 else verts[:, -1 - e] for e in joint_map], 1)
    if trans is None or np.linalg.norm(trans) == 0:
        if center_idx is not None:
            c = joints[:, center_idx][:, None]
            joints, verts = joints - c, verts - c
    else:
        t = np.asarray(trans, np.float64)[:, None]
        joints, verts = joints + t, verts + t
    return verts * scale, joints * scale


def smpl_betas(model, betas, B, *, model_fallback=True):
    """SMPL_Layer's rule: absent or all-zero betas (of the whole batch) -> the model's stored betas."""
    if betas is None or (model_fallback and np.linalg.norm(betas) == 0):
        return np.repeat(np.asarray(model["betas"], np.float64)[None], B, 0)
    return np.asarray(betas, np.float64)


def mano_betas(model, betas, B):
    """ManoLayer's rule: absent or single-element betas -> the model's stored betas; anything else is used as given."""
    if betas is None or np.asarray(betas).size == 1:
        return np.repeat(np.asarray(model["betas"], np.float64)[None], B, 0)
    return np.asarray(betas, np.float64)


def smpl_forward(model, pose, betas=None, trans=None, center_idx=None, **mut):
    """-> verts [B, 6890, 3], joints [B, 24, 3] in metres (float64)."""
    B, J = pose.shape[0], len(model["parents"])
    b = smpl_betas(model, betas, B, model_fallback=mut.pop("model_fallback", True))
    return _forward(model, pose, b, list(model["parents"]), trans, center_idx, list(range(J)), 1.0, **mut)


def mano_forward(model, pose, betas=None, trans=None, center_idx=None, *, hands_mean=True, tips=None, **mut):
    """-> verts [B, 778, 3], joints [B, 21, 3] in millimetres (float64).  pose [B, 48]: root + 45 finger values, to
    which the model's hands_mean is added (zero for flat_hand_mean)."""
    pose = np.array(pose, np.float64)
    if hands_mean:
        pose[:, 3:] = np.asarray(model["hands_mean"], np.float64)[None] + pose[:, 3:]
    tips = MANO_TIPS[model["side"]] if tips is None else tips
    jm = list(range(16)) + [-1 - t for t in tips]
    joint_map = [jm[i] for i in MANO_REORDER]
    b = mano_betas(model, betas, pose.shape[0])
    return _forward(model, pose, b, list(MANO_PARENTS), trans, center_idx, joint_map, 1000.0, **mut)


def tf32_round(a: np.ndarray) -> np.ndarray:
    """Round to TF32 (10 explicit mantissa bits, nearest-even) -- the tensor-core input precision the layer avoids."""
    x = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    x = (x + 0xFFF + ((x >> 13) & 1)) & ~np.uint64(0x1FFF)
    return x.astype(np.uint32).view(np.float32).astype(np.float64)
