"""The body models Pose2Mesh builds its target meshes with, for a whole batch on the GPU (SURVEY.md §8 row f6):

    SMPLLayer   smplpytorch/smplpytorch/pytorch/smpl_layer.py:65-158  (SMPL_Layer.forward)
    ManoLayer   manopth/manopth/manolayer.py  (ManoLayer.forward as lib/_mano.py:37 configures it: use_pca=False,
                axis-angle root and joints, either flat_hand_mean, either side)

Same forward signatures, same th_* buffer names and the same outputs as the reference layers: SMPL in metres, MANO
in millimetres with the five tip vertices appended and the 21-joint reorder.  The reference's batch-wide quirks are
kept, and decided on the device, so a forward never synchronises with the host and can be captured in a CUDA graph:

  * SMPL betas: absent, or the whole batch's betas all zero -> every sample uses the model's stored th_betas.
  * MANO betas: absent or a single-element tensor -> th_betas; an explicit all-zero [B, 10] batch is used as given.
  * trans is added when the batch's trans holds any non-zero (or NaN) value; otherwise, with center_idx set,
    everything is re-centred on that output joint.

Everything runs in libp2m_b200.so (p2m_body_model_*): fp32 on the CUDA cores, three kernel launches per forward.
CUDA tensors only; inputs are made contiguous float32.

Gradients are opt-in: with ``differentiable=True`` (constructor or from_reference) the outputs come from an autograd
Function whose backward is p2m_body_model_backward (five launches), the gradient the reference layer's autograd gives
with respect to pose, betas and trans (not the model buffers).  The forward runs the same launches, so its outputs are
bitwise those of the default layer.  Betas the forward does not use (an all-zero SMPL batch) get a zero gradient;
absent or single-element betas get none.  Double backward is not supported.  Deliberate differences from the reference
layers:

  * by default forward only: an input that requires grad raises, so a layer used to build targets never records a
    graph by accident;
  * a single-element betas tensor counts as absent for SMPL as well (the reference raises for a non-zero one);
  * the zero tests compare every value with 0, where the reference's float32 norm also calls values below ~1e-19
    zero (their squares underflow).

Build a layer from the model's arrays, or with ``from_reference(layer)`` from an already-loaded reference layer
(loading the licence-gated .pkl needs chumpy and stays with the reference).  The th_* buffers are the model: native
handles are built from them lazily, one per device, and rebuilt after load_state_dict or refresh().
"""
from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import torch
from torch.autograd.function import once_differentiable
from torch.nn import Module

from . import _lib

MANO_PARENTS = (-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14)  # manolayer.py lev1/2/3_idxs
MANO_TIPS = {"right": (745, 317, 444, 556, 673), "left": (745, 317, 445, 556, 673)}
MANO_REORDER = (0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20)


def _host(a, shape=None, dtype=np.float32) -> np.ndarray:
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().numpy()
    a = np.ascontiguousarray(np.asarray(a, dtype=dtype))
    return a if shape is None else np.ascontiguousarray(a.reshape(shape))


class _BodyModel(Module):
    """The reference's th_* buffers (the model itself), the kinematic tree and output-joint map, and per-device native
    handles.  A handle is built from the buffers when the layer first runs on a device; load_state_dict rebuilds it,
    and after editing a buffer in place call refresh()."""

    def __init__(self, v_template, shapedirs, posedirs, J_regressor, weights, parents, betas, pose_mean, joint_map,
                 scale, center_idx, differentiable=False):
        super().__init__()
        self.differentiable = bool(differentiable)
        vt = _host(v_template)
        V = vt.size // 3
        J = len(parents)
        sd = _host(shapedirs)
        S = sd.size // (V * 3)
        self.n_vertex, self.num_joints, self.n_betas = V, J, S
        self._parents = _host(parents, (J,), np.int32)
        self._joint_map = _host(joint_map, (-1,), np.int32)
        self.n_out_joints = len(self._joint_map)
        self.scale = float(scale)
        self.center_idx = center_idx
        t = lambda a, shape: torch.from_numpy(_host(a, shape).copy())  # noqa: E731
        self.register_buffer("th_betas", t(betas, (1, S)))
        self.register_buffer("th_shapedirs", t(sd, (V, 3, S)))
        self.register_buffer("th_posedirs", t(posedirs, (V, 3, 9 * (J - 1))))
        self.register_buffer("th_v_template", t(vt, (1, V, 3)))
        self.register_buffer("th_J_regressor", t(J_regressor, (J, V)))
        self.register_buffer("th_weights", t(weights, (V, J)))
        if pose_mean is not None:  # MANO's hands_mean, added to the 45 finger values
            self.register_buffer("th_hands_mean", t(pose_mean, (1, 3 * (J - 1))))
        self.kintree_parents = [int(p) for p in self._parents]
        self._handles = {}
        self._lock = threading.Lock()

    # ------------------------------------------------------------------------------------------- native handle
    def handle(self, device_index: int) -> int:
        with self._lock:
            h = self._handles.get(device_index)
            if h is None:
                V, J, S = self.n_vertex, self.num_joints, self.n_betas
                a = {"v_template": _host(self.th_v_template, (V, 3)), "shapedirs": _host(self.th_shapedirs, (V, 3, S)),
                     "posedirs": _host(self.th_posedirs, (V, 3, 9 * (J - 1))),
                     "J_regressor": _host(self.th_J_regressor, (J, V)), "weights": _host(self.th_weights, (V, J)),
                     "model_betas": _host(self.th_betas, (S,)),
                     "pose_mean": _host(self.th_hands_mean, (3 * (J - 1),)) if hasattr(self, "th_hands_mean") else None}
                fp = lambda x: x.ctypes.data_as(_lib.c_float_p) if x is not None else None  # noqa: E731
                d = _lib.BodyModelDesc()
                d.n_vertex, d.n_joint, d.n_betas, d.n_out_joints = V, J, S, self.n_out_joints
                d.v_template, d.shapedirs, d.posedirs = fp(a["v_template"]), fp(a["shapedirs"]), fp(a["posedirs"])
                d.J_regressor, d.weights = fp(a["J_regressor"]), fp(a["weights"])
                d.parents = self._parents.ctypes.data_as(_lib.c_int32_p)
                d.model_betas, d.pose_mean = fp(a["model_betas"]), fp(a["pose_mean"])
                d.joint_map = self._joint_map.ctypes.data_as(_lib.c_int32_p)
                d.scale, d.device = self.scale, device_index
                out = C.c_void_p()
                _lib.check(_lib.load().p2m_body_model_create(C.byref(d), C.byref(out)), "p2m_body_model_create")
                h = out.value
                self._handles[device_index] = h
            return h

    def refresh(self):
        """Drop the native handles, so the next forward on each device rebuilds them from the th_* buffers."""
        with self._lock:
            handles, self._handles = self._handles, {}
        if handles:
            lib = _lib.load()
            for h in handles.values():
                lib.p2m_body_model_destroy(h)

    def _load_from_state_dict(self, *args, **kwargs):
        super()._load_from_state_dict(*args, **kwargs)
        self.refresh()

    def __del__(self):
        try:
            self.refresh()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------- forward
    def _no_grad(self, **tensors):
        if self.differentiable:
            return
        for name, t in tensors.items():
            if isinstance(t, torch.Tensor) and t.requires_grad:
                raise RuntimeError(f"{name} requires grad: this layer is forward only; build it with "
                                   "differentiable=True to differentiate through it, or pass a detached tensor")

    def _prepare(self, pose, betas, trans, pose_width):
        """Check and normalise the inputs (torch ops only, so autograd follows them): -> pose, betas, trans, centre."""
        _lib.cuda_tensor(pose, "the pose")
        if pose.dim() != 2 or pose.shape[1] != pose_width or pose.shape[0] == 0:
            raise ValueError(f"pose must be [B, {pose_width}] with B > 0; got {tuple(pose.shape)}")
        B, dev = pose.shape[0], pose.device
        pose = pose.contiguous().float()
        if betas is not None and betas.numel() == 1:  # the reference's default argument, torch.zeros(1)
            betas = None
        if betas is not None:
            if not betas.is_cuda or betas.device != dev:
                raise RuntimeError(f"betas must be a CUDA tensor on {dev}")
            if tuple(betas.shape) != (B, self.n_betas):
                raise ValueError(f"betas must be [{B}, {self.n_betas}] (one row per pose); got {tuple(betas.shape)}")
            betas = betas.contiguous().float()
        if trans is not None:
            if trans.numel() == 1 and not trans.is_cuda and trans.requires_grad:  # a host scalar to differentiate
                trans = trans.to(dev).reshape(1, 1).expand(B, 3)
            elif trans.numel() == 1 and not trans.is_cuda:  # the default torch.zeros(1), or a host scalar
                value = float(trans)
                trans = None if value == 0.0 else torch.full((B, 3), value, device=dev)
            elif trans.numel() == 1:  # a scalar is broadcast to every coordinate, as the reference does
                trans = trans.reshape(1, 1).expand(B, 3)
        if trans is not None:
            if not trans.is_cuda or trans.device != dev:
                raise RuntimeError(f"trans must be a CUDA tensor on {dev}")
            if tuple(trans.shape) != (B, 3):
                raise ValueError(f"trans must be [{B}, 3]; got {tuple(trans.shape)}")
            trans = trans.contiguous().float()
        center = -1
        if self.center_idx is not None:  # an output joint; negative indices count from the end, as in the reference
            if not -self.n_out_joints <= int(self.center_idx) < self.n_out_joints:
                raise ValueError(f"center_idx {self.center_idx} out of range for {self.n_out_joints} joints")
            center = int(self.center_idx) % self.n_out_joints
        return pose, betas, trans, center

    def _forward_native(self, pose, betas, trans, betas_rule, center):
        B, dev = pose.shape[0], pose.device
        lib = _lib.load()
        h = self.handle(dev.index)
        verts = torch.empty((B, self.n_vertex, 3), device=dev, dtype=torch.float32)
        joints = torch.empty((B, self.n_out_joints, 3), device=dev, dtype=torch.float32)
        nbytes = lib.p2m_body_model_workspace_bytes(h, B)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        _lib.call("p2m_body_model_forward", dev, h, pose, betas, betas_rule, trans, center, verts, joints, B, ws,
                  nbytes)
        return verts, joints

    def _backward_native(self, pose, betas, trans, betas_rule, center, grad_verts, grad_joints, want_betas,
                         want_trans):
        B, dev = pose.shape[0], pose.device
        lib = _lib.load()
        h = self.handle(dev.index)
        f32 = lambda g: None if g is None else g.contiguous().float()  # noqa: E731
        grad_verts, grad_joints = f32(grad_verts), f32(grad_joints)
        grad_pose = torch.empty_like(pose)
        grad_betas = torch.empty_like(betas) if want_betas and betas is not None else None
        grad_trans = torch.empty_like(trans) if want_trans and trans is not None else None
        nbytes = lib.p2m_body_model_backward_workspace_bytes(h, B)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        _lib.call("p2m_body_model_backward", dev, h, pose, betas, betas_rule, trans, center, grad_verts, grad_joints,
                  grad_pose, grad_betas, grad_trans, B, ws, nbytes)
        return grad_pose, grad_betas, grad_trans

    def _run(self, pose, betas, trans, betas_rule, pose_width):
        pose, betas, trans, center = self._prepare(pose, betas, trans, pose_width)
        if self.differentiable:
            return _BodyModelFunction.apply(self, betas_rule, center, pose, betas, trans)
        return self._forward_native(pose, betas, trans, betas_rule, center)


class _BodyModelFunction(torch.autograd.Function):
    """The native forward's outputs, with p2m_body_model_backward as their vector-Jacobian product.  The backward
    recomputes what it needs from the saved inputs; it is not itself differentiable (no double backward)."""

    @staticmethod
    def forward(ctx, layer, betas_rule, center, pose, betas, trans):
        ctx.layer, ctx.betas_rule, ctx.center = layer, betas_rule, center
        ctx.set_materialize_grads(False)  # an unused output passes NULL, not a zero tensor
        ctx.save_for_backward(pose, betas, trans)
        return layer._forward_native(pose, betas, trans, betas_rule, center)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_verts, grad_joints):
        pose, betas, trans = ctx.saved_tensors
        want = ctx.needs_input_grad
        gp, gb, gt = ctx.layer._backward_native(pose, betas, trans, ctx.betas_rule, ctx.center, grad_verts,
                                                grad_joints, want[4], want[5])
        return None, None, None, gp if want[3] else None, gb, gt


class SMPLLayer(_BodyModel):
    """Batched smplpytorch SMPL_Layer on the GPU (forward only unless differentiable=True).

    Arrays in the reference's layouts: v_template [V, 3], shapedirs [V, 3, S], posedirs [V, 3, 9 (J - 1)],
    J_regressor [J, V], weights [V, J], kintree_parents [J], betas [S] (the model's stored betas).  The root's entry
    of kintree_parents is ignored, as SMPL_Layer.forward ignores it (the SMPL pkl stores 2^32 - 1 there)."""

    def __init__(self, v_template, shapedirs, posedirs, J_regressor, weights, kintree_parents, betas,
                 center_idx=None, gender="neutral", differentiable=False):
        # the root's entry is never read by SMPL_Layer.forward; the SMPL pkl's kintree_table stores 2^32 - 1 there
        parents = [-1] + [int(p) for p in list(kintree_parents)[1:]]
        super().__init__(v_template, shapedirs, posedirs, J_regressor, weights, parents, betas, None,
                         list(range(len(parents))), 1.0, center_idx, differentiable)
        self.gender = gender

    @classmethod
    def from_reference(cls, layer, differentiable=False) -> "SMPLLayer":
        """Copy the buffers of an already-loaded smplpytorch SMPL_Layer."""
        return cls(layer.th_v_template, layer.th_shapedirs, layer.th_posedirs, layer.th_J_regressor, layer.th_weights,
                   list(layer.kintree_parents), layer.th_betas, center_idx=layer.center_idx,
                   gender=getattr(layer, "gender", "neutral"), differentiable=differentiable)

    def forward(self, th_pose_axisang, th_betas=torch.zeros(1), th_trans=torch.zeros(1)):
        """th_pose_axisang [B, 3 J] -> verts [B, V, 3], joints [B, J, 3] (metres)."""
        self._no_grad(th_pose_axisang=th_pose_axisang, th_betas=th_betas, th_trans=th_trans)
        return self._run(th_pose_axisang, th_betas, th_trans, _lib.P2M_BETAS_ZERO_MEANS_MODEL, 3 * self.num_joints)


class ManoLayer(_BodyModel):
    """Batched manopth ManoLayer on the GPU (forward only unless differentiable=True) in the configuration Pose2Mesh uses (lib/_mano.py:37):
    use_pca=False, axis-angle root and joints, either flat_hand_mean, either side.  The rest of ManoLayer is not
    supported, and Pose2Mesh uses none of it: use_pca=True, root_rot_mode other than 'axisang' (6-D root),
    joint_rot_mode='rotmat', and a truthy root_palm or share_betas in forward raise ValueError.

    Arrays as SMPLLayer (J = 16), plus hands_mean [45] (ignored with flat_hand_mean).  The kinematic chain is the one
    ManoLayer.forward hard-codes, not a pkl's kintree_table."""

    def __init__(self, v_template, shapedirs, posedirs, J_regressor, weights, betas, hands_mean, center_idx=None,
                 flat_hand_mean=True, side="right", use_pca=False, root_rot_mode="axisang", joint_rot_mode="axisang",
                 ncomps=45, differentiable=False):
        if use_pca:
            raise ValueError("ManoLayer: use_pca=True is not supported (Pose2Mesh uses use_pca=False)")
        if root_rot_mode != "axisang":
            raise ValueError(f"ManoLayer: root_rot_mode={root_rot_mode!r} is not supported (only 'axisang')")
        if joint_rot_mode != "axisang":
            raise ValueError(f"ManoLayer: joint_rot_mode={joint_rot_mode!r} is not supported (only 'axisang')")
        if side not in MANO_TIPS:
            raise ValueError(f"ManoLayer: side must be 'right' or 'left'; got {side!r}")
        mean = np.zeros(45, np.float32) if flat_hand_mean else _host(hands_mean, (45,))
        jm = list(range(16)) + [-1 - t for t in MANO_TIPS[side]]
        super().__init__(v_template, shapedirs, posedirs, J_regressor, weights, MANO_PARENTS, betas, mean,
                         [jm[i] for i in MANO_REORDER], 1000.0, center_idx, differentiable)
        self.side, self.flat_hand_mean, self.use_pca, self.ncomps, self.rot = side, flat_hand_mean, False, 45, 3
        self.root_rot_mode = self.joint_rot_mode = "axisang"

    @classmethod
    def from_reference(cls, layer, differentiable=False) -> "ManoLayer":
        """Copy the buffers of an already-loaded manopth ManoLayer (its th_hands_mean already holds zeros when
        flat_hand_mean)."""
        return cls(layer.th_v_template, layer.th_shapedirs, layer.th_posedirs, layer.th_J_regressor, layer.th_weights,
                   layer.th_betas, layer.th_hands_mean, center_idx=layer.center_idx,
                   flat_hand_mean=bool(layer.flat_hand_mean), side=layer.side, use_pca=bool(layer.use_pca),
                   root_rot_mode=getattr(layer, "root_rot_mode", "axisang"),
                   joint_rot_mode=getattr(layer, "joint_rot_mode", "axisang"), differentiable=differentiable)

    def forward(self, th_pose_coeffs, th_betas=torch.zeros(1), th_trans=torch.zeros(1), root_palm=torch.Tensor([0]),
                share_betas=torch.Tensor([0])):
        """th_pose_coeffs [B, 48] (root + 45 finger values) -> verts [B, 778, 3], joints [B, 21, 3] (millimetres)."""
        if bool(root_palm):
            raise ValueError("ManoLayer: root_palm is not supported (Pose2Mesh does not use it)")
        if bool(share_betas):
            raise ValueError("ManoLayer: share_betas is not supported (Pose2Mesh does not use it)")
        self._no_grad(th_pose_coeffs=th_pose_coeffs, th_betas=th_betas, th_trans=th_trans)
        return self._run(th_pose_coeffs, th_betas, th_trans, _lib.P2M_BETAS_AS_GIVEN, 3 * self.num_joints)
