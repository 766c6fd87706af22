"""The datasets' training targets for a whole batch on the GPU (SURVEY.md §8 row f11):

    camera_frame_coords(layer, dataset, ...)   each dataset's get_smpl_coord / get_mano_coord:
                                               data/{Human36M,AMASS,FreiHAND,MuCo,COCO,SURREAL,PW3D}/dataset.py
    Human36MTargets, COCOTargets, MuCoTargets, AMASSTargets, PW3DTargets
                                               the targets and meta of each dataset's __getitem__ for pose2mesh_net and
                                               posenet, with the lift target's rotation and flip (j3d_processing)
    SURREALTargets, FreiHANDTargets            the same for the datasets that take the body model's own joints as
                                               targets (SMPL's 24, MANO's 21) instead of a regressor's

All run in libp2m_b200.so (p2m_camera_frame_coords, p2m_sample_targets, p2m_layer_joint_targets): a prep kernel, the
body model's three launches and a finish kernel per camera-frame call, one more launch for a dataset's assembly.  CUDA
tensors only; nothing is read back to the host, so a call can be captured in a CUDA graph.

The datasets call the body model once per sample, so its quirks apply per sample here: the betas clamp (any
|beta| > 3 -> zeros) and SMPL_Layer's "all-zero betas -> the model's betas" rule are decided for each sample on its
own, and a sample's result does not depend on the rest of the batch.  The reference keeps one layer per gender; a call
takes one layer, so callers group samples by gender.  Deliberate differences from the reference:

  * the root rotation log(R exp(root)) is taken in fp64 with a log map that is accurate near angle 0 and near pi and
    rounded to float32 where the reference stores it; below pi the axis-angle vector is unique and matches
    transforms3d's to rounding, at pi only the rotation is defined;
  * an exactly zero root is the identity rotation (the reference divides 0 / 0 and raises in mat2axangle);
  * the layer must have center_idx None, as every layer the datasets build does.

The 2-D joints come out in image pixels, before the crop and normalisation: feed them to
postprocess.normalize_pose2d (the use_gt_input path) or to inputs.training_pose2d (the datasets' detector noise).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .body_model import ManoLayer, SMPLLayer
from .inputs import augment_tensors

FACE_KPS_VERTEX = (331, 2802, 6262, 3489, 3990)  # lib/smpl.py:22, appended to MuCo's joints
FITTING_THR = 25.0                               # data/Human36M/dataset.py:37, millimetres
JOINT_SETS = {"human36": _lib.P2M_JOINTS_HUMAN36, "coco": _lib.P2M_JOINTS_COCO}


@dataclass(frozen=True)
class _Preset:
    flags: int
    mano: bool = False      # FreiHAND's MANO layer; every other preset takes an SMPL layer
    trans: bool = False     # reads trans
    camera: bool = False    # reads R and t
    extra: tuple = ()       # vertex joints appended to the layer's joints


PRESETS = {
    # Human36M/dataset.py:253-299: rotated root, clamped betas, + R trans + t / 1000 - J_0 + R J_0, mm
    "human36m": _Preset(_lib.P2M_FRAME_ROTATE_ROOT | _lib.P2M_FRAME_CLAMP_BETAS | _lib.P2M_FRAME_H36M_COMPENSATE |
                        _lib.P2M_FRAME_TO_MM, trans=True, camera=True),
    # AMASS/dataset.py:182-213: rotated root, + t, mm
    "amass": _Preset(_lib.P2M_FRAME_ROTATE_ROOT | _lib.P2M_FRAME_ADD_T | _lib.P2M_FRAME_TO_MM, camera=True),
    # FreiHAND/dataset.py:110-134: rotated root, t into the MANO layer, the layer's mm
    "freihand": _Preset(_lib.P2M_FRAME_ROTATE_ROOT | _lib.P2M_FRAME_LAYER_TRANS_T, mano=True, camera=True),
    # MuCo/dataset.py:196-216: clamped betas, trans into the layer, the 5 face-keypoint vertices appended, mm
    "muco": _Preset(_lib.P2M_FRAME_CLAMP_BETAS | _lib.P2M_FRAME_LAYER_TRANS | _lib.P2M_FRAME_TO_MM, trans=True,
                    extra=FACE_KPS_VERTEX),
    # COCO/dataset.py:147-166: clamped betas, mm
    "coco": _Preset(_lib.P2M_FRAME_CLAMP_BETAS | _lib.P2M_FRAME_TO_MM),
    # SURREAL/dataset.py:62-80, PW3D/dataset.py:84-102: trans into the layer, mm
    "surreal": _Preset(_lib.P2M_FRAME_LAYER_TRANS | _lib.P2M_FRAME_TO_MM, trans=True),
    "pw3d": _Preset(_lib.P2M_FRAME_LAYER_TRANS | _lib.P2M_FRAME_TO_MM, trans=True),
}


def _cuda(x, what: str, shape, device=None) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.requires_grad:
        raise ValueError(f"{what} requires grad; the targets are not differentiable")
    if tuple(x.shape) != tuple(shape):
        raise ValueError(f"{what} must be {list(shape)}; got {tuple(x.shape)}")
    if device is not None and x.device != device:
        raise ValueError(f"{what} is on {x.device}, expected {device}")
    return x.contiguous().float()


def camera_frame_coords(layer, dataset: str, pose, betas, trans=None, R=None, t=None):
    """The dataset's get_smpl_coord / get_mano_coord for a batch: -> (mesh [B, V, 3], joints [B, J', 3]) float32.

    layer    an SMPLLayer (every preset but 'freihand') or a ManoLayer ('freihand'), with center_idx None.
    dataset  one of PRESETS: 'human36m', 'amass', 'freihand', 'muco', 'coco', 'surreal', 'pw3d'.
    pose [B, 3 J], betas [B, 10]; trans [B, 3] for 'human36m', 'muco', 'surreal', 'pw3d'; the camera R [B, 3, 3] and
    t [B, 3] for 'human36m', 'amass', 'freihand' (inputs a preset does not read are ignored).
    Units: millimetres (MANO's own millimetres for 'freihand').  J' = the layer's joints, + 5 face keypoints for
    'muco'."""
    if dataset not in PRESETS:
        raise ValueError(f"dataset must be one of {sorted(PRESETS)}; got {dataset!r}")
    p = PRESETS[dataset]
    want = ManoLayer if p.mano else SMPLLayer
    if not isinstance(layer, want):
        raise ValueError(f"the {dataset!r} preset takes a {want.__name__}; got {type(layer).__name__}")
    if layer.center_idx is not None:
        raise ValueError("camera_frame_coords needs a layer with center_idx None, as the datasets build them")
    _lib.cuda_tensor(pose, "pose")
    B, dev = pose.shape[0] if pose.dim() == 2 else -1, pose.device
    if B < 1:
        raise ValueError(f"pose must be [B, {3 * layer.num_joints}] with B > 0; got {tuple(pose.shape)}")
    pose = _cuda(pose, "pose", (B, 3 * layer.num_joints), dev)
    betas = _cuda(betas, "betas", (B, layer.n_betas), dev)
    if p.trans and trans is None:
        raise ValueError(f"the {dataset!r} preset needs trans [B, 3]")
    trans = _cuda(trans, "trans", (B, 3), dev) if p.trans else None
    if p.camera:
        if R is None or t is None:
            raise ValueError(f"the {dataset!r} preset needs the camera R [B, 3, 3] and t [B, 3]")
        R, t = _cuda(R, "R", (B, 3, 3), dev), _cuda(t, "t", (B, 3), dev)
    else:
        R = t = None
    flags = p.flags | (0 if p.mano else _lib.P2M_FRAME_ZERO_BETAS_MODEL)
    lib = _lib.load()
    h = layer.handle(dev.index)
    mesh = torch.empty((B, layer.n_vertex, 3), device=dev, dtype=torch.float32)
    joints = torch.empty((B, layer.n_out_joints + len(p.extra), 3), device=dev, dtype=torch.float32)
    nbytes = lib.p2m_camera_frame_workspace_bytes(h, B)
    ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    extra = (C.c_int32 * max(len(p.extra), 1))(*p.extra)
    _lib.call("p2m_camera_frame_coords", dev, h, flags, pose, betas, trans, R, t, extra, len(p.extra), mesh, joints,
              B, ws, nbytes)
    return mesh, joints


class _SampleTargets:
    """The target side of one dataset's __getitem__ (pose2mesh_net and posenet) for a batch: camera_frame_coords with
    the dataset's preset, then one assembly launch (p2m_sample_targets).  Built once from the SMPL layer, the H36M
    regressor (J_regressor_h36m_correct.npy) and the COCO regressor (J_regressor_coco.npy), both [17, V] (the four
    datasets use the same two files), the input joint set ('human36' or 'coco') and fitting_thr.  A call returns a
    dict of float32 device tensors shaped as the dataloader collates them (J = 17 for human36, 19 for coco):

        mesh [B, V, 3]                  metres, rooted at the Human3.6M pelvis (the annotation's for Human36M, the
                                        regressed one otherwise)
        lift_pose3d [B, J, 3]           coco: the regressed joints + pelvis, neck, rooted at the pelvis;
                                        human36: the Human3.6M joints rooted at joint 0 (mm)
        reg_pose3d [B, 17, 3]           the Human3.6M joints rooted at joint 0 (mm)
        mesh_valid [B, V, 1], lift_pose3d_valid [B, J, 1], reg_pose3d_valid [B, 17, 1]
                                        0 where the dataset's fitting test fails, for the masks it zeroes
        joint_valid [B, J, 1]           posenet's mask
        joint_img [B, J, 2]             image pixels: the dataset's projection of the input set's joints
        fitting_error [B]               the dataset's fitting error (0 where it has none)

    rot [B] (degrees) and flip [B], augm_params' outputs, augment lift_pose3d as j3d_processing does (x, y rotated by
    -rot degrees in float64, then the flip pairs swapped and x negated); None means none, bit for bit the call without
    them.  The other targets are never augmented (data/Human36M/dataset.py:373, the same in every dataset).

    Six launches per call."""

    LAUNCHES = 6
    DATASET = PRESET = None
    FITTING_THR = None

    def __init__(self, layer: SMPLLayer, joint_regressor_h36m, joint_regressor_coco, input_joint_set: str = "human36",
                 fitting_thr: float = None):
        name = type(self).__name__
        if not isinstance(layer, SMPLLayer):
            raise ValueError(f"{name} takes an SMPLLayer; got {type(layer).__name__}")
        if input_joint_set not in JOINT_SETS:
            raise ValueError(f"input_joint_set must be one of {sorted(JOINT_SETS)}; got {input_joint_set!r}")
        V = layer.n_vertex
        host = lambda a: np.ascontiguousarray(  # noqa: E731
            (a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)), dtype=np.float64)
        self.reg_h36m, self.reg_coco = host(joint_regressor_h36m), host(joint_regressor_coco)
        for rname, r in (("joint_regressor_h36m", self.reg_h36m), ("joint_regressor_coco", self.reg_coco)):
            if r.shape != (17, V):
                raise ValueError(f"{rname} must be [17, {V}]; got {tuple(r.shape)}")
        self.layer, self.input_joint_set = layer, input_joint_set
        self.fitting_thr = float(self.FITTING_THR if fitting_thr is None else fitting_thr)
        self.num_joints = 19 if input_joint_set == "coco" else 17
        self._handles = {}

    def handle(self, device_index: int) -> int:
        h = self._handles.get(device_index)
        if h is None:
            dp = C.POINTER(C.c_double)
            out = C.c_void_p()
            _lib.check(_lib.load().p2m_h36m_regressors_create(self.reg_h36m.ctypes.data_as(dp),
                                                              self.reg_coco.ctypes.data_as(dp), self.reg_h36m.shape[1],
                                                              device_index, C.byref(out)),
                       "p2m_h36m_regressors_create")
            h = self._handles[device_index] = out.value
        return h

    def __del__(self):
        try:
            lib = _lib.load()
            for h in self._handles.values():
                lib.p2m_h36m_regressors_destroy(h)
            self._handles = {}
        except Exception:
            pass

    def _assemble(self, mesh_cam, rot, flip, joint_cam=None, f=None, c=None, s=None, t=None, keypoints=None,
                  keypoints_valid=None) -> dict:
        B, dev, V, J = mesh_cam.shape[0], mesh_cam.device, self.layer.n_vertex, self.num_joints
        n_s = 0
        if f is not None:
            f, c = _cuda(f, "f", (B, 2), dev), _cuda(c, "c", (B, 2), dev)
        if joint_cam is not None:
            joint_cam = _cuda(joint_cam, "joint_cam", (B, 17, 3), dev)
        if s is not None:
            _lib.cuda_tensor(s, "s")
            s = s.reshape(-1, 1) if s.dim() == 1 else s          # the reference's np.array(s) broadcasts [1] or [2]
            if s.dim() != 2 or s.shape[1] not in (1, 2):
                raise ValueError(f"s must be [{B}] or [{B}, 2]; got {tuple(s.shape)}")
            s = _cuda(s, "s", (B, s.shape[1]), dev)
            n_s = s.shape[1]
            t = _cuda(t, "t", (B, 2), dev)
            keypoints = _cuda(keypoints, "keypoints", (B, 17, 2), dev)
            keypoints_valid = _cuda(keypoints_valid, "keypoints_valid", (B, 17), dev)
        rot, flip = augment_tensors(rot, flip, B, dev)
        e = lambda *sh: torch.empty(sh, device=dev, dtype=torch.float32)  # noqa: E731
        out = {"mesh": e(B, V, 3), "lift_pose3d": e(B, J, 3), "reg_pose3d": e(B, 17, 3), "mesh_valid": e(B, V, 1),
               "lift_pose3d_valid": e(B, J, 1), "reg_pose3d_valid": e(B, 17, 1), "joint_valid": e(B, J, 1),
               "joint_img": e(B, J, 2), "fitting_error": e(B)}
        _lib.call("p2m_sample_targets", dev, self.handle(dev.index), self.DATASET, JOINT_SETS[self.input_joint_set],
                  C.c_float(self.fitting_thr), mesh_cam, joint_cam, f, c, s, n_s, t, keypoints, keypoints_valid, rot,
                  flip, B, out["mesh"], out["lift_pose3d"], out["reg_pose3d"], out["mesh_valid"],
                  out["lift_pose3d_valid"], out["reg_pose3d_valid"], out["joint_valid"], out["joint_img"],
                  out["fitting_error"])
        return out


class Human36MTargets(_SampleTargets):
    """Human36M.__getitem__'s targets (data/Human36M/dataset.py:301-333,344-418).  A call takes the SMPL parameters
    pose [B, 72], betas [B, 10], trans [B, 3], the camera R [B, 3, 3], t [B, 3], focal f [B, 2], principal point
    c [B, 2] and the annotation's absolute joint_cam [B, 17, 3] (mm).  Fitting test: 25 mm against the annotation;
    zeroes the mesh mask and, for the coco set, the lift mask; joint_valid is lift_pose3d_valid."""

    DATASET, FITTING_THR = _lib.P2M_DATASET_HUMAN36M, FITTING_THR

    def __call__(self, pose, betas, trans, R, t, f, c, joint_cam, rot=None, flip=None) -> dict:
        mesh_cam, _ = camera_frame_coords(self.layer, "human36m", pose, betas, trans, R, t)
        return self._assemble(mesh_cam, rot, flip, joint_cam=joint_cam, f=f, c=c)


class COCOTargets(_SampleTargets):
    """COCO.__getitem__'s targets (data/COCO/dataset.py:182-287).  A call takes the SMPLify fit's pose [B, 72] and
    betas [B, 10], its weak-perspective camera s [B] or [B, 2] and t [B, 2], and the annotation's keypoints [B, 17, 2]
    (image pixels) with keypoints_valid [B, 17].  joint_img = (xy / 1000) s + t.  Fitting test: 3 px in a 64 x 64 crop
    of the input set's box (aspect 1) between the keypoints and the regressed COCO joints, over the visible keypoints
    (none visible: NaN, the sample stays valid); zeroes the mesh, lift and reg masks and posenet's joint_valid."""

    DATASET, FITTING_THR = _lib.P2M_DATASET_COCO, 3.0

    def __call__(self, pose, betas, s, t, keypoints, keypoints_valid, rot=None, flip=None) -> dict:
        mesh_cam, _ = camera_frame_coords(self.layer, "coco", pose, betas)
        return self._assemble(mesh_cam, rot, flip, s=s, t=t, keypoints=keypoints, keypoints_valid=keypoints_valid)


class MuCoTargets(_SampleTargets):
    """MuCo.__getitem__'s targets (data/MuCo/dataset.py:232-330).  A call takes pose [B, 72], betas [B, 10], trans
    [B, 3], focal f [B, 2] and principal point c [B, 2].  joint_img = cam2pixel(joint, f, c).  Fitting test: 45 mm with
    the reference's quirk kept (the Human3.6M-ordered joints handed to a function expecting MuCo's 21, so rooted at row 14
    and permuted by MuCo's names: about 755 mm on a standing pose, INTEGRATION.md); zeroes the mesh, lift and reg masks;
    posenet's joint_valid is all ones."""

    DATASET, FITTING_THR = _lib.P2M_DATASET_MUCO, 45.0

    def __call__(self, pose, betas, trans, f, c, rot=None, flip=None) -> dict:
        mesh_cam, _ = camera_frame_coords(self.layer, "muco", pose, betas, trans)
        return self._assemble(mesh_cam, rot, flip, f=f, c=c)


class AMASSTargets(_SampleTargets):
    """AMASS.__getitem__'s targets (data/AMASS/dataset.py:229-309).  A call takes pose [B, 72], betas [B, 10], the
    camera R [B, 3, 3], t [B, 3], focal f [B, 2] and principal point c [B, 2].  joint_img = cam2pixel(joint / 1000, f,
    c).  No fitting test: every mask is 1, fitting_error 0."""

    DATASET, FITTING_THR = _lib.P2M_DATASET_AMASS, 0.0

    def __call__(self, pose, betas, R, t, f, c, rot=None, flip=None) -> dict:
        mesh_cam, _ = camera_frame_coords(self.layer, "amass", pose, betas, None, R, t)
        return self._assemble(mesh_cam, rot, flip, f=f, c=c)


class PW3DTargets(_SampleTargets):
    """PW3D.__getitem__'s targets (data/PW3D/dataset.py:208-261), the test split of the *_cocoJ_test_3dpw configs.  The
    reference hard-codes the coco input set, so input_joint_set must be 'coco'.  A call takes pose [B, 72], betas
    [B, 10], trans [B, 3], focal f [B, 2] and principal point c [B, 2].  joint_img = cam2pixel(joint, f, c) of the
    regressed COCO joints with pelvis and neck (mm, as MuCo's).  No fitting test and no augmentation (the reference
    hard-codes rot = flip = 0): every mask is 1, fitting_error 0."""

    DATASET, FITTING_THR = _lib.P2M_DATASET_PW3D, 0.0

    def __init__(self, layer: SMPLLayer, joint_regressor_h36m, joint_regressor_coco, input_joint_set: str = "coco"):
        if input_joint_set != "coco":
            raise ValueError(f"PW3DTargets takes the 'coco' input joint set only; got {input_joint_set!r}")
        super().__init__(layer, joint_regressor_h36m, joint_regressor_coco, "coco")

    def __call__(self, pose, betas, trans, f, c) -> dict:
        mesh_cam, _ = camera_frame_coords(self.layer, "pw3d", pose, betas, trans)
        return self._assemble(mesh_cam, None, None, f=f, c=c)


class _LayerJointTargets:
    """The target side of SURREAL's and FreiHAND's __getitem__ for a batch: camera_frame_coords with the dataset's
    preset, then one assembly launch (p2m_layer_joint_targets).  These datasets take the layer's own joints (J = 24
    SMPL joints, 21 MANO joints) as both the lift and the regression target, so no regressor is needed.  A call returns
    the keys of _SampleTargets, float32 device tensors:

        mesh [B, V, 3]                  metres, (mesh - joint 0) / 1000 in float32
        lift_pose3d, reg_pose3d [B, J, 3]
                                        the joints rooted at joint 0 in float32 (mm)
        mesh_valid [B, V, 1], lift_pose3d_valid, reg_pose3d_valid, joint_valid [B, J, 1]
                                        all ones: neither dataset has a fitting test
        joint_img [B, J, 2]             SURREAL only: cam2pixel of the absolute joints (image pixels)
        fitting_error [B]               0

    Six launches per call."""

    LAUNCHES = 6
    DATASET = LAYER = None

    def __init__(self, layer):
        name = type(self).__name__
        if not isinstance(layer, self.LAYER):
            raise ValueError(f"{name} takes a {self.LAYER.__name__}; got {type(layer).__name__}")
        if layer.center_idx is not None:
            raise ValueError(f"{name} needs a layer with center_idx None, as the datasets build them")
        self.layer, self.num_joints = layer, layer.n_out_joints

    def _assemble(self, mesh_cam, joint_cam, f=None, c=None, rot=None, flip=None) -> dict:
        """The assembly alone, on camera-frame mesh_cam [B, V, 3] and joint_cam [B, J, 3] (mm)."""
        _lib.cuda_tensor(mesh_cam, "mesh_cam")
        if mesh_cam.dim() != 3 or mesh_cam.shape[2] != 3 or mesh_cam.shape[0] < 1 or mesh_cam.shape[1] < 1:
            raise ValueError(f"mesh_cam must be [B, V, 3] with B, V > 0; got {tuple(mesh_cam.shape)}")
        B, V, J, dev = mesh_cam.shape[0], mesh_cam.shape[1], self.num_joints, mesh_cam.device
        mesh_cam = _cuda(mesh_cam, "mesh_cam", (B, V, 3), dev)
        joint_cam = _cuda(joint_cam, "joint_cam", (B, J, 3), dev)
        surreal = self.DATASET == _lib.P2M_DATASET_SURREAL
        if surreal:
            f, c = _cuda(f, "f", (B, 2), dev), _cuda(c, "c", (B, 2), dev)
        rot, flip = augment_tensors(rot, flip, B, dev)
        e = lambda *sh: torch.empty(sh, device=dev, dtype=torch.float32)  # noqa: E731
        out = {"mesh": e(B, V, 3), "lift_pose3d": e(B, J, 3), "reg_pose3d": e(B, J, 3), "mesh_valid": e(B, V, 1),
               "lift_pose3d_valid": e(B, J, 1), "reg_pose3d_valid": e(B, J, 1), "joint_valid": e(B, J, 1)}
        if surreal:
            out["joint_img"] = e(B, J, 2)
        out["fitting_error"] = e(B)
        _lib.call("p2m_layer_joint_targets", dev, self.DATASET, mesh_cam, joint_cam, V, J, f, c, rot, flip, B,
                  out["mesh"], out["lift_pose3d"], out["reg_pose3d"], out["mesh_valid"], out["lift_pose3d_valid"],
                  out["reg_pose3d_valid"], out["joint_valid"], out.get("joint_img"), out["fitting_error"])
        return out


class SURREALTargets(_LayerJointTargets):
    """SURREAL.__getitem__'s targets (data/SURREAL/dataset.py:143-203), 24 SMPL joints rooted at joint 0.  A call
    takes pose [B, 72], betas [B, 10], trans [B, 3], focal f [B, 2] and principal point c [B, 2]; joint_img =
    cam2pixel(joint, f, c) of the absolute joints, in fp64 and rounded once.  rot [B] (degrees) and flip [B],
    augm_params' outputs, augment lift_pose3d as j3d_processing does with SMPL's flip pairs.  The reference's quirk is
    kept: reg_pose3d is the same augmented array (both targets are its reassigned joint_coord_cam), while the mesh is
    never augmented.  posenet_smplJ_train_surreal flips (AUG.flip True) but PoseNet reads only lift_pose3d; the
    pose2mesh SURREAL configs, which read reg_pose3d, never augment."""

    DATASET, LAYER = _lib.P2M_DATASET_SURREAL, SMPLLayer

    def __call__(self, pose, betas, trans, f, c, rot=None, flip=None) -> dict:
        mesh_cam, joint_cam = camera_frame_coords(self.layer, "surreal", pose, betas, trans)
        return self._assemble(mesh_cam, joint_cam, f, c, rot, flip)


class FreiHANDTargets(_LayerJointTargets):
    """FreiHAND.__getitem__'s targets (data/FreiHAND/dataset.py:139-192), 21 MANO joints (the tips appended) rooted at
    joint 0, the wrist.  A call takes pose [B, 48], betas [B, 10] and the camera R [B, 3, 3], t [B, 3].  No joint_img
    (the reference's projection is commented out and its input is always the detection) and no augmentation (the
    reference hard-codes rot = flip = 0)."""

    DATASET, LAYER = _lib.P2M_DATASET_FREIHAND, ManoLayer

    def __call__(self, pose, betas, R, t) -> dict:
        mesh_cam, joint_cam = camera_frame_coords(self.layer, "freihand", pose, betas, None, R, t)
        return self._assemble(mesh_cam, joint_cam)
