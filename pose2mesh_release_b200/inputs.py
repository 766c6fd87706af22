"""The datasets' network inputs for a whole training batch on the GPU (SURVEY.md §8 row f12):

    synthesize_pose(joints, area)           lib/noise_utils.py:17-285, the COCO joints' synthetic detector errors
    Human36MErrorModel.generate_syn_error   data/Human36M/dataset.py:143-155, the Human3.6M joints' error model
    training_pose2d(joints_px, ...)         the train branch of the datasets' replace_joint_img with the crop and
                                            normalisation around it (data/Human36M/dataset.py:359-392,436-445); with
                                            box_joints and noise=False, the test split's branch (:446-452); with rot /
                                            flip, the sample's rotation and flip (lib/aug_utils.py:33-64,140-195);
                                            the 'smpl' / 'mano' sets are SURREAL's, FreiHAND's and 3DPW's noise-free
                                            crop (data/SURREAL/dataset.py:143-186, data/FreiHAND/dataset.py:157-176)
    augm_params(B, flip, rotate_factor)     lib/aug_utils.py:98-117, each sample's flip and rotation

All run in libp2m_b200.so (p2m_synthesize_pose, p2m_h36m_syn_error, p2m_training_pose2d_augmented,
p2m_augm_params), one launch per call, no workspace and no host synchronisation, so a call can be captured in a CUDA
graph.  CUDA tensors only.

The random stream is the library's counter-based rule (include/p2m_b200.h): `seed` is an int64 [2] tensor on the
inputs' device, read by the kernel; when it is None it is drawn from torch's generator, so torch.manual_seed
reproduces a run.  A sample's output depends only on its own inputs, its batch index and the seed.  The outputs follow
the reference's distributions, not its numpy / random streams.  Deliberate differences (INTEGRATION.md): where the
reference's miss candidate list ends up empty after it drew one to three inv-source survivors it raises, here the miss
candidate is absent; the crop-space area is (scale * w) * (scale * h) of the box, the reference's rot-0 affine map of
its corners to rounding.
"""
from __future__ import annotations

import math

import torch

from . import _lib
from .postprocess import INPUT_SHAPE

NUM_KPS = 17
AREA_BOXES = {"tight": _lib.P2M_AREA_TIGHT, "crop": _lib.P2M_AREA_CROP}
JOINT_SETS = {"human36": _lib.P2M_JOINTS_HUMAN36, "coco": _lib.P2M_JOINTS_COCO, "smpl": _lib.P2M_JOINTS_SMPL,
              "mano": _lib.P2M_JOINTS_MANO}
LAYER_JOINTS = {"smpl": 24, "mano": 21}   # the sets that take no detector noise


def _cuda(x, what: str, device=None) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.requires_grad:
        raise ValueError(f"{what} requires grad; the training inputs are not differentiable")
    if device is not None and x.device != device:
        raise ValueError(f"{what} is on {x.device}, expected {device}")
    return x.contiguous().float()


def _seed(seed, device) -> torch.Tensor:
    if seed is None:
        return torch.empty(2, dtype=torch.int64, device=device).random_()
    _lib.cuda_tensor(seed, "seed")
    if seed.dtype != torch.int64 or tuple(seed.shape) != (2,) or seed.device != device:
        raise ValueError(f"seed must be an int64 [2] tensor on {device}; got {seed.dtype} {tuple(seed.shape)} on "
                         f"{seed.device}")
    return seed.contiguous()


def synthesize_pose(joints: torch.Tensor, area: torch.Tensor, seed: torch.Tensor = None) -> torch.Tensor:
    """synthesize_pose(joints, area, num_overlap=0) for a batch: joints [B, 17, 3] (x, y, visibility) in crop pixels,
    area [B] (the crop-space box area) -> [B, 17, 3] float32 rows (x, y, 1), or (0, 0, 0) where every candidate error
    was absent."""
    _lib.cuda_tensor(joints, "joints")
    dev = joints.device
    j = _cuda(joints, "joints", dev)
    if j.dim() != 3 or j.shape[1:] != (NUM_KPS, 3) or j.shape[0] < 1:
        raise ValueError(f"joints must be [B, 17, 3] with B > 0; got {tuple(joints.shape)}")
    B = j.shape[0]
    a = _cuda(area, "area", dev)
    if tuple(a.shape) != (B,):
        raise ValueError(f"area must be [{B}]; got {tuple(area.shape)}")
    s = _seed(seed, dev)
    out = torch.empty_like(j)
    _lib.call("p2m_synthesize_pose", dev, j, a, s, B, out)
    return out


class Human36MErrorModel:
    """The Human3.6M joints' synthetic detector error (Chang et al.'s statistics, which the reference ships as
    data/Human36M/noise_stats.py): error_distribution is that list of dicts {'Joint', 'mean': (x, y), 'std': (x, y),
    'weight'}, joint_names the dataset's joint order (Human36M.human36_joints_name), which the table is sorted by as
    get_stat does.  Every name must have exactly one entry, finite, with std >= 0 and 0 <= weight <= 1."""

    def __init__(self, error_distribution, joint_names):
        names = list(joint_names)
        if len(names) != NUM_KPS:
            raise ValueError(f"joint_names must name {NUM_KPS} joints; got {len(names)}")
        table = (_lib.H36MError * NUM_KPS)()
        for i, name in enumerate(names):
            hits = [ed for ed in error_distribution if ed.get("Joint") == name]
            if len(hits) != 1:
                raise ValueError(f"error_distribution must hold exactly one entry for {name!r}; found {len(hits)}")
            ed = hits[0]
            try:
                mean = [float(v) for v in ed["mean"]]
                std = [float(v) for v in ed["std"]]
                weight = float(ed["weight"])
            except (KeyError, TypeError, ValueError) as e:
                raise ValueError(f"error_distribution entry {name!r} needs 'mean', 'std' (2 each) and 'weight'") from e
            if len(mean) != 2 or len(std) != 2:
                raise ValueError(f"error_distribution entry {name!r}: mean and std take two values")
            if not all(math.isfinite(v) for v in mean + std + [weight]) or min(std) < 0 or not 0 <= weight <= 1:
                raise ValueError(f"error_distribution entry {name!r} must be finite with std >= 0 and "
                                 f"0 <= weight <= 1")
            table[i].mean[:], table[i].std[:], table[i].weight = mean, std, weight
        self.joint_names = tuple(names)
        self.table = table

    def generate_syn_error(self, B: int, seed: torch.Tensor = None, device=None) -> torch.Tensor:
        """The raw noise of B samples, [B, 17, 2] float32 (pixels of a 256-pixel crop), on seed's device (else
        `device`, else the current CUDA device)."""
        if B < 1:
            raise ValueError(f"B must be positive; got {B}")
        dev = _device(seed, device)
        s = _seed(seed, dev)
        out = torch.empty((B, NUM_KPS, 2), device=dev, dtype=torch.float32)
        _lib.call("p2m_h36m_syn_error", dev, self.table, s, B, out)
        return out


def _device(seed, device) -> torch.device:
    dev = seed.device if isinstance(seed, torch.Tensor) else torch.device(device or "cuda", torch.cuda.current_device())
    if dev.index is None:
        dev = torch.device(dev.type, torch.cuda.current_device())
    return dev


def augm_params(B: int, flip: bool, rotate_factor: float, seed: torch.Tensor = None, device=None):
    """augm_params(is_train=True) for B samples under cfg.AUG.flip = flip and cfg.AUG.rotate_factor = rotate_factor:
    -> (flip int32 [B], rot float32 [B] degrees) on seed's device (else `device`, else the current CUDA device).  flip is
    1 with probability 1/2 when enabled; rot is clip(N(0, 1) rotate_factor, +-2 rotate_factor), then 0 with probability
    1/2.  The draws come from the augmentation's own streams: the same seed tensor can drive training_pose2d's noise
    without correlating the two.  Pass both results to training_pose2d and to the targets' call."""
    if not isinstance(B, int) or B < 1:
        raise ValueError(f"B must be a positive int; got {B!r}")
    rf = float(rotate_factor)
    if not math.isfinite(rf) or rf < 0:
        raise ValueError(f"rotate_factor must be finite and >= 0; got {rotate_factor!r}")
    dev = _device(seed, device)
    s = _seed(seed, dev)
    f = torch.empty(B, device=dev, dtype=torch.int32)
    r = torch.empty(B, device=dev, dtype=torch.float32)
    _lib.call("p2m_augm_params", dev, B, 1 if flip else 0, rf, s, f, r)
    return f, r


def augment_tensors(rot, flip, B: int, dev):
    """rot [B] float and flip [B] (any integer or bool dtype) as the kernels read them; either may be None."""
    if rot is not None:
        _lib.cuda_tensor(rot, "rot")
        if tuple(rot.shape) != (B,) or rot.device != dev or not rot.is_floating_point():
            raise ValueError(f"rot must be a float [{B}] tensor on {dev}; got {rot.dtype} {tuple(rot.shape)} on "
                             f"{rot.device}")
        rot = rot.contiguous().float()
    if flip is not None:
        _lib.cuda_tensor(flip, "flip")
        if tuple(flip.shape) != (B,) or flip.device != dev or flip.is_floating_point() or flip.is_complex():
            raise ValueError(f"flip must be an integer [{B}] tensor on {dev}; got {flip.dtype} {tuple(flip.shape)} "
                             f"on {flip.device}")
        flip = (flip != 0).to(torch.int32).contiguous()
    return rot, flip


def training_pose2d(joints_px: torch.Tensor, input_joint_set: str, *, noise: bool = True,
                    error_model: Human36MErrorModel = None, area_box: str = "tight", box_joints: torch.Tensor = None,
                    seed: torch.Tensor = None, input_shape=INPUT_SHAPE, rot: torch.Tensor = None,
                    flip: torch.Tensor = None, flip_before_noise: bool = False) -> torch.Tensor:
    """A training batch's pose2d: joints_px [B, J, 2] image pixels (Human36MTargets' joint_img) -> [B, J, 2].

    The crop box comes from box_joints [B, Jb, 2] (the ground-truth joints, for detections; default joints_px), each
    joint is mapped into the input_shape (height, width) crop, then, with noise=True, input_joint_set 'coco' (J = 19:
    the 17 COCO joints, pelvis, neck) puts rows 0-16 through synthesize_pose with every joint visible and the area of
    area_box ('tight': the joints' tight box, as Human3.6M, COCO and AMASS do; 'crop': the processed box, as MuCo
    does), and 'human36' (J = 17) adds error_model's noise scaled from 256 pixels to the crop.  Last, / input size and
    zero mean, unit std per pose.  With noise=False the result equals postprocess.normalize_pose2d(joints_px) bit for
    bit when box_joints is None.

    rot [B] (degrees) and flip [B] are augm_params' outputs (None: no rotation / flip, bit for bit the call without
    them).  The rotation goes into the crop's affine map (get_affine_transform); the flip is x -> input_w - x - 1 and
    the joint set's flip pairs swapped, after the noise as Human3.6M, COCO and AMASS do, or with
    flip_before_noise=True before it, in float64 on the crop map's output, as MuCo's j2d_processing does.

    input_joint_set 'smpl' (J = 24, SURREAL) and 'mano' (J = 21, FreiHAND) take noise=False: their inputs are the 2-D
    joints themselves.  'mano' has no flip pairs, so it takes no flip.  SURREAL's j2d_processing flips in the joints'
    own dtype: its float32 detections flip after the crop is rounded (flip_before_noise=False), the float64
    cam2pixel joints of use_gt_input before (flip_before_noise=True)."""
    if input_joint_set not in JOINT_SETS:
        raise ValueError(f"input_joint_set must be one of {sorted(JOINT_SETS)}; got {input_joint_set!r}")
    if area_box not in AREA_BOXES:
        raise ValueError(f"area_box must be one of {sorted(AREA_BOXES)}; got {area_box!r}")
    _lib.cuda_tensor(joints_px, "joints_px")
    dev = joints_px.device
    x = _cuda(joints_px, "joints_px", dev)
    if x.dim() != 3 or x.shape[2] != 2 or x.shape[0] < 1 or not 1 <= x.shape[1] <= 32:
        raise ValueError(f"joints_px must be [B, J, 2] with B > 0 and J <= 32; got {tuple(joints_px.shape)}")
    B, J = x.shape[:2]
    if input_joint_set in LAYER_JOINTS:
        if noise:
            raise ValueError(f"the {input_joint_set!r} joint set has no detector noise: pass noise=False")
        if J != LAYER_JOINTS[input_joint_set]:
            raise ValueError(f"the {input_joint_set!r} joint set takes {LAYER_JOINTS[input_joint_set]} joints; got "
                             f"J = {J}")
        if input_joint_set == "mano" and flip is not None:
            raise ValueError("the 'mano' joint set has no flip pairs: flip must be None")
    mode = _lib.P2M_NOISE_NONE
    table = None
    if noise and input_joint_set == "coco":
        if J < NUM_KPS:
            raise ValueError(f"the COCO noise needs the 17 COCO joints first; got J = {J}")
        mode = _lib.P2M_NOISE_COCO
    elif noise:
        if error_model is None:
            raise ValueError("the 'human36' joint set's noise needs error_model (a Human36MErrorModel)")
        if J != NUM_KPS:
            raise ValueError(f"the Human3.6M noise takes 17 joints; got J = {J}")
        mode, table = _lib.P2M_NOISE_H36M, error_model.table
    nb = 0
    if box_joints is not None:
        bj = _cuda(box_joints, "box_joints", dev)
        if bj.dim() != 3 or bj.shape[0] != B or bj.shape[2] != 2 or not 1 <= bj.shape[1] <= 32:
            raise ValueError(f"box_joints must be [{B}, Jb, 2] with Jb <= 32; got {tuple(box_joints.shape)}")
        box_joints, nb = bj, bj.shape[1]
    rot, flip = augment_tensors(rot, flip, B, dev)
    if flip is not None and input_joint_set in ("coco", "human36") and \
            (J != NUM_KPS if input_joint_set == "human36" else J < NUM_KPS):
        raise ValueError(f"a flip of the {input_joint_set!r} joints needs "
                         f"{'17' if input_joint_set == 'human36' else 'at least 17'} joints; got J = {J}")
    s = _seed(seed, dev) if mode != _lib.P2M_NOISE_NONE else None
    out = torch.empty_like(x)
    _lib.call("p2m_training_pose2d_augmented", dev, x, B, J, box_joints, nb, mode, AREA_BOXES[area_box], table, s,
              int(input_shape[0]), int(input_shape[1]), rot, flip, JOINT_SETS[input_joint_set],
              1 if flip_before_noise else 0, out)
    return out
