"""The demo's camera fit on the GPU (SURVEY.md §8 row f7):

    fit_cameras(joints_px, pred_joints3d)     demo/run.py:149-197 optimize_cam_param with lib/models/project_net.py,
                                              for every person of a batch in one launch
    convert_crop_cam_to_orig_img(...)         demo/run.py:24-43

Both run in libp2m_b200.so (p2m_fit_camera, p2m_crop_cam_to_orig); CUDA tensors only.

One deliberate difference: the reference's loss takes target[:, :17] and raises a shape error for any other joint
count; here the first J target rows are used for J predicted joints (J = 17 for the human36 and coco joint sets).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

CROP_SIZE = 500                                          # virtual_crop_size, demo/run.py:211
LR_SCHEDULE = ((0, 0.1), (501, 0.05), (1001, 0.001))    # run.py:163,182-187: lr changes AFTER steps 500 and 1000
N_ITER = 1500


def _cuda(x, what: str) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.requires_grad:
        raise ValueError(f"{what} requires grad; the camera fit is not differentiable")
    return x


def _image_sizes(image_size, batch: int, device) -> torch.Tensor:
    """(width, height) for all people, or a [B, 2] tensor / sequence -> [B, 2] float32 on device."""
    wh = torch.as_tensor(image_size, dtype=torch.float32).to(device).reshape(-1, 2)
    if wh.shape[0] == 1:
        wh = wh.expand(batch, 2)
    if wh.shape[0] != batch:
        raise ValueError(f"image_size must be (width, height) or one pair per person ({batch}); got {tuple(wh.shape)}")
    return wh.contiguous()


def fit_cameras(joints_px: torch.Tensor, pred_joints3d: torch.Tensor, crop_size: int = CROP_SIZE, init=None,
                n_iter: int = N_ITER, lr_schedule=LR_SCHEDULE, image_size=None):
    """Fit the weak-perspective camera (s, tx, ty) of every person as optimize_cam_param does.

    joints_px      [B, Jin, 2 | 3] (or [Jin, 2 | 3]) image pixels; extra columns (confidences) are ignored.  Integer
                   tensors follow the reference's integer arrays (transformed points truncated towards zero), float32
                   tensors take their tight box in float32, everything else in float64, as numpy does.
    pred_joints3d  [B, J, 3] the model's joints (J <= Jin <= 32); the loss uses the first J target rows.
    init           [B, 3] initial cameras, or None: one torch.rand((1, 3)) per person, in order, from the global CPU
                   generator, as constructing one OptimzeCamLayer per person does (project_net.py:12).
    lr_schedule    ((first_step, lr), ...): step i (0-based) runs at the lr of the last phase starting at or before i.
    image_size     (width, height) or [B, 2]: also return ``orig_cam`` = convert_crop_cam_to_orig_img.

    Returns a dict of device tensors: ``cam_param`` [B, 3], ``bbox`` [B, 4] (bbox1, float32), ``target`` [B, Jin, 2]
    (the crop-space targets), ``loss`` [B] (the L1 loss of the final camera) and, with image_size, ``orig_cam`` [B, 4].
    A person whose box the reference rejects (process_bbox returns None) or whose joints hold a NaN gets NaN outputs.
    Nothing is read back to the host, so with ``init`` given a call can be captured in a CUDA graph."""
    squeeze = joints_px.dim() == 2 if isinstance(joints_px, torch.Tensor) else False
    jp, p3 = _cuda(joints_px, "joints_px"), _cuda(pred_joints3d, "pred_joints3d")
    if squeeze:
        jp, p3 = jp.unsqueeze(0), (p3.unsqueeze(0) if p3.dim() == 2 else p3)
    if jp.dim() != 3 or jp.shape[-1] < 2 or p3.dim() != 3 or p3.shape[-1] != 3 or p3.shape[0] != jp.shape[0]:
        raise ValueError(f"joints_px must be [B, Jin, 2|3] and pred_joints3d [B, J, 3]; got {tuple(jp.shape)}, "
                         f"{tuple(p3.shape)}")
    if p3.device != jp.device:
        raise ValueError(f"joints_px is on {jp.device}, pred_joints3d on {p3.device}")
    B, n_in, cols = jp.shape
    J = p3.shape[1]
    if jp.dtype == torch.float32:
        kind = _lib.P2M_CAM_INPUT_F32
    elif jp.is_floating_point():
        kind = _lib.P2M_CAM_INPUT_F64
    else:
        kind = _lib.P2M_CAM_INPUT_INT
    dev = jp.device
    x = jp.to(torch.float64).contiguous()
    p3 = p3.to(torch.float32).contiguous()
    if init is None:
        init = torch.cat([torch.rand((1, 3)) for _ in range(B)])
    else:
        init = torch.as_tensor(init)
        if init.requires_grad:
            raise ValueError("init requires grad; the camera fit is not differentiable")
    init = init.to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()
    if init.shape[0] != B:
        raise ValueError(f"init must be [B, 3] with B = {B}; got {tuple(init.shape)}")
    phases = list(lr_schedule)
    steps = (C.c_int32 * max(len(phases), 1))(*[int(s) for s, _ in phases])
    rates = (C.c_double * max(len(phases), 1))(*[float(r) for _, r in phases])
    out = {"cam_param": torch.empty((B, 3), device=dev, dtype=torch.float32),
           "bbox": torch.empty((B, 4), device=dev, dtype=torch.float32),
           "target": torch.empty((B, n_in, 2), device=dev, dtype=torch.float32),
           "loss": torch.empty((B,), device=dev, dtype=torch.float32)}
    wh = orig = None
    if image_size is not None:
        wh = _image_sizes(image_size, B, dev)
        orig = out["orig_cam"] = torch.empty((B, 4), device=dev, dtype=torch.float32)
    _lib.call("p2m_fit_camera", dev, x, cols, kind, n_in, p3, J, init, B, int(crop_size), int(n_iter), steps, rates,
              len(phases), wh, out["cam_param"], out["bbox"], out["target"], out["loss"], orig)
    if squeeze:
        out = {k: v[0] for k, v in out.items()}
    return out


def convert_crop_cam_to_orig_img(cam: torch.Tensor, bbox: torch.Tensor, img_width, img_height) -> torch.Tensor:
    """demo/run.py:24-43: cam [B, 3] in crop coordinates and bbox [B, 4] (x, y, w, h) -> [B, 4] (sx, sy, tx, ty) in
    the original image, float32 in numpy's operation order.  img_width / img_height: numbers or [B] tensors."""
    cam, bbox = _cuda(cam, "cam"), _cuda(bbox, "bbox")
    squeeze = cam.dim() == 1
    cam = cam.reshape(-1, 3).to(torch.float32).contiguous()
    bbox = bbox.reshape(-1, 4).to(torch.float32).contiguous()
    B = cam.shape[0]
    if bbox.shape[0] != B or bbox.device != cam.device:
        raise ValueError(f"cam {tuple(cam.shape)} and bbox {tuple(bbox.shape)} must describe the same people")
    w = torch.as_tensor(img_width, dtype=torch.float32).to(cam.device).reshape(-1).expand(B)
    h = torch.as_tensor(img_height, dtype=torch.float32).to(cam.device).reshape(-1).expand(B)
    wh = torch.stack([w, h], 1).contiguous()
    out = torch.empty((B, 4), device=cam.device, dtype=torch.float32)
    _lib.call("p2m_crop_cam_to_orig", cam.device, cam, bbox, wh, B, out)
    return out[0] if squeeze else out
