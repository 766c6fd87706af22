"""The demo's mesh overlay on the GPU (SURVEY.md §8 row f10):

    render_meshes(images, verts, faces, cams, colors)    demo/renderer.py Renderer.render (renderer.py:66-114) for
                                                          every person of every image in one call (demo/run.py:46-67)

Runs in libp2m_b200.so (p2m_render_workspace_bytes, p2m_render_meshes); CUDA tensors only.

Coverage, depth test (nearer z wins, the lower face on a tie), back-face culling, clipping at z = +-1 and compositing
order (people in order, the later one winning where two overlap) are the reference's.  Coverage is exact: positions
snapped to 1/256 px, int64 edge functions and the top-left fill rule, so a pixel on an edge shared by two faces is
drawn once.  The shading is this library's own and does not reproduce pyrender's shader: flat Lambert of the
reference's scene (ambient 0.3, three 0.8 directional lights along the camera axis), no specular term, no tone mapping,
no anti-aliasing: c_k = clamp(color_k (0.3 + (2.4/pi) max(0, -n_z)), 0, 1) for the face normal n in mesh coordinates,
stored as floor(255 c + 0.5).  Channel k of the output takes colour component k, as the reference writes pyrender's
RGB into its BGR image.  Vertices beyond +-2^20 px drop their triangle (instead of GL's clipping).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

MAX_PEOPLE = 65535
MAX_FACES = 65535
MAX_SIDE = 16384


def _cuda(x, what: str) -> torch.Tensor:
    _lib.cuda_tensor(x, what)
    if x.requires_grad:
        raise ValueError(f"{what} requires grad; the renderer is not differentiable")
    return x


def _faces(faces, n_vertex: int, device) -> torch.Tensor:
    """[F, 3] int32 on device.  Host faces are range-checked here; CUDA faces are not read back (the kernel skips
    out-of-range ones)."""
    if isinstance(faces, torch.Tensor) and faces.is_cuda:
        if faces.requires_grad:
            raise ValueError("faces requires grad")
        if faces.dtype.is_floating_point or faces.dtype.is_complex or faces.dtype == torch.bool:
            raise ValueError(f"faces must be integer; got {faces.dtype}")
        if faces.device != device:
            raise ValueError(f"faces is on {faces.device}, verts on {device}")
        f = faces
    else:
        a = faces.numpy() if isinstance(faces, torch.Tensor) else np.asarray(faces)
        if a.dtype.kind not in "iu":
            raise ValueError(f"faces must be integer; got {a.dtype}")
        if a.size and (a.min() < 0 or a.max() >= n_vertex):
            raise ValueError(f"faces index outside [0, {n_vertex})")
        f = torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)
    if f.dim() != 2 or f.shape[1] != 3:
        raise ValueError(f"faces must be [F, 3]; got {tuple(f.shape)}")
    if f.shape[0] > MAX_FACES:
        raise ValueError(f"at most {MAX_FACES} faces; got {f.shape[0]}")
    return f.to(torch.int32).contiguous()


@torch.no_grad()
def render_meshes(images, verts, faces, cams, colors, image_index=None, return_maps: bool = False):
    """Draw every person's mesh over its image, as Renderer.render does one person at a time.

    images       [N, H, W, 3] or [H, W, 3] uint8, CUDA (left untouched)
    verts        [P, V, 3] (or [V, 3]) the meshes in metres, the perm_reverse-gathered vertices the demo renders
    faces        [F, 3] integer, numpy, CPU or CUDA
    cams         [P, 4] (or [4]) orig_cam (sx, sy, tx, ty), as fit_cameras(..., image_size=...) returns it; a person
                 whose fit was rejected has NaN there and is not drawn
    colors       [P, 3] (or [3]) RGB in [0, 1], e.g. from colorsys.hsv_to_rgb
    image_index  [P] integer: the image each person goes on (None: all on image 0; out of range: not drawn)

    Returns a new uint8 tensor shaped like ``images``; with return_maps, also ``face_map`` and ``person_map`` (int32,
    -1 where nothing is drawn) and ``depth_map`` (float32, NaN there), shaped like the images without the channels.
    One memset and two launches on the current stream, nothing read back: a call can be captured in a CUDA graph."""
    img = _cuda(images, "images")
    squeeze = img.dim() == 3
    if squeeze:
        img = img.unsqueeze(0)
    if img.dim() != 4 or img.shape[-1] != 3 or img.dtype != torch.uint8:
        raise ValueError(f"images must be [N, H, W, 3] or [H, W, 3] uint8; got {tuple(images.shape)} {images.dtype}")
    N, H, W = img.shape[:3]
    if N == 0 or not (0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
        raise ValueError(f"need N > 0 images of 1 .. {MAX_SIDE} pixels per side; got {N} x {H} x {W}")
    dev = img.device
    v = _cuda(verts, "verts")
    v = v.unsqueeze(0) if v.dim() == 2 else v
    c, col = _cuda(cams, "cams"), _cuda(colors, "colors")
    c = c.unsqueeze(0) if c.dim() == 1 else c
    col = col.unsqueeze(0) if col.dim() == 1 else col
    if v.dim() != 3 or v.shape[-1] != 3:
        raise ValueError(f"verts must be [P, V, 3]; got {tuple(verts.shape)}")
    P, V = v.shape[:2]
    if c.shape != (P, 4) or col.shape != (P, 3):
        raise ValueError(f"cams must be [P, 4] and colors [P, 3] for P = {P}; got {tuple(cams.shape)}, "
                         f"{tuple(colors.shape)}")
    if P > MAX_PEOPLE:
        raise ValueError(f"at most {MAX_PEOPLE} people per call; got {P}")
    for t, name in ((v, "verts"), (c, "cams"), (col, "colors")):
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, images on {dev}")
        if not t.is_floating_point():
            raise ValueError(f"{name} must be floating point; got {t.dtype}")
    f = _faces(faces, V, dev)
    if image_index is None:
        idx = torch.zeros(P, dtype=torch.int32, device=dev)
    else:
        idx = _cuda(image_index, "image_index")
        if idx.dtype.is_floating_point or idx.dtype == torch.bool or idx.shape != (P,) or idx.device != dev:
            raise ValueError(f"image_index must be an integer [P] tensor on {dev}; got {tuple(idx.shape)} {idx.dtype}")
        idx = idx.to(torch.int32)
    v = v.to(torch.float32).contiguous()
    c = c.to(torch.float32).contiguous()
    col = col.to(torch.float32).contiguous()
    idx = idx.contiguous()
    img_in = img.contiguous()
    out = torch.empty_like(img_in)
    maps = None
    if return_maps:
        maps = (torch.empty((N, H, W), dtype=torch.int32, device=dev), torch.empty((N, H, W), dtype=torch.int32, device=dev),
                torch.empty((N, H, W), dtype=torch.float32, device=dev))
    ws_bytes = _lib.load().p2m_render_workspace_bytes(N, H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None  # noqa: E731
    _lib.call("p2m_render_meshes", dev, ptr(v), P, V, ptr(f), f.shape[0], ptr(c), ptr(col), ptr(idx), img_in, N, H, W,
              out, *(ptr(m) for m in (maps or (None, None, None))), ws, ws_bytes)
    if squeeze:
        out = out[0]
        maps = maps and tuple(m[0] for m in maps)
    return (out, *maps) if return_maps else out
