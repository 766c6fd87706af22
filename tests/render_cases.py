"""Meshes and cameras for the renderer's tests (pose2mesh_release_b200.render, oracle/render_oracle.py)."""
from __future__ import annotations

import numpy as np

from oracle import graph_oracle

# With W = H = 64, sx = sy = 1/32 and tx = ty = -32 the projection is the identity: u = x, v = y, exactly.
PIXEL_SIZE = 64
PIXEL_CAM = np.array([1 / 32, 1 / 32, -32.0, -32.0], np.float32)


def sphere_points(n_vertex: int, seed: int = 0) -> np.ndarray:
    """The unit-sphere points graph_oracle.synthetic_sphere_faces triangulates (same generator, same draws)."""
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(n_vertex, 3))
    return p / np.linalg.norm(p, axis=1, keepdims=True)


def outward(points: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """faces of a convex hull around the origin, each wound so that its normal points away from the origin (the
    hull's simplices come in either order)."""
    a, b, c = (points[faces[:, k]] for k in range(3))
    flip = np.einsum("ij,ij->i", np.cross(b - a, c - a), a + b + c) < 0
    out = faces.copy()
    out[flip, 1], out[flip, 2] = faces[flip, 2], faces[flip, 1]
    return out


def sphere_mesh(n_vertex: int, seed: int = 0):
    """(points [n, 3] float64, outward faces [2 n - 4, 3] int64) of the seeded synthetic sphere."""
    p = sphere_points(n_vertex, seed)
    return p, outward(p, graph_oracle.synthetic_sphere_faces(n_vertex, seed))


def coverage(verts, faces, cam, H, W):
    """How many of the faces cover each pixel, each face rasterised on its own: [H, W] int."""
    from oracle import render_oracle as ro

    verts = np.asarray(verts, np.float32)
    faces = np.asarray(faces).reshape(-1, 3)
    F = len(faces)
    tri = verts[faces]  # [F, 3, 3]: one person per face
    keys = ro.raster_keys(tri, np.array([[0, 1, 2]]), np.repeat(np.asarray(cam, np.float32)[None], F, 0),
                          np.arange(F), F, H, W)
    return (keys != ro.EMPTY).reshape(F, H, W).sum(0)


def front(tri_uv: np.ndarray) -> np.ndarray:
    """tri_uv [..., 3, 2]: rewind each triangle so that its (u, v) signed area is negative (the kept orientation)."""
    t = np.array(tri_uv, copy=True)
    a = (t[..., 1, 0] - t[..., 0, 0]) * (t[..., 2, 1] - t[..., 0, 1]) - (t[..., 2, 0] - t[..., 0, 0]) * (t[..., 1, 1] - t[..., 0, 1])
    sw = a > 0
    t[sw, 1], t[sw, 2] = tri_uv[sw, 2], tri_uv[sw, 1]
    return t
