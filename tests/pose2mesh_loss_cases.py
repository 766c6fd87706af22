"""Seeded inputs of the Trainer's objective (lib/core/base.py:129-143) at a given size: a synthetic sphere mesh, its
random placement into a padded output of n_padded rows, a sparse regressor with zero rows and columns, and validity
masks with zero entries and whole zero samples."""
import functools

import numpy as np
import torch

from pose2mesh_release_b200 import graph as pg

FACE_SEED = {6890: 2, 778: 1}   # the seeds that give SMPL's and MANO's level sizes (graph.synthetic_sphere_faces)


@functools.lru_cache(maxsize=None)
def sphere(n_vertex):
    """(faces, unit points) of the seeded convex-hull sphere: the points are the hull's vertices."""
    seed = FACE_SEED.get(n_vertex, 0)
    pts = np.random.default_rng(seed).normal(size=(n_vertex, 3))
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    return pg.synthetic_sphere_faces(n_vertex, seed), pts


def make_case(n_vertex, n_padded, batch, n_reg_joint, n_lift_joint, seed):
    face, pts = sphere(n_vertex)
    rng = np.random.default_rng(seed)
    B, nv, nj, nl = batch, n_vertex, n_reg_joint, n_lift_joint
    perm = rng.permutation(n_padded)                       # real vertex v is padded row perm[v]
    scale = rng.uniform(0.3, 0.9, size=(B, 1, 1))
    gt_mesh = pts[None] * scale + rng.uniform(-0.5, 0.5, size=(B, 1, 3)) + 0.01 * rng.normal(size=(B, nv, 3))
    pred = gt_mesh + 0.02 * rng.normal(size=(B, nv, 3))
    cam_mesh = rng.normal(size=(B, n_padded, 3))          # padding rows: values the objective must ignore
    cam_mesh[:, perm[:nv]] = pred
    jr = rng.uniform(size=(nj, nv)) * (rng.uniform(size=(nj, nv)) < 0.03)
    jr[:, rng.uniform(size=nv) < 0.1] = 0.0                # zero columns
    jr[min(1, nj - 1)] = 0.0                               # a zero row
    jr /= np.maximum(jr.sum(1, keepdims=True), 1e-12)
    gt_reg = np.einsum("jv,bvc->bjc", jr, gt_mesh * 1000) + 20.0 * rng.normal(size=(B, nj, 3))
    lift = 300.0 * rng.normal(size=(B, nl, 3))
    gt_lift = lift + 30.0 * rng.normal(size=(B, nl, 3))
    mesh_valid = (rng.uniform(size=(B, nv, 1)) > 0.1).astype(np.float64)
    reg_valid = (rng.uniform(size=(B, nj, 1)) > 0.2).astype(np.float64)
    lift_valid = (rng.uniform(size=(B, nl, 1)) > 0.2).astype(np.float64)
    if B >= 2:                                             # whole zero samples
        mesh_valid[B - 1] = 0.0
        reg_valid[0] = 0.0
        lift_valid[B // 2] = 0.0
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))  # noqa: E731
    return dict(face=face, perm_reverse=perm, joint_regressor=f32(jr), cam_mesh=f32(cam_mesh), lift_pose=f32(lift),
                gt_mesh=f32(gt_mesh), gt_reg3dpose=f32(gt_reg), gt_lift3dpose=f32(gt_lift), mesh_valid=f32(mesh_valid),
                reg3dpose_valid=f32(reg_valid), lift3dpose_valid=f32(lift_valid))


INPUTS = ("cam_mesh", "lift_pose", "gt_mesh", "gt_reg3dpose", "gt_lift3dpose", "mesh_valid", "reg3dpose_valid",
          "lift3dpose_valid")
