"""The mesh-overlay oracle (oracle/render_oracle.py) against the reference's projection and GL's rasterisation rules,
and the renderer's argument checks that need no GPU."""
import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

import render_cases as rc
from oracle import camera_oracle as co
from oracle import render_oracle as ro

S = rc.PIXEL_SIZE


def random_cams(g, n):
    return np.stack([g.uniform(0.1, 2, n), g.uniform(0.1, 2, n), g.normal(0, 0.5, n), g.normal(0, 0.5, n)], 1)


# ------------------------------------------------------------------------------------------------ projection
def test_projection_equals_reference_matrices():
    g = np.random.default_rng(0)
    H, W = 1080, 1920
    for cam in random_cams(g, 8) * np.array([1, 1, 1, 1]) * g.choice([-1, 1], (8, 4)):
        x = g.normal(0, 0.5, (200, 3))
        u_ref, v_ref, z_ref = ro.gl_projection(x, cam, H, W)
        u, v, z = ro.project(x[None], cam[None], H, W, dtype=np.float64)
        for got, ref in ((u[0], u_ref), (v[0], v_ref), (z[0], z_ref)):
            np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())
        u32, v32, _ = ro.project(x[None], cam[None], H, W)  # the kernel's float32 order: float32 rounding away
        np.testing.assert_allclose(u32[0], u_ref, rtol=0, atol=1e-3)
        np.testing.assert_allclose(v32[0], v_ref, rtol=0, atol=1e-3)


def test_projection_agrees_with_the_camera_fit():
    """orig_cam = convert_crop_cam_to_orig_img(cam, bbox1) puts a vertex where OptimzeCamLayer's crop projection
    ((x + t) s) crop/2 + crop/2, mapped back through the square bbox1, puts it: u = cx + s h/2 (x + tx)."""
    g = np.random.default_rng(1)
    B, H, W, crop = 16, 1080, 1920, 500
    cam = np.stack([g.uniform(0.5, 1.5, B), g.normal(0, 0.2, B), g.normal(0, 0.2, B)], 1).astype(np.float32)
    side = g.uniform(100, 900, B)
    bbox = np.stack([g.uniform(-100, 1500, B), g.uniform(-100, 700, B), side, side], 1).astype(np.float32)
    orig = co.orig_cam_f32(cam, bbox, W, H)
    x = g.normal(0, 0.4, (B, 50, 3))
    u, v, _ = ro.project(x, orig, H, W, dtype=np.float64)
    c64, b64 = cam.astype(np.float64), bbox.astype(np.float64)
    cx, cy, h = b64[:, 0] + b64[:, 2] / 2, b64[:, 1] + b64[:, 3] / 2, b64[:, 3]
    s, tx, ty = c64[:, :1], c64[:, 1:2], c64[:, 2:3]
    np.testing.assert_allclose(u, cx[:, None] + s * h[:, None] / 2 * (x[..., 0] + tx), rtol=0, atol=2e-3)
    np.testing.assert_allclose(v, cy[:, None] + s * h[:, None] / 2 * (x[..., 1] + ty), rtol=0, atol=2e-3)
    crop_u = ((x[..., 0] + tx) * s) * (crop / 2) + crop / 2  # project_net.py OptimzeCamLayer.forward
    np.testing.assert_allclose(u, b64[:, :1] + crop_u * b64[:, 2:3] / crop, rtol=0, atol=2e-3)


def test_pixel_camera_is_the_identity():
    g = np.random.default_rng(2)
    x = np.round(g.uniform(-20, 80, (1, 100, 3)) * 256) / 256
    u, v, _ = ro.project(x, rc.PIXEL_CAM[None], S, S)
    assert np.array_equal(u, x[..., 0].astype(np.float32)) and np.array_equal(v, x[..., 1].astype(np.float32))


# ------------------------------------------------------------------------------------------------ fill rule
def _inside_convex(points2d, px, margin=1e-6):
    hull = ConvexHull(points2d)
    return (px @ hull.equations[:, :2].T + hull.equations[:, 2] < -margin).all(1)


def _centres():
    r, i = np.mgrid[0:S, 0:S]
    return np.stack([i.ravel() + 0.5, r.ravel() + 0.5], 1)


def test_fan_on_pixel_centres_and_edges_covers_each_pixel_once():
    ring = np.array([[30.5, 20.0], [36.0, 22.5], [40.5, 30.5], [38.0, 37.0], [30.5, 42.5], [24.0, 38.0],
                     [20.5, 30.5], [22.0, 24.5]])
    centre = np.array([30.5, 30.5])
    tris = rc.front(np.stack([np.repeat(centre[None], len(ring), 0), ring, np.roll(ring, -1, 0)], 1))
    verts = np.concatenate([tris, np.zeros(tris.shape[:2] + (1,))], 2).reshape(-1, 3)
    cov = rc.coverage(verts, np.arange(len(verts)).reshape(-1, 3), rc.PIXEL_CAM, S, S).ravel()
    assert cov.max() == 1
    inside = _inside_convex(ring, _centres())
    assert inside.sum() > 250 and (cov[inside] == 1).all()


@pytest.mark.parametrize("step, origin", [(3.0, (4.5, 6.5)), (2.5, (5.0, 3.5)), (1.0, (10.5, 10.5))])
def test_regular_grid_covers_each_pixel_once(step, origin):
    n = 16
    gy, gx = np.mgrid[0:n, 0:n]
    pts = np.stack([origin[0] + step * gx.ravel(), origin[1] + step * gy.ravel(), np.zeros(n * n)], 1)
    q = (gy[:-1, :-1] * n + gx[:-1, :-1]).ravel()
    faces = np.concatenate([np.stack([q, q + 1, q + n + 1], 1), np.stack([q, q + n + 1, q + n], 1)])
    tri_uv = rc.front(pts[faces][..., :2])
    verts = np.concatenate([tri_uv, np.zeros(tri_uv.shape[:2] + (1,))], 2).reshape(-1, 3)
    cov = rc.coverage(verts, np.arange(len(verts)).reshape(-1, 3), rc.PIXEL_CAM, S, S).ravel()
    assert cov.max() == 1
    inside = _inside_convex(pts[:, :2], _centres())
    assert (cov[inside] == 1).all()


@pytest.mark.parametrize("seed", [0, 3])
def test_closed_convex_mesh_covers_its_silhouette_once(seed):
    p, faces = rc.sphere_mesh(400, seed)
    verts = (p * 0.8).astype(np.float32)
    cam = np.array([0.7, 0.8, 0.05, -0.1], np.float32)
    H, W = 72, 80
    cov = rc.coverage(verts, faces, cam, H, W).ravel()
    assert cov.max() == 1
    u, v, _ = ro.project(verts[None], cam[None], H, W)
    r, i = np.mgrid[0:H, 0:W]
    centres = np.stack([i.ravel() + 0.5, r.ravel() + 0.5], 1)
    uv = np.stack([np.rint(u[0] * 256), np.rint(v[0] * 256)], 1) / 256
    inside = _inside_convex(uv, centres)
    outside = ~_inside_convex(uv, centres, margin=-1e-6)
    assert inside.sum() > 1000 and (cov[inside] == 1).all() and (cov[outside] == 0).all()
    # the back faces alone cover nothing, the front faces are those whose normal has n_z < 0
    n = np.cross(verts[faces[:, 1]] - verts[faces[:, 0]], verts[faces[:, 2]] - verts[faces[:, 0]])
    assert rc.coverage(verts, faces[n[:, 2] > 0], cam, H, W).sum() == 0


# ------------------------------------------------------------------------------------------------ GL semantics
def tri(u, v, z=0.0):
    """One triangle at pixel positions (for PIXEL_CAM) in the kept orientation, as a [1, 3, 3] person."""
    t = rc.front(np.array([[[u[0], v[0]], [u[1], v[1]], [u[2], v[2]]]], np.float64))[0]
    return np.concatenate([t, np.broadcast_to(np.asarray(z, np.float64).reshape(-1, 1), (3, 1))], 1)[None]


BIG = tri((5.2, 50.3, 12.1), (4.7, 20.2, 55.9))
BLANK = np.full((1, S, S, 3), 17, np.uint8)
F1 = np.array([[0, 1, 2]])


def draw(verts, faces=F1, cams=None, colors=None, image_index=None, images=BLANK):
    verts = np.asarray(verts, np.float32)
    P = len(verts)
    cams = np.repeat(rc.PIXEL_CAM[None], P, 0) if cams is None else cams
    colors = np.full((P, 3), 0.5, np.float32) if colors is None else colors
    return ro.render(images, verts, faces, cams, colors, image_index)


def test_depth_tie_goes_to_the_lower_face_and_nearer_wins():
    v = np.concatenate([BIG[0], BIG[0]])[None]
    _, fm, _, _ = draw(v, faces=np.array([[3, 4, 5], [0, 1, 2]]))
    assert set(np.unique(fm)) == {-1, 0}
    v2 = v.copy()
    v2[0, 3:, 2] = 0.25  # face 0 farther
    _, fm, _, dm = draw(v2, faces=np.array([[3, 4, 5], [0, 1, 2]]))
    assert set(np.unique(fm)) == {-1, 1} and np.nanmax(dm) == 0


def test_later_person_wins_whatever_the_depth():
    near, far = BIG.copy(), BIG.copy()
    near[..., 2], far[..., 2] = -0.9, 0.9
    _, _, pm, dm = draw(np.concatenate([near, far]))
    assert set(np.unique(pm)) == {-1, 1} and np.nanmin(dm) == np.float32(0.9)


def test_fragments_beyond_the_clip_planes_are_dropped():
    assert (draw(tri((5, 50, 12), (5, 20, 55), z=1.5))[1] == -1).all()
    assert (draw(tri((5, 50, 12), (5, 20, 55), z=-1.01))[1] == -1).all()
    full = draw(tri((5, 50, 12), (5, 20, 55), z=0.0))[1] >= 0
    part, dm = (lambda o: (o[1] >= 0, o[3]))(draw(tri((5, 50, 12), (5, 20, 55), z=(-3.0, 0.5, 0.5))))
    assert 0 < part.sum() < full.sum() and np.nanmin(dm) >= -1 and np.nanmax(dm) <= 1
    edge = draw(tri((5, 50, 12), (5, 20, 55), z=1.0))
    assert (edge[1] >= 0).sum() == full.sum() and np.nanmax(edge[3]) == 1


def test_back_faces_and_a_mirrored_camera_are_culled():
    assert (draw(BIG)[1] >= 0).sum() > 200
    assert (draw(BIG[:, [0, 2, 1]])[1] == -1).all()
    mirrored = rc.PIXEL_CAM.copy()
    mirrored[0], mirrored[2] = -mirrored[0], -mirrored[2] - 2 * 32   # u -> 64 - u: mirrored, still on the image
    assert (draw(BIG, cams=mirrored[None])[1] == -1).all()
    assert (draw(BIG[:, [0, 2, 1]], cams=mirrored[None])[1] >= 0).sum() > 200
    rotated = mirrored.copy()
    rotated[1], rotated[3] = -rotated[1], -rotated[3] - 2 * 32         # and v -> 64 - v: a rotation, kept
    assert (draw(BIG, cams=rotated[None])[1] >= 0).sum() > 200


def test_invalid_inputs_are_skipped():
    v = np.concatenate([BIG, BIG])
    nan_cam = np.repeat(rc.PIXEL_CAM[None], 2, 0)
    nan_cam[1, 2] = np.nan
    _, _, pm, _ = draw(v, cams=nan_cam)
    assert set(np.unique(pm)) == {-1, 0}
    _, _, pm, _ = draw(v, image_index=np.array([0, 1]))
    assert set(np.unique(pm)) == {-1, 0}
    _, _, pm, _ = draw(v, image_index=np.array([-1, 0]))
    assert set(np.unique(pm)) == {-1, 1}
    _, fm, _, _ = draw(np.concatenate([BIG[0], BIG[0]])[None], faces=np.array([[0, 1, 7], [3, 4, 5]]))
    assert set(np.unique(fm)) == {-1, 1}
    far = BIG.copy()
    far[0, 0, 0] = 2.0 ** 20 + 100   # beyond the guard band: the whole triangle goes
    assert (draw(far)[1] == -1).all()
    nanv = BIG.copy()
    nanv[0, 1, 2] = np.nan
    assert (draw(nanv)[1] == -1).all()


def test_flat_shading_and_compositing():
    g = np.random.default_rng(4)
    images = g.integers(0, 256, (1, S, S, 3), dtype=np.uint8)
    colors = np.array([[1.0, 0.5, 0.0]], np.float32)
    out, fm, _, _ = draw(BIG, colors=colors, images=images)   # a flat triangle faces the camera: n_z = -1
    hit = fm[0] >= 0
    light = np.float32(0.3) + np.float32(2.4 / np.pi)
    want = np.floor(np.minimum(colors[0] * light, 1) * 255 + 0.5).astype(np.uint8)
    assert (out[0][hit] == want).all() and tuple(want) == (255, 136, 0)
    assert np.array_equal(out[0][~hit], images[0][~hit])
    # a face tilted about the v axis by 45 degrees: -n_z = 0.707
    t = tri((-0.6, 0.6, 0.1), (-0.5, -0.4, 0.6))
    t[0, :, 2] = 0.5 * t[0, :, 0]
    t[0, :, 0] = 0.5 * t[0, :, 0]
    out, fm, _, _ = draw(t, cams=np.array([[1, 1, 0, 0]], np.float32), colors=colors, images=images)
    hit = fm[0] >= 0
    n = np.cross(t[0, 1] - t[0, 0], t[0, 2] - t[0, 0])
    want = colors[0] * (0.3 + 2.4 / np.pi * max(0.0, -n[2] / np.linalg.norm(n))) * 255 + 0.5
    assert hit.sum() > 50 and 0.7 < -n[2] / np.linalg.norm(n) < 0.71
    assert (np.abs(out[0][hit].astype(np.float64) - np.floor(want)) <= 1).all()


# ------------------------------------------------------------------------------------------------ argument checks
def test_cpu_tensors_raise():
    from pose2mesh_release_b200.render import render_meshes

    with pytest.raises(RuntimeError, match="CUDA"):
        render_meshes(torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(1, 3, 3), np.array([[0, 1, 2]]),
                      torch.zeros(1, 4), torch.zeros(1, 3))


def test_native_limits_are_checked_before_any_device_work():
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    assert lib.p2m_render_workspace_bytes(2, 3, 5) == 2 * 3 * 5 * 8
    assert lib.p2m_render_workspace_bytes(0, 3, 5) == 0
    for P, F, N, H, W in ((65536, 1, 1, 8, 8), (1, 65536, 1, 8, 8), (1, 1, 1, 16385, 8), (1, 1, 1, 8, 16385),
                          (1, 1, 0, 8, 8), (-1, 1, 1, 8, 8)):
        st = lib.p2m_render_meshes(None, P, 3, None, F, None, None, None, None, N, H, W, None, None, None, None, None,
                                   0, None)
        assert st == 1, (P, F, N, H, W)
        assert b"render_meshes" in lib.p2m_last_error()
