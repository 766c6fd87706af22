"""TEST INFRASTRUCTURE ONLY — numpy restatement of the mesh-overlay kernels (csrc/render.cu, SURVEY.md §8 f10).

    gl_projection(verts, cam, H, W)   the reference's chain in float64: Rx(180°) (demo/renderer.py:70-71), the
                                      WeakPerspectiveCamera matrix (renderer.py:28-35), GL's viewport and the top-down
                                      read-back -> (u, v, z_ndc)
    project(verts, cams, H, W)        the kernel's projection u = W/2 (1 + sx (x + tx)), v = H/2 (1 + sy (y + ty)),
                                      z in `dtype`, one operation at a time in the kernel's order
    raster_keys(...)                  k_raster: the per-pixel 64-bit keys (0xFFFF - person | z order bits | face)
    render(...)                       k_raster + k_resolve: images_out, face_map, person_map, depth_map

Coverage, depth test, culling, clipping and compositing order are the reference's (renderer.py:66-114, run.py:46-67);
the flat Lambert shading is the library's own definition, not pyrender's shader.
"""
import math

import numpy as np

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
GUARD_PX = 2.0 ** 20
LIGHT = np.float32(2.4 / math.pi)
CHUNK = 1 << 22  # candidate pixels per vectorised step


def gl_projection(verts, cam, H, W):
    """verts [V, 3] and one orig_cam (sx, sy, tx, ty) through the reference's matrices in float64 -> u, v, z [V]."""
    x = np.asarray(verts, np.float64)
    sx, sy, tx, ty = (float(c) for c in cam)
    Rx = np.diag([1.0, -1.0, -1.0, 1.0])  # trimesh rotation_matrix(radians(180), [1, 0, 0]), up to cos(pi) rounding
    P = np.eye(4)
    P[0, 0], P[1, 1] = sx, sy
    P[0, 3], P[1, 3] = tx * sx, -ty * sy
    P[2, 2] = -1
    clip = (P @ Rx @ np.concatenate([x, np.ones((len(x), 1))], 1).T).T
    ndc = clip[:, :3] / clip[:, 3:]
    x_win = (ndc[:, 0] + 1) * W / 2
    y_win = (ndc[:, 1] + 1) * H / 2  # GL's window y points up; pyrender returns rows top-down
    return x_win, H - y_win, ndc[:, 2]


def project(verts, cams, H, W, dtype=np.float32):
    """verts [P, V, 3], cams [P, 4] -> u, v, z [P, V] in `dtype` in the kernel's operation order."""
    T = np.dtype(dtype).type
    x = np.asarray(verts, dtype)
    c = np.asarray(cams, dtype)
    hw, hh = T(W) * T(0.5), T(H) * T(0.5)
    with np.errstate(all="ignore"):
        u = hw * (T(1) + c[:, 0, None] * (x[..., 0] + c[:, 2, None]))
        v = hh * (T(1) + c[:, 1, None] * (x[..., 1] + c[:, 3, None]))
    return u, v, x[..., 2].copy()


def _z_order(z32):
    b = np.asarray(z32, np.float32).view(np.uint32).copy()
    b[b == 0x80000000] = 0
    return np.where(b & 0x80000000, ~b, b | np.uint32(0x80000000)).astype(np.uint64)


def raster_keys(verts, faces, cams, image_index, n_image, H, W, return_count=False):
    """k_raster: the winning key of every pixel, [n_image * H * W] uint64 (EMPTY where uncovered); with return_count
    also the number of fragments (covered pixel centres of kept triangles, inside the clip planes)."""
    verts = np.asarray(verts, np.float32)
    cams = np.asarray(cams, np.float32)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    P, V = verts.shape[:2]
    img = np.zeros(P, np.int64) if image_index is None else np.asarray(image_index, np.int64)
    keys = np.full(n_image * H * W, EMPTY, np.uint64)
    n_frag = 0
    if P == 0 or len(faces) == 0:
        return (keys, n_frag) if return_count else keys
    u, v, z = project(verts, cams, H, W)
    with np.errstate(invalid="ignore"):
        ok_v = np.isfinite(verts).all(-1) & (np.abs(u) <= GUARD_PX) & (np.abs(v) <= GUARD_PX)
    U = np.where(ok_v, np.rint(np.where(ok_v, u, 0) * np.float32(256)), 0).astype(np.int64)
    Vv = np.where(ok_v, np.rint(np.where(ok_v, v, 0) * np.float32(256)), 0).astype(np.int64)
    face_ok = ((faces >= 0) & (faces < V)).all(1)
    fi = np.where(face_ok[:, None], faces, 0)
    ok = (np.isfinite(cams).all(1) & (img >= 0) & (img < n_image))[:, None] & face_ok[None, :] & ok_v[:, fi].all(-1)
    tu, tv, tz = U[:, fi], Vv[:, fi], z[:, fi]  # [P, F, 3]
    area = (tu[..., 1] - tu[..., 0]) * (tv[..., 2] - tv[..., 0]) - (tu[..., 2] - tu[..., 0]) * (tv[..., 1] - tv[..., 0])
    i0 = np.maximum((tu.min(-1) + 127) >> 8, 0)
    i1 = np.minimum((tu.max(-1) - 128) >> 8, W - 1)
    r0 = np.maximum((tv.min(-1) + 127) >> 8, 0)
    r1 = np.minimum((tv.max(-1) - 128) >> 8, H - 1)
    keep = ok & (area < 0) & (i0 <= i1) & (r0 <= r1)
    pp, ff = np.nonzero(keep)
    tu, tv, tz, area = tu[pp, ff], tv[pp, ff], tz[pp, ff], area[pp, ff]
    i0, i1, r0, r1 = i0[pp, ff], i1[pp, ff], r0[pp, ff], r1[pp, ff]
    tag = ((np.uint64(0xFFFF) - pp.astype(np.uint64)) << np.uint64(48)) | ff.astype(np.uint64)
    # edge k is opposite vertex k: a1 -> a2, a2 -> a0, a0 -> a1; w_k = gu (pu - u_a) + gv (pv - v_a)
    base, su, sv, bias = [], [], [], []
    for k, (a, b) in enumerate(((1, 2), (2, 0), (0, 1))):
        gu, gv = tv[:, b] - tv[:, a], tu[:, a] - tu[:, b]
        base.append(gu * (128 - tu[:, a]) + gv * (128 - tv[:, a]))
        su.append(gu * 256)
        sv.append(gv * 256)
        bias.append(np.where((gu > 0) | ((gu == 0) & (gv > 0)), 0, 1))
    den = (-area).astype(np.float64)
    bw = i1 - i0 + 1
    n = bw * (r1 - r0 + 1)
    ends = np.cumsum(n)
    lo = 0
    while lo < len(n):  # chunks of whole triangles
        hi = max(int(np.searchsorted(ends, (ends[lo - 1] if lo else 0) + CHUNK, side="right")), lo + 1)
        t = np.repeat(np.arange(lo, hi), n[lo:hi])
        local = np.arange(len(t)) - np.repeat(ends[lo:hi] - n[lo:hi] - (ends[lo - 1] if lo else 0), n[lo:hi])
        i, r = i0[t] + local % bw[t], r0[t] + local // bw[t]
        w = [base[k][t] + i * su[k][t] + r * sv[k][t] for k in range(3)]
        inside = (w[0] >= bias[0][t]) & (w[1] >= bias[1][t]) & (w[2] >= bias[2][t])
        t, i, r, w = t[inside], i[inside], r[inside], [x[inside] for x in w]
        zz = tz[t].astype(np.float64)
        num = (w[0].astype(np.float64) * zz[:, 0] + w[1].astype(np.float64) * zz[:, 1]) + w[2].astype(np.float64) * zz[:, 2]
        z32 = (num / den[t]).astype(np.float32)
        clip = (z32 >= -1) & (z32 <= 1)
        t, i, r, z32 = t[clip], i[clip], r[clip], z32[clip]
        key = tag[t] | (_z_order(z32) << np.uint64(16))
        np.minimum.at(keys, (img[pp[t]] * H + r) * W + i, key)
        n_frag += len(key)
        lo = hi
    return (keys, n_frag) if return_count else keys


def render(images, verts, faces, cams, colors, image_index=None):
    """images [N, H, W, 3] uint8 -> (images_out, face_map, person_map, depth_map) with the kernels' bits."""
    images = np.asarray(images, np.uint8)
    N, H, W = images.shape[:3]
    verts = np.asarray(verts, np.float32)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    colors = np.asarray(colors, np.float32).reshape(-1, 3)
    keys = raster_keys(verts, faces, cams, image_index, N, H, W)
    out = images.reshape(-1, 3).copy()
    face_map = np.full(keys.shape, -1, np.int32)
    person_map = np.full(keys.shape, -1, np.int32)
    depth_map = np.full(keys.shape, np.nan, np.float32)
    q = np.nonzero(keys != EMPTY)[0]
    k = keys[q]
    p = (np.uint64(0xFFFF) - (k >> np.uint64(48))).astype(np.int64)
    f = (k & np.uint64(0xFFFF)).astype(np.int64)
    zk = ((k >> np.uint64(16)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    zb = np.where(zk & 0x80000000, zk & np.uint32(0x7FFFFFFF), ~zk).astype(np.uint32)
    a, b, c = (verts[p, faces[f, j]] for j in range(3))
    d1, d2 = b - a, c - a
    nx = d1[:, 1] * d2[:, 2] - d1[:, 2] * d2[:, 1]
    ny = d1[:, 2] * d2[:, 0] - d1[:, 0] * d2[:, 2]
    nz = d1[:, 0] * d2[:, 1] - d1[:, 1] * d2[:, 0]
    with np.errstate(all="ignore"):
        length = np.sqrt((nx * nx + ny * ny) + nz * nz)
        lam = np.fmax(np.float32(0), -(nz / length))  # NaN -> 0, as fmaxf
        intensity = np.float32(0.3) + LIGHT * lam
        ck = np.fmin(np.fmax(colors[p] * intensity[:, None], np.float32(0)), np.float32(1))
    out[q] = np.floor(ck * np.float32(255) + np.float32(0.5)).astype(np.uint8)
    face_map[q], person_map[q], depth_map[q] = f, p, zb.view(np.float32)
    shp = (N, H, W)
    return out.reshape(N, H, W, 3), face_map.reshape(shp), person_map.reshape(shp), depth_map.reshape(shp)
