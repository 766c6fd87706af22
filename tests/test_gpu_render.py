"""The mesh overlay on the GPU (SURVEY.md §8 row f10, pose2mesh_release_b200.render) against
oracle/render_oracle.py, bit for bit: the face, person and depth maps and the composited images.

People are the seeded synthetic SMPL / MANO models of tests/body_models.py with the seeded synthetic sphere as their
template (a closed surface of the real vertex and face counts), posed by body_model.SMPLLayer / ManoLayer, with
cameras from camera.fit_cameras on their joints."""
import numpy as np
import pytest
import torch

import body_models as bm
import render_cases as rc
from oracle import render_oracle as ro

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def people(kind, P, W, H, seed, centres=None):
    """P posed meshes and their fitted orig_cam: (verts [P, V, 3] float32, faces [F, 3], cams [P, 4], colors [P, 3]),
    device tensors but faces (numpy)."""
    from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer
    from pose2mesh_release_b200.camera import fit_cameras

    rng = np.random.RandomState(seed)
    if kind == "smpl":
        m = bm.smpl_model()
        pts, faces = rc.sphere_mesh(6890, 0)
        vt = (pts * np.array([0.35, 0.85, 0.15])).astype(np.float32)
        layer = SMPLLayer(vt, m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"], m["betas"])
        pose = bm.random_axisang(rng, P * 24, 0.02, 0.3).reshape(P, 72)
        verts, joints = layer(cuda(pose.astype(np.float32)))
        scale = 1.0
    else:
        m = bm.mano_model("right")
        pts, faces = rc.sphere_mesh(778, 1)
        vt = (pts * np.array([0.35, 0.85, 0.15]) * 0.12).astype(np.float32)
        layer = ManoLayer(vt, m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                          m["hands_mean"], flat_hand_mean=False, side="right")
        pose = bm.random_axisang(rng, P * 16, 0.02, 0.3).reshape(P, 48)
        verts, joints = layer(cuda(pose.astype(np.float32)))
        scale = 1e-3  # millimetres -> metres, the mesh the demo renders
    verts, joints = (verts * scale).contiguous(), (joints * scale).contiguous()
    J = 17 if kind == "smpl" else 21
    j = joints[:, :J].cpu().numpy().astype(np.float64)
    if centres is None:
        centres = np.stack([rng.uniform(0.2, 0.8, P) * W, rng.uniform(0.3, 0.7, P) * H], 1)
    S = rng.uniform(0.2, 0.35, (P, 1, 1)) * H * (1 if kind == "smpl" else 15)  # px per metre: a 1.7 m / 0.2 m mesh
    px = (j[:, :, :2] - j[:, :, :2].mean(1, keepdims=True)) * S + np.asarray(centres)[:, None] + rng.normal(0, 2, (P, J, 2))
    init = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    cams = fit_cameras(cuda(px), joints[:, :J], init=cuda(init), image_size=(W, H))["orig_cam"]
    colors = cuda(rng.uniform(0.2, 1.0, (P, 3)).astype(np.float32))
    return verts, faces, cams, colors


def images(N, H, W, seed):
    return cuda(np.random.default_rng(seed).integers(0, 256, (N, H, W, 3), dtype=np.uint8))


def check(imgs, verts, faces, cams, colors, image_index=None, min_covered=1):
    from pose2mesh_release_b200.render import render_meshes

    got = render_meshes(imgs, verts, faces, cams, colors, image_index=image_index, return_maps=True)
    f_host = faces.cpu().numpy() if isinstance(faces, torch.Tensor) else faces
    ref = ro.render(imgs.cpu().numpy(), verts.cpu().numpy(), f_host, cams.cpu().numpy(), colors.cpu().numpy(),
                    None if image_index is None else image_index.cpu().numpy())
    for name, g, r in zip(("images", "face_map", "person_map", "depth_map"), got, ref):
        g = g.cpu().numpy()
        assert g.shape == r.shape and g.dtype == r.dtype, name
        bad = ~((g == r) | (np.isnan(g) & np.isnan(r))) if g.dtype.kind == "f" else g != r
        assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:5])
    assert (ref[1] >= 0).sum() >= min_covered
    return got


# ------------------------------------------------------------------------------------------------ bitwise
@pytest.mark.parametrize("N, H, W, P", [(3, 1080, 1920, 8), (2, 479, 641, 5)])
def test_smpl_people_bitwise_equal_to_oracle(N, H, W, P):
    rng = np.random.default_rng(P)
    idx = np.sort(rng.integers(0, N, P)).astype(np.int32)
    # overlapping pairs: consecutive people on one image stand close together
    base = np.stack([rng.uniform(0.3, 0.7, P) * W, rng.uniform(0.4, 0.6, P) * H], 1)
    base[1::2] = base[0::2][: len(base[1::2])] + np.array([0.08 * W, 0.02 * H])
    verts, faces, cams, colors = people("smpl", P, W, H, seed=P, centres=base)
    assert torch.isfinite(cams).all()
    got = check(images(N, H, W, 0), verts, faces, cams, colors, cuda(idx), min_covered=20000)
    pm = got[2].cpu().numpy()
    assert len(np.unique(pm[pm >= 0])) >= P - 2   # a later neighbour may hide an earlier person entirely


def test_mano_hands_bitwise_equal_to_oracle():
    B = 16
    verts, faces, cams, colors = people("mano", B, 224, 224, seed=3, centres=np.full((B, 2), 112.0))
    check(images(B, 224, 224, 1), verts, faces, cams, colors, cuda(np.arange(B, dtype=np.int32)),
          min_covered=B * 2000)


# ------------------------------------------------------------------------------------------------ edge cases
def test_large_triangles_bitwise_equal_to_oracle():
    """A camera zoomed in until single faces cover most of the image: the warp-shared path."""
    p, faces = rc.sphere_mesh(40, 2)
    verts = cuda((p * 0.5).astype(np.float32)[None].repeat(2, 0))
    cams = cuda(np.array([[6.0, 10.0, 0.02, -0.03], [1.5, 2.6, 0.1, 0.0]], np.float32))
    got = check(images(1, 479, 641, 2), verts, faces, cams, cuda(np.array([[0.9, 0.4, 0.1], [0.2, 0.5, 1.0]],
                                                                            np.float32)), min_covered=200000)
    assert (got[2].cpu().numpy() == 1).sum() > 10000


def test_partial_invalid_and_guard_band_people_bitwise_equal_to_oracle():
    W, H = 640, 480
    verts, faces, cams, colors = people("smpl", 5, W, H, seed=11, centres=np.array(
        [[5.0, 240], [320, 470], [320, 240], [400, 250], [300, 200]]))
    cams = cams.clone()
    cams[2] = float("nan")                 # a person the camera fit rejected
    verts = verts.clone()
    verts[3, :100, 0] = 1e5                # vertices past the 2^20 px guard band: their faces are skipped
    f = cuda(faces.astype(np.int32))
    f[7, 1] = 6890                         # a CUDA faces tensor with out-of-range indices is not read back
    f[100, 0] = -3
    got = check(images(1, H, W, 3), verts, f, cams, colors, min_covered=5000)
    fm, pm = got[1].cpu().numpy(), got[2].cpu().numpy()
    assert not (pm == 2).any() and not np.isin(fm, [7, 100]).any()
    assert (pm == 0).any() and (pm == 1).any()   # half outside the image, still drawn


# ------------------------------------------------------------------------------------------------ behaviour
def test_deterministic_input_untouched_and_graph_capturable():
    from pose2mesh_release_b200.render import render_meshes

    W, H = 800, 600
    verts, faces, cams, colors = people("smpl", 4, W, H, seed=21)
    imgs = images(2, H, W, 4)
    before = imgs.clone()
    idx = cuda(np.array([0, 1, 0, 1], np.int32))
    f = cuda(faces.astype(np.int32))
    a = render_meshes(imgs, verts, f, cams, colors, image_index=idx, return_maps=True)
    b = render_meshes(imgs, verts, f, cams, colors, image_index=idx, return_maps=True)
    assert torch.equal(imgs, before)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x,
                           y.view(torch.uint8) if y.is_floating_point() else y)
    empty = a[1] < 0
    assert empty.any() and torch.equal(a[0][empty], imgs[empty])
    single = render_meshes(imgs[1], verts[1:2], f, cams[1:2], colors[1:2])
    assert single.shape == (H, W, 3)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        render_meshes(imgs, verts, f, cams, colors, image_index=idx, return_maps=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = render_meshes(imgs, verts, f, cams, colors, image_index=idx, return_maps=True)
    for t in c:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(a, c):
        assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x,
                           y.view(torch.uint8) if y.is_floating_point() else y)


def test_argument_errors():
    from pose2mesh_release_b200.render import render_meshes

    verts, faces, cams, colors = people("mano", 2, 224, 224, seed=5)
    imgs = images(1, 224, 224, 0)
    with pytest.raises(ValueError, match="faces"):
        render_meshes(imgs, verts, np.array([[0, 1, 778]]), cams, colors)
    with pytest.raises(ValueError, match="cams"):
        render_meshes(imgs, verts, faces, cams[:1], colors)
    with pytest.raises(ValueError, match="uint8"):
        render_meshes(imgs.float(), verts, faces, cams, colors)
    with pytest.raises(ValueError, match="65535"):
        render_meshes(imgs, verts, np.zeros((65536, 3), np.int32), cams, colors)
    with pytest.raises(ValueError, match="image_index"):
        render_meshes(imgs, verts, faces, cams, colors, image_index=cuda(np.zeros(3, np.int32)))
    with pytest.raises(RuntimeError, match="CUDA"):
        render_meshes(imgs, verts.cpu(), faces, cams, colors)
