"""The demo's camera fit on the GPU (SURVEY.md §8 row f7, pose2mesh_release_b200.camera) against

  * oracle/camera_oracle.py::fit_f32_kernel_order, the kernel's operation order in float32 numpy: bit for bit;
  * the unmodified reference (tests/golden/camera_fit.npz): crop target and box bit for bit, camera and loss within
    2 x the spread of the reference's own one-ulp rerun (tests/camera_cases.py)."""
import numpy as np
import pytest
import torch

import camera_cases as cc
from helpers import graph_from_fixture
from oracle import camera_oracle as co

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def synthetic(B, seed, kind="f64", n_in=17):
    """Image poses [B, n_in, 2 | 3] of the given dtype kind, 3-D joints [B, 17, 3] and inits [B, 3]."""
    g = np.random.default_rng(seed)
    p3d = g.normal(0, 0.3, (B, 17, 3)).astype(np.float32)
    s, t = g.uniform(0.6, 1.3, (B, 1, 1)), g.normal(0, 0.1, (B, 1, 2))
    S, O = g.uniform(80, 300, (B, 1, 1)), g.uniform(100, 600, (B, 1, 2))
    px = np.concatenate([(p3d[:, :, :2] + t) * s * S + O + g.normal(0, 3, (B, 17, 2)),
                         g.uniform(100, 600, (B, n_in - 17, 2))], 1)
    if kind == "int":
        px = np.round(px).astype(np.int64)
    elif kind == "f32":
        px = px.astype(np.float32)
    elif kind == "coco":
        px = np.concatenate([px, g.uniform(0, 1, (B, n_in, 1))], 2)
    return px, p3d, g.uniform(0, 1, (B, 3)).astype(np.float32)


def oracle(px, p3d, init, wh=None, **kw):
    bbox, tgt = co.crop_targets(px)
    cam, loss = co.fit_f32_kernel_order(p3d, tgt, init, **kw)
    out = {"cam_param": cam, "bbox": bbox, "target": tgt, "loss": loss}
    if wh is not None:
        ok = ~np.isnan(bbox).any(1)
        orig = co.orig_cam_f32(cam, bbox, wh[:, 0], wh[:, 1])
        orig[~ok] = np.nan
        out["orig_cam"] = orig
    return out


def assert_bitwise(got, ref):
    for k, v in ref.items():
        g = got[k].cpu().numpy()
        assert g.shape == v.shape, k
        assert np.array_equal(g, v, equal_nan=True), (k, np.argwhere(~((g == v) | (np.isnan(g) & np.isnan(v))))[:5])


# ------------------------------------------------------------------------------------------------ kernel order
@pytest.mark.parametrize("B", [1, 7, 64, 1000])
def test_bitwise_equal_to_kernel_order_oracle(B):
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(B, seed=B)
    wh = np.stack([np.full(B, 1280.0), np.full(B, 720.0)], 1).astype(np.float32)
    got = fit_cameras(cuda(px), cuda(p3d), init=cuda(init), image_size=cuda(wh))
    assert_bitwise(got, oracle(px, p3d, init, wh))


@pytest.mark.parametrize("kind", ["int", "f32", "coco"])
def test_input_dtypes_bitwise_equal_to_kernel_order_oracle(kind):
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(48, seed=5, kind=kind, n_in=19 if kind == "coco" else 17)
    got = fit_cameras(cuda(px), cuda(p3d), init=cuda(init))
    assert_bitwise(got, oracle(px, p3d, init))


def test_short_schedule_bitwise_equal_to_kernel_order_oracle():
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(16, seed=9)
    sched = ((0, 0.2), (3, 0.01), (40, 0.3), (41, 0.02))
    got = fit_cameras(cuda(px), cuda(p3d), init=cuda(init), n_iter=77, lr_schedule=sched, crop_size=333)
    bbox, tgt = co.crop_targets(px, crop=333)
    cam, loss = co.fit_f32_kernel_order(p3d, tgt, init, crop=333, n_iter=77, schedule=sched)
    assert_bitwise(got, {"cam_param": cam, "loss": loss, "bbox": bbox, "target": tgt})


# ------------------------------------------------------------------------------------------------ reference fixture
def _fixture_groups(z):
    """(case indices, joints array) per input dtype / row count of the fixture."""
    kinds = z["kind"]
    return [([cc.DEMO], z["joints_demo"][None]),
            (list(np.nonzero(kinds == 1)[0]), z["joints_h36m_int"]),
            (list(np.nonzero(kinds == 2)[0]), z["joints_h36m_f64"]),
            (list(cc.COCO), z["joints_coco"]),
            ([cc.ZERO], z["joints_zero"][None])]


def test_reference_fixture():
    from pose2mesh_release_b200.camera import fit_cameras

    z = cc.fixture()
    targets = cc.targets(z)
    cam = np.zeros((cc.N_CASES, 3), np.float32)
    loss = np.zeros(cc.N_CASES, np.float32)
    for cases, joints in _fixture_groups(z):
        wh = z["img_wh"][cases].astype(np.float32)
        got = fit_cameras(cuda(joints), cuda(z["pred_joints3d"][cases]), init=cuda(z["init"][cases]),
                          image_size=cuda(wh))
        assert np.array_equal(got["bbox"].cpu().numpy(), z["bbox"][cases])
        assert np.array_equal(got["target"].cpu().numpy(), np.stack([targets[i] for i in cases]))
        assert_bitwise(got, oracle(joints, z["pred_joints3d"][cases], z["init"][cases], wh))
        cam[cases], loss[cases] = got["cam_param"].cpu().numpy(), got["loss"].cpu().numpy()
    assert cc.violations(z, cam, loss) == []
    assert np.array_equal(cam[cc.ZERO], [1, 0, 0]) and loss[cc.ZERO] == 0


def test_demo_pose_end_to_end():
    """demo/run.py:150-189 at B = 1 on native kernels: normalize_pose2d -> FlatPose2Mesh.predict_vertices_and_joints ->
    fit_cameras, with the model and joint regressor make_golden_camera.py used for case 0."""
    from oracle import meshnet_oracle as mo
    from pose2mesh_release_b200 import pose2mesh_net, postprocess
    from pose2mesh_release_b200.camera import fit_cameras

    z = cc.fixture()
    mats, zg = graph_from_fixture("smpl_small")
    torch.manual_seed(123)
    flat = pose2mesh_net.get_model(17, mats)
    sd = {k: v.detach().clone() for k, v in flat.state_dict().items()}
    mo.randomize_bn_({("bn." + k): v for k, v in sd.items() if "batch_norm" in k or ".bn." in k}, seed=3)
    flat.load_state_dict(sd)
    flat = flat.to(dev()).eval()
    jr = torch.rand(17, 1200, generator=torch.Generator().manual_seed(6))
    jr = jr / jr.sum(1, keepdim=True)
    joints_px = cuda(z["joints_demo"])[None]                                   # int64, as the demo loads it
    pose2d = postprocess.normalize_pose2d(joints_px)
    _, joints, _ = flat.predict_vertices_and_joints(pose2d, np.asarray(zg["perm_reverse"]), 1200, jr.to(dev()))
    wh = z["img_wh"][:1].astype(np.float32)
    got = fit_cameras(joints_px, joints, init=cuda(z["init"][:1]), image_size=cuda(wh))
    assert np.array_equal(got["bbox"].cpu().numpy(), z["bbox"][:1])
    assert np.array_equal(got["target"].cpu().numpy()[0], cc.targets(z)[0])
    assert_bitwise(got, oracle(z["joints_demo"][None], joints.cpu().numpy(), z["init"][:1], wh))
    assert cc.violations(z, got["cam_param"].cpu().numpy(), got["loss"].cpu().numpy(), [cc.DEMO]) == []


# ------------------------------------------------------------------------------------------------ behaviour
def test_seeded_default_init_follows_the_reference_draws():
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, _ = synthetic(5, seed=3)
    torch.manual_seed(42)
    got = fit_cameras(cuda(px), cuda(p3d), n_iter=10)
    torch.manual_seed(42)
    init = torch.cat([torch.nn.Parameter(torch.rand((1, 3))).detach() for _ in range(5)])  # project_net.py:12, per person
    ref = fit_cameras(cuda(px), cuda(p3d), init=init.to(dev()), n_iter=10)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
    assert torch.equal(fit_cameras(cuda(px), cuda(p3d), init=init.to(dev()), n_iter=0)["cam_param"].cpu(), init)


def test_deterministic_and_independent_of_batch_position():
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(200, seed=11)
    a = fit_cameras(cuda(px), cuda(p3d), init=cuda(init))
    b = fit_cameras(cuda(px), cuda(p3d), init=cuda(init))
    perm = np.random.default_rng(0).permutation(200)
    c = fit_cameras(cuda(px[perm]), cuda(p3d[perm]), init=cuda(init[perm]))
    single = fit_cameras(cuda(px[17:18]), cuda(p3d[17:18]), init=cuda(init[17:18]))
    for k in a:
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(a[k][torch.as_tensor(perm, device=dev())], c[k]), k
        assert torch.equal(a[k][17:18], single[k]), k


def test_nan_isolation():
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(8, seed=13)
    clean = fit_cameras(cuda(px), cuda(p3d), init=cuda(init), image_size=(640, 480))
    bad = px.copy()
    bad[2] = bad[2, :1]              # every joint at one point: process_bbox returns None
    bad[5, 3, 1] = np.nan            # one NaN joint
    got = fit_cameras(cuda(bad), cuda(p3d), init=cuda(init), image_size=(640, 480))
    keep = [0, 1, 3, 4, 6, 7]
    for k in clean:
        assert torch.equal(got[k][keep], clean[k][keep]), k
        assert torch.isnan(got[k][[2, 5]]).all(), k


def test_cuda_graph_replay_matches_eager():
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(32, seed=17)
    x, p, i0 = cuda(px), cuda(p3d), cuda(init)
    wh = cuda(np.array([[800.0, 600.0]], np.float32))
    eager = fit_cameras(x, p, init=i0, image_size=wh)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fit_cameras(x, p, init=i0, image_size=wh)
    torch.cuda.current_stream().wait_stream(s)
    x_in = x.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fit_cameras(x_in, p, init=i0, image_size=wh)
    x_in.copy_(x)
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k
    px2 = px + 7
    x_in.copy_(cuda(px2))                        # replays follow the data
    g.replay()
    torch.cuda.synchronize()
    ref = fit_cameras(cuda(px2), p, init=i0, image_size=wh)
    for k in ref:
        assert torch.equal(out[k], ref[k]), k


def test_one_launch():
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(300, seed=19)
    x, p, i0, wh = cuda(px), cuda(p3d), cuda(init), cuda(np.array([[640.0, 480.0]], np.float32))
    fit_cameras(x, p, init=i0, image_size=wh)
    lib = _lib.load()
    lib.p2m_launch_count_reset()
    fit_cameras(x, p, init=i0, image_size=wh)
    assert lib.p2m_launch_count() == 1


def test_convert_crop_cam_to_orig_img_alone():
    from pose2mesh_release_b200.camera import convert_crop_cam_to_orig_img

    g = np.random.default_rng(23)
    cam = g.uniform(0.5, 1.5, (50, 3)).astype(np.float32)
    bbox = np.concatenate([g.uniform(0, 300, (50, 2)), g.uniform(50, 400, (50, 1)).repeat(2, 1)], 1).astype(np.float32)
    got = convert_crop_cam_to_orig_img(cuda(cam), cuda(bbox), 1024, 768).cpu().numpy()
    assert np.array_equal(got, co.orig_cam_f32(cam, bbox, 1024, 768))


def test_argument_errors():
    from pose2mesh_release_b200.camera import fit_cameras

    px, p3d, init = synthetic(4, seed=1)
    x, p, i0 = cuda(px), cuda(p3d), cuda(init)
    with pytest.raises(RuntimeError, match="bad argument"):           # J > 32
        fit_cameras(cuda(np.tile(px, (1, 3, 1))[:, :40]), cuda(np.tile(p3d, (1, 3, 1))[:, :33]), init=i0)
    with pytest.raises(RuntimeError, match="bad argument"):           # J > Jin
        fit_cameras(x[:, :16], p, init=i0)
    with pytest.raises(RuntimeError, match="CUDA"):
        fit_cameras(torch.from_numpy(px), p, init=i0)
    with pytest.raises(RuntimeError, match="CUDA"):
        fit_cameras(x, torch.from_numpy(p3d), init=i0)
    with pytest.raises(RuntimeError, match="schedule"):
        fit_cameras(x, p, init=i0, lr_schedule=())
    with pytest.raises(ValueError, match="requires grad"):
        fit_cameras(x, p.clone().requires_grad_(True), init=i0)
