"""The datasets' targets on the GPU (pose2mesh_release_b200.targets) against the float64 oracle
(oracle/targets_oracle.py) and the unmodified reference's outputs (tests/golden/targets.npz).

Bounds.  The body model itself is within 4e-6 of each sample's largest |coordinate| of float64
(test_gpu_body_model.py).  After it come at most four float32 roundings of the translation terms and of the mm scaling
(4 * 2^-24 of the sample's scale, 2.4e-7) and the float32 root rotation, which the kernel and the oracle round from
different fp64 computations and so may differ by one ulp of the angle (2^-24 pi, a 2e-7 relative move of the mesh).
ORACLE_REL = 1e-5 of the sample's largest |coordinate| covers the sum with a factor of two; the golden adds the
reference's own float32 error of the same size (GOLDEN_REL = 2e-5).  The Human3.6M assembly works in fp64 on the
float32 mesh and rounds each output once, so its outputs inherit the mesh's bound (pixels: times 2 f / z).
"""
import os

import numpy as np
import pytest
import torch

import body_model_oracle as bo
import body_models as bm
from oracle import targets_oracle as to

from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer
from pose2mesh_release_b200.targets import PRESETS, Human36MTargets, camera_frame_coords

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "targets.npz"))
SMPL, MANO = bm.smpl_model(), bm.mano_model("right", False)
ORACLE_REL = 1e-5
GOLDEN_REL = 2e-5
SMPL_PRESETS = [p for p in PRESETS if p != "freihand"]


def dev():
    return torch.device("cuda:0")


def cuda(a):
    return None if a is None else torch.as_tensor(np.asarray(a, np.float32)).to(dev())


_LAYERS = {}


def layer(mano=False):
    key = "mano" if mano else "smpl"
    if key not in _LAYERS:
        m = MANO if mano else SMPL
        _LAYERS[key] = (ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"],
                                  m["betas"], m["hands_mean"], flat_hand_mean=False, side="right") if mano else
                        SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"],
                                  m["parents"], m["betas"]))
    return _LAYERS[key]


def rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                  2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                  2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1)
    return R.reshape(n, 3, 3).astype(np.float32)


def inputs(n, preset, seed):
    """Seeded pose, betas (every third sample all zero, every fifth with a |beta| > 3), trans, R, t as float32."""
    rng = np.random.RandomState(seed)
    mano = preset == "freihand"
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    pose = f32(rng.normal(0, 0.4, (n, 48 if mano else 72)))
    pose[:, :3] = bm.random_axisang(rng, n, 0.05, 3.1)
    betas = f32(np.clip(rng.normal(0, 1.0, (n, 10)), -2.9, 2.9))
    betas[2::3] = 0
    betas[4::5, 7] = -3.5
    trans = f32(rng.normal(0, 0.3, (n, 3)))
    t = f32(rng.normal(0, 0.05 if mano else 0.3, (n, 3)) + ([0, 0, 0.5] if mano else [0, 0, 4.0]))
    if preset == "human36m":
        t = t * 1000
    return pose, betas, trans, rotations(rng, n), t


def oracle(preset, pose, betas, trans, R, t):
    mano = preset == "freihand"
    m = MANO if mano else SMPL
    fwd = (lambda q, b, tr: bo.mano_forward(m, q, b, tr)) if mano else (lambda q, b, tr: bo.smpl_forward(m, q, b, tr))
    return to.camera_frame(fwd, m["betas"], preset, pose, betas, trans, R, t, mano=mano)


def device(preset, pose, betas, trans, R, t):
    mesh, joints = camera_frame_coords(layer(preset == "freihand"), preset, cuda(pose), cuda(betas), cuda(trans),
                                       cuda(R), cuda(t))
    torch.cuda.synchronize()
    return mesh.cpu().numpy().astype(np.float64), joints.cpu().numpy().astype(np.float64)


def assert_close(got, want, rel, what=""):
    """Element-wise, per sample: |got - want| <= rel * the sample's largest |want|."""
    for b in range(want.shape[0]):
        scale = np.abs(want[b]).max()
        err = np.abs(got[b] - want[b]).max()
        assert err <= rel * scale, f"{what} sample {b}: {err:.3e} > {rel:.1e} * {scale:.3e}"


# ------------------------------------------------------------------------------------------------ accuracy
SIZES = [("human36m", b) for b in (1, 15, 16, 17, 256, 1000)] + \
        [(p, b) for p in SMPL_PRESETS if p != "human36m" for b in (1, 17, 256)] + [("freihand", 1), ("freihand", 1024)]


@pytest.mark.parametrize("preset,B", SIZES)
def test_camera_frame_vs_oracle(preset, B):
    args = inputs(B, preset, seed=B + 7 * len(preset))
    gm, gj = device(preset, *args)
    om, oj = oracle(preset, *args)
    scale = np.maximum(np.abs(om).max(axis=(1, 2)), np.abs(oj).max(axis=(1, 2)))[:, None, None]
    assert (np.abs(gm - om) <= ORACLE_REL * scale).all(), np.abs(gm - om).max(axis=(1, 2)).max()
    assert (np.abs(gj - oj) <= ORACLE_REL * scale).all(), np.abs(gj - oj).max(axis=(1, 2)).max()


@pytest.mark.parametrize("preset", PRESETS)
def test_camera_frame_vs_golden(preset):
    args = [GOLDEN[f"{preset}__{k}"] for k in ("pose", "betas", "trans", "R", "t")]
    gm, gj = device(preset, *args)
    rows = slice(None) if preset == "freihand" else GOLDEN["rows"]
    scale = np.maximum(np.abs(gm).max(axis=(1, 2)), np.abs(gj).max(axis=(1, 2)))[:, None, None]
    assert (np.abs(gm[:, rows] - GOLDEN[f"{preset}__mesh"]) <= GOLDEN_REL * scale).all()
    assert (np.abs(gj - GOLDEN[f"{preset}__joints"]) <= GOLDEN_REL * scale).all()


def h36m_module(joint_set):
    return Human36MTargets(layer(), GOLDEN["reg_h36m"], GOLDEN["reg_coco"], joint_set)


def h36m_inputs(B, seed, noise=(4.0, 60.0)):
    """The human36m preset's inputs and an annotation joint_cam near the fitted mesh's H36M joints: even samples
    within `noise[0]` mm per coordinate (fit error well below 25 mm), odd ones `noise[1]` (well above)."""
    pose, betas, trans, R, t = inputs(B, "human36m", seed)
    rng = np.random.RandomState(seed + 1)
    mesh, _ = oracle("human36m", pose, betas, trans, R, t)
    reg = np.einsum("jv,bvc->bjc", GOLDEN["reg_h36m"], mesh)
    sd = np.where(np.arange(B) % 2 == 0, noise[0], noise[1])[:, None, None]
    joint_cam = np.asarray(reg + sd * rng.normal(size=reg.shape), np.float32)
    f = np.asarray(rng.uniform(1100, 1200, (B, 2)), np.float32)
    c = np.asarray(rng.uniform(480, 540, (B, 2)), np.float32)
    return (pose, betas, trans, R, t, f, c, joint_cam), mesh


def run_h36m(mod, args):
    out = mod(*[cuda(a) for a in args])
    torch.cuda.synchronize()
    return {k: v.cpu().numpy().astype(np.float64) for k, v in out.items()}


@pytest.mark.parametrize("joint_set", ["human36", "coco"])
@pytest.mark.parametrize("B", [1, 17, 256])
def test_h36m_targets_vs_oracle(joint_set, B):
    args, mesh_cam = h36m_inputs(B, seed=100 + B)
    got = run_h36m(h36m_module(joint_set), args)
    want = to.h36m_targets(mesh_cam, args[7], args[5], args[6], GOLDEN["reg_h36m"], GOLDEN["reg_coco"], joint_set)
    scale = np.abs(mesh_cam).max(axis=(1, 2))
    for k, s in (("mesh", scale / 1000), ("lift_pose3d", scale), ("reg_pose3d", scale)):
        assert (np.abs(got[k] - want[k]).max(axis=(1, 2)) <= ORACLE_REL * s).all(), k
    assert (np.abs(got["joint_img"] - want["joint_img"]).max(axis=(1, 2)) <= ORACLE_REL * (2 * 1200 + scale)).all()
    assert (np.abs(got["fitting_error"] - want["fitting_error"]) <= ORACLE_REL * scale).all()
    err = want["fitting_error"]
    assert not ((err > 20) & (err < 30)).any()  # a safe margin either side of the 25 mm threshold
    for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["joint_valid"], got["lift_pose3d_valid"])
    assert (got["mesh_valid"][0::2] == 1).all() and (got["mesh_valid"][1::2] == 0).all()


@pytest.mark.parametrize("joint_set", ["human36", "coco"])
def test_h36m_targets_vs_golden(joint_set):
    args = [GOLDEN[f"human36m__{k}"] for k in ("pose", "betas", "trans", "R", "t")] + \
           [GOLDEN[f"h36m__{k}"] for k in ("f", "c", "joint_cam")]
    got = run_h36m(h36m_module(joint_set), args)
    rows = GOLDEN["rows"]
    g = lambda k: GOLDEN[f"h36m_{joint_set}__{k}"]  # noqa: E731
    scale = np.abs(g("lift_pose3d")).max() + np.abs(args[7]).max()
    assert np.abs(got["mesh"][:, rows] - g("mesh")).max() <= GOLDEN_REL * scale / 1000
    assert np.abs(got["lift_pose3d"] - g("lift_pose3d")).max() <= GOLDEN_REL * scale
    assert np.abs(got["reg_pose3d"] - g("reg_pose3d")).max() <= GOLDEN_REL * scale
    assert np.abs(got["joint_img"] - g("joint_img")).max() <= GOLDEN_REL * (2 * 1200 + scale)
    assert np.abs(got["fitting_error"] - g("fitting_error")).max() <= GOLDEN_REL * scale
    assert np.array_equal(got["mesh_valid"][:, rows], g("mesh_valid"))
    assert np.array_equal(got["lift_pose3d_valid"], g("lift_pose3d_valid"))


# ------------------------------------------------------------------------------------------------ rotation edges
def rotvec_matrix(v):
    from scipy.spatial.transform import Rotation
    return Rotation.from_rotvec(np.asarray(v, np.float64)).as_matrix()


@pytest.mark.parametrize("preset", ["human36m", "amass"])
def test_root_rotation_edges(preset):
    """Roots whose rotated angle is near 0, near pi and exactly pi, and exactly zero roots (which give R's own
    rotation), compared as meshes and joints against the oracle (scipy's rotations, independent of the kernel's log
    map; at pi the two may pick opposite axis-angle vectors of the same rotation)."""
    n = 8
    pose, betas, trans, R, t = inputs(n, preset, seed=5)
    axes = np.random.RandomState(6).normal(size=(n, 3))
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    Rt = np.transpose(R, (0, 2, 1)).astype(np.float64)
    from scipy.spatial.transform import Rotation
    # root = log(R^T exp(w)) so that R exp(root) = exp(w), for target angles |w| near 0 and near pi
    angles = np.array([1e-7, 1e-5, 1e-3, np.pi - 1e-3, np.pi - 1e-6, np.pi, 0.0, 0.0])
    target = axes * angles[:, None]
    root = Rotation.from_matrix(Rt @ rotvec_matrix(target)).as_rotvec()
    root[6] = 0.0
    root[7] = 0.0
    pose[:, :3] = root.astype(np.float32)
    gm, gj = device(preset, pose, betas, trans, R, t)
    om, oj = oracle(preset, pose, betas, trans, R, t)
    assert_close(gm, om, ORACLE_REL, "mesh")
    assert_close(gj, oj, ORACLE_REL, "joints")


# ------------------------------------------------------------------------------------------------ per-sample quirks
@pytest.mark.parametrize("preset", ["human36m", "muco", "coco", "freihand"])
def test_per_sample_betas_rules(preset):
    """Zero-betas, clamped-betas and normal samples in one batch: each matches its own B = 1 call bit for bit and
    its own B = 1 oracle call."""
    B = 18
    args = inputs(B, preset, seed=42)
    gm, gj = device(preset, *args)
    for b in (0, 1, 2, 4, 5, 14):
        one = [a[b:b + 1] for a in args]
        m1, j1 = device(preset, *one)
        assert np.array_equal(m1[0], gm[b]) and np.array_equal(j1[0], gj[b])
        om, oj = oracle(preset, *one)
        assert_close(m1, om, ORACLE_REL, f"sample {b}")
    if preset != "freihand":  # a zero row (sample 2) and, under the clamp, a row with |beta| > 3 (sample 4) both
        # take the model's betas: the same bits as the model's betas given explicitly
        for b in (2, 4) if PRESETS[preset].flags & _lib.P2M_FRAME_CLAMP_BETAS else (2,):
            one = [a[b:b + 1].copy() for a in args]
            one[1][0] = SMPL["betas"]
            m1, _ = device(preset, *one)
            assert np.array_equal(m1[0], gm[b])


# ------------------------------------------------------------------------------------------------ robustness
def test_determinism_position_and_nan_isolation():
    B = 40
    pose, betas, trans, R, t = inputs(B, "human36m", seed=9)
    a = device("human36m", pose, betas, trans, R, t)
    b = device("human36m", pose, betas, trans, R, t)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    perm = np.random.RandomState(3).permutation(B)
    c = device("human36m", pose[perm], betas[perm], trans[perm], R[perm], t[perm])
    assert np.array_equal(c[0], a[0][perm]) and np.array_equal(c[1], a[1][perm])
    pose2 = pose.copy()
    pose2[7, 5] = np.nan
    d = device("human36m", pose2, betas, trans, R, t)
    keep = np.arange(B) != 7
    assert np.array_equal(d[0][keep], a[0][keep]) and np.isnan(d[0][7]).any()
    args, _ = h36m_inputs(B, seed=11)
    mod = h36m_module("coco")
    x = run_h36m(mod, args)
    args2 = [a.copy() for a in args]
    args2[7][3, 2, 0] = np.nan
    y = run_h36m(mod, args2)
    for k in x:
        assert np.array_equal(np.delete(x[k], 3, 0), np.delete(y[k], 3, 0)), k


def test_graph_capture_and_launch_count():
    lib = _lib.load()
    B = 32
    args, _ = h36m_inputs(B, seed=21)
    mod = h36m_module("human36")
    dargs = [cuda(a) for a in args]
    eager = {k: v.clone() for k, v in mod(*dargs).items()}
    torch.cuda.synchronize()
    lib.p2m_launch_count_reset()
    mod(*dargs)
    assert lib.p2m_launch_count() == Human36MTargets.LAUNCHES
    lib.p2m_launch_count_reset()
    camera_frame_coords(layer(), "muco", dargs[0], dargs[1], dargs[2])
    assert lib.p2m_launch_count() == 5
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mod(*dargs)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = mod(*dargs)
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


# ------------------------------------------------------------------------------------------------ argument errors
def test_argument_errors():
    pose, betas, trans, R, t = [cuda(a) for a in inputs(4, "human36m", seed=1)]
    L = layer()
    with pytest.raises(RuntimeError):
        camera_frame_coords(L, "human36m", pose.cpu(), betas, trans, R, t)
    with pytest.raises(RuntimeError):
        camera_frame_coords(L, "human36m", pose, betas, trans, R.cpu(), t)
    with pytest.raises(ValueError):
        camera_frame_coords(L, "human36m", pose, betas[:3], trans, R, t)
    with pytest.raises(ValueError):
        camera_frame_coords(L, "human36m", pose, betas, trans, R[:, :2], t)
    with pytest.raises(ValueError):
        camera_frame_coords(L, "human36m", pose, betas, None, R, t)
    with pytest.raises(ValueError):
        camera_frame_coords(L, "nope", pose, betas, trans, R, t)
    with pytest.raises(ValueError):
        camera_frame_coords(layer(mano=True), "human36m", pose[:, :48], betas, trans, R, t)
    with pytest.raises(ValueError):
        camera_frame_coords(L, "freihand", pose, betas, trans, R, t)
    with pytest.raises(ValueError):
        Human36MTargets(L, GOLDEN["reg_h36m"][:, :100], GOLDEN["reg_coco"])
    with pytest.raises(ValueError):
        Human36MTargets(L, GOLDEN["reg_h36m"], GOLDEN["reg_coco"], "mpii")
    mod = h36m_module("human36")
    f = cuda(np.ones((4, 2)))
    with pytest.raises(ValueError):
        mod(pose, betas, trans, R, t, f, f, cuda(np.ones((4, 16, 3))))
    with pytest.raises(RuntimeError):
        mod(pose, betas, trans, R, t, f.cpu(), f, cuda(np.ones((4, 17, 3))))
    # the C entry points check what the Python layer does not: a host array among the data arrays
    nbytes = _lib.load().p2m_camera_frame_workspace_bytes(L.handle(0), 4)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    st = lib_call_status("p2m_camera_frame_coords", L.handle(0), 0, pose.data_ptr(), betas.data_ptr(), None, None,
                         None, None, 0, pose.data_ptr(), pose.data_ptr(), 4, ws.data_ptr(), nbytes)
    assert st == 1 and b"device memory" in _lib.load().p2m_last_error()


def lib_call_status(name, *args):
    return getattr(_lib.load(), name)(*args, None)


# ------------------------------------------------------------------------------------------------ drop-in use
def test_outputs_feed_the_losses():
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L

    B = 8
    args, _ = h36m_inputs(B, seed=31)
    tg = h36m_module("coco")(*[cuda(a) for a in args])
    g = torch.Generator().manual_seed(1)
    face = pg.synthetic_sphere_faces(6890, 2)
    coord_loss, normal_loss, edge_loss, _, _ = L.get_loss(face)
    pred_mesh = tg["mesh"] + 0.01 * torch.randn(tg["mesh"].shape, generator=g).to(dev())
    pred_lift = tg["lift_pose3d"] + torch.randn(tg["lift_pose3d"].shape, generator=g).to(dev())
    lm = coord_loss(pred_mesh, tg["mesh"], tg["mesh_valid"])
    ll = coord_loss(pred_lift, tg["lift_pose3d"], tg["lift_pose3d_valid"])
    ln, le = normal_loss(pred_mesh, tg["mesh"]), edge_loss(pred_mesh, tg["mesh"])
    v = tg["mesh_valid"]
    want_m = ((pred_mesh * v - tg["mesh"] * v).abs()).mean()
    want_l = ((pred_lift * tg["lift_pose3d_valid"] - tg["lift_pose3d"] * tg["lift_pose3d_valid"]).abs()).mean()
    assert abs(lm.item() - want_m.item()) <= 1e-5 * max(1.0, want_m.item())
    assert abs(ll.item() - want_l.item()) <= 1e-5 * max(1.0, want_l.item())
    assert torch.isfinite(ln) and torch.isfinite(le)
    assert (tg["mesh_valid"][1::2] == 0).all()  # the dropped samples contribute nothing
