"""The training sample's augmentation on the GPU (inputs.augm_params, training_pose2d(rot, flip, flip_before_noise),
Human36MTargets(rot, flip)) against oracle/samples_oracle.py on the same seeds and against the unmodified reference
(tests/golden/samples.npz).

Bounds.  augm_params' flips and zeroed rotations are decisions on the same uniforms as the oracle's, so they are
equal; a rotation is one float32 rounding of an fp64 value whose log / cos differ from numpy's by a few fp64 ulps: one
float32 ulp.  The rotated crop map is fp64 from float32 point pairs; the device's (sin, cos)(pi rot / 180) differ from
numpy's by a few fp64 ulps, so a crop point is within one float32 ulp of the oracle's (of the pre-flip value for a
flipped x, which the flip subtracts from the width in float32).  The normalised pose2d is then compared with
test_gpu_inputs.py's 1e-5.  The lift target is fp64 rotated and rounded once: one float32 ulp of the row's largest
|x|, |y| beyond the unaugmented target's own bound.
"""
import numpy as np
import pytest
import torch

from oracle import samples_oracle as so
from inputs_cases import P_FAIL, chi2_p, error_table, ordered_table
from oracle import inputs_oracle as io
from oracle import targets_oracle as to
from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200.inputs import Human36MErrorModel, augm_params, training_pose2d
from pose2mesh_release_b200.targets import AMASSTargets, COCOTargets, MuCoTargets
from test_gpu_targets import GOLDEN as TGOLDEN
from test_gpu_targets import ORACLE_REL, cuda, h36m_inputs, h36m_module, inputs, layer, oracle
from test_samples_cpu import GOLDEN, within_ulp

pytestmark = pytest.mark.gpu
SEED = (0x5EED_0001_2345_6789, 0x0000_00AB_CDEF_0123)


def dev():
    return torch.device("cuda:0")


def seed_t(seed=SEED):
    return torch.tensor([np.int64(np.uint64(seed[0])), np.int64(np.uint64(seed[1]))], dtype=torch.int64,
                        device=dev())


def poses(B, J, rng):
    """Image-pixel poses with wide and tall boxes."""
    centre = rng.uniform([200, 200], [1000, 800], (B, 1, 2))
    size = rng.uniform(60, 500, (B, 1, 1)) * np.where(np.arange(B) % 2 == 0, 1.0, 0.4)[:, None, None]
    wide = np.where(np.arange(B) % 3 == 0, 1.6, 0.5)[:, None, None]
    off = rng.uniform(-1, 1, (B, J, 2)) * np.concatenate([size * wide, size], 2)
    return (centre + off).astype(np.float32)


def aug_for(B, rng):
    """Every combination of flip and a zero / nonzero rotation, then random ones."""
    flip = rng.integers(0, 2, B).astype(np.int32)
    rot = np.where(rng.uniform(size=B) < 0.3, 0.0, rng.uniform(-60, 60, B)).astype(np.float32)
    for i, (f, r) in enumerate(((0, 0.0), (1, 0.0), (0, 17.3), (1, -40.0))[:B]):
        flip[i], rot[i] = f, r
    return flip, rot


@pytest.mark.parametrize("B", [1, 7, 256, 1000])
def test_augm_params_match_oracle(B):
    for flip, rf in ((True, 30.0), (False, 30.0), (True, 0.0)):
        f, r = augm_params(B, flip, rf, seed_t())
        wf, wr = so.augm_params(B, flip, rf, SEED)
        np.testing.assert_array_equal(f.cpu().numpy(), wf)
        got = r.cpu().numpy()
        np.testing.assert_array_equal(got == 0, wr == 0)
        assert within_ulp(got, wr).all()
        assert f.dtype == torch.int32 and r.dtype == torch.float32


@pytest.mark.parametrize("k", range(4))
def test_augm_params_match_reference_counts(k):
    fl, rf = GOLDEN["augm_settings"][k]
    M, nb = int(GOLDEN["augm_M"]), int(GOLDEN["augm_bins"])
    f, r = (t.cpu().numpy() for t in augm_params(M, bool(fl), rf, seed_t((0xC0FFEE, 5 + k))))
    ref_flip, ref_zero = int(GOLDEN["augm_flips"][k]), int(GOLDEN["augm_zero"][k])
    ps = [chi2_p(np.array([ref_flip, M - ref_flip]), np.array([f.sum(), M - f.sum()])),
          chi2_p(np.array([ref_zero, M - ref_zero]), np.array([(r == 0).sum(), M - (r == 0).sum()]))]
    if rf > 0:
        nz = r[r != 0].astype(np.float64)
        ps.append(chi2_p(GOLDEN["augm_hist"][k], np.histogram(nz, bins=nb, range=(-2 * rf, 2 * rf))[0]))
    else:
        assert (r == 0).all()
    assert min(ps) > P_FAIL, ps


@pytest.mark.parametrize("joint_set", ["coco", "human36"])
@pytest.mark.parametrize("flip_before_noise", [False, True])
def test_crop_matches_reference_fixture(joint_set, flip_before_noise):
    """No noise: the normalised device output against the reference's crop normalised in float64."""
    joints = GOLDEN[f"{joint_set}__joints"]
    want = GOLDEN[f"{joint_set}__crop_{'before' if flip_before_noise else 'after'}"]
    C_ = joints.shape[0]
    for a in range(want.shape[1]):
        fl, rot = GOLDEN["aug_cases"][a]
        if rot == 0:
            continue                     # the rot-0 path is the existing closed form (test_gpu_inputs.py)
        got = training_pose2d(torch.from_numpy(joints).to(dev()), joint_set, noise=False,
                              rot=torch.full((C_,), float(rot), device=dev()),
                              flip=torch.full((C_,), int(fl), device=dev(), dtype=torch.int32),
                              flip_before_noise=flip_before_noise).cpu().numpy()
        np.testing.assert_allclose(got, io.normalize(want[:, a]), atol=1e-5, rtol=0)


@pytest.mark.parametrize("B", [1, 7, 256, 1000])
@pytest.mark.parametrize("noise", ["none", "coco", "h36m"])
@pytest.mark.parametrize("flip_before_noise", [False, True])
def test_training_pose2d_augmented_matches_oracle(B, noise, flip_before_noise):
    rng = np.random.default_rng(B * 7 + len(noise))
    joint_set = "human36" if noise == "h36m" else "coco"
    J = 17 if joint_set == "human36" else 19
    px = poses(B, J, rng)
    flip, rot = aug_for(B, rng)
    model = Human36MErrorModel(*error_table())
    got = training_pose2d(torch.from_numpy(px).to(dev()), joint_set, noise=noise != "none", error_model=model,
                          seed=seed_t(), rot=torch.from_numpy(rot).to(dev()), flip=torch.from_numpy(flip).to(dev()),
                          flip_before_noise=flip_before_noise).cpu().numpy()
    rows = np.arange(B) if B <= 256 else np.unique(np.r_[0:8, B - 8:B, 0:B:37])
    want, _ = so.training_pose2d(px, noise, joint_set, SEED, ordered_table(), rot=rot, flip=flip,
                                 flip_before_noise=flip_before_noise)
    np.testing.assert_allclose(got[rows], want[rows], atol=1e-5, rtol=0)


@pytest.mark.parametrize("noise", ["coco", "h36m"])
def test_noise_order(noise):
    """The same seed and flips: the device matches the oracle's order and differs from the other one."""
    B = 256
    rng = np.random.default_rng(5)
    joint_set = "human36" if noise == "h36m" else "coco"
    px = poses(B, 17 if joint_set == "human36" else 19, rng)
    flip = np.ones(B, np.int32)
    rot = np.zeros(B, np.float32)
    model = Human36MErrorModel(*error_table())
    for before in (False, True):
        got = training_pose2d(torch.from_numpy(px).to(dev()), joint_set, error_model=model, seed=seed_t(),
                              flip=torch.from_numpy(flip).to(dev()), flip_before_noise=before).cpu().numpy()
        same, _ = so.training_pose2d(px, noise, joint_set, SEED, ordered_table(), rot=rot, flip=flip,
                                     flip_before_noise=before)
        other, _ = so.training_pose2d(px, noise, joint_set, SEED, ordered_table(), rot=rot, flip=flip,
                                      flip_before_noise=not before)
        np.testing.assert_allclose(got, same, atol=1e-5, rtol=0)
        assert (np.abs(got - other).max(axis=(1, 2)) > 1e-3).mean() > 0.5


def test_unaugmented_paths_are_bitwise():
    rng = np.random.default_rng(3)
    B = 300
    model = Human36MErrorModel(*error_table())
    z_rot, z_flip = torch.zeros(B, device=dev()), torch.zeros(B, dtype=torch.int32, device=dev())
    for joint_set, J, noise in (("coco", 19, True), ("human36", 17, True), ("coco", 19, False)):
        x = torch.from_numpy(poses(B, J, rng)).to(dev())
        for before in (False, True):
            kw = dict(noise=noise, error_model=model, seed=seed_t())
            base = training_pose2d(x, joint_set, **kw)
            assert torch.equal(base, training_pose2d(x, joint_set, rot=z_rot, flip=z_flip, flip_before_noise=before,
                                                     **kw))
    # the flip alone is exact: without noise it is the mirrored crop of the same map
    x = torch.from_numpy(poses(B, 19, rng)).to(dev())
    one = torch.ones(B, dtype=torch.int32, device=dev())
    a = training_pose2d(x, "coco", noise=False, flip=one)
    b = training_pose2d(x, "coco", noise=False, flip=one, flip_before_noise=True)
    assert torch.isfinite(a).all() and (a - b).abs().max() < 1e-5


@pytest.mark.parametrize("joint_set", ["human36", "coco"])
@pytest.mark.parametrize("B", [1, 7, 256, 1000])
def test_h36m_targets_augmented(joint_set, B):
    args, mesh_cam = h36m_inputs(B, seed=300 + B)
    mod = h36m_module(joint_set)
    cargs = [cuda(a) for a in args]
    rng = np.random.default_rng(B)
    flip, rot = aug_for(B, rng)
    base = mod(*cargs)
    aug = mod(*cargs, rot=torch.from_numpy(rot).to(dev()), flip=torch.from_numpy(flip).to(dev()))
    zero = mod(*cargs, rot=torch.zeros(B, device=dev()), flip=torch.zeros(B, dtype=torch.int32, device=dev()))
    for k in base:
        assert torch.equal(base[k], zero[k]), k
        if k != "lift_pose3d":
            assert torch.equal(base[k], aug[k]), k                       # only the lift target is augmented
    got = aug["lift_pose3d"].cpu().numpy().astype(np.float64)
    lift = base["lift_pose3d"].cpu().numpy().astype(np.float64)
    # a flip without rotation is exact: pairs swapped, x negated
    pure = (flip == 1) & (rot == 0)
    want = so.j3d_processing(lift, rot, flip, joint_set)
    np.testing.assert_array_equal(got[pure], want[pure])
    np.testing.assert_array_equal(got[(flip == 0) & (rot == 0)], lift[(flip == 0) & (rot == 0)])
    # rotated: against the oracle's float64 lift target
    ref = to.h36m_targets(mesh_cam, args[7], args[5], args[6], TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"],
                          joint_set)["lift_pose3d"]
    if joint_set == "human36":
        ref = ref.astype(np.float32).astype(np.float64)                  # the annotation's float32 rooting
    want = so.j3d_processing(ref, rot, flip, joint_set)
    scale = np.abs(mesh_cam).max(axis=(1, 2))
    xy = np.abs(want[:, :, :2]).max(axis=2, keepdims=True)
    tol = ORACLE_REL * scale[:, None, None] + np.spacing(xy.astype(np.float32)).astype(np.float64)
    assert (np.abs(got - want) <= tol).all(), np.abs(got - want).max()


def test_determinism_batch_position_nan_isolation():
    rng = np.random.default_rng(17)
    B = 64
    s = seed_t()
    f, r = augm_params(B, True, 30.0, s)
    f2, r2 = augm_params(B, True, 30.0, s.clone())
    assert torch.equal(f, f2) and torch.equal(r, r2)
    fb, rb = augm_params(B + 40, True, 30.0, s)
    assert torch.equal(fb[:B], f) and torch.equal(rb[:B], r)
    x = torch.from_numpy(poses(B, 19, rng)).to(dev())
    a = training_pose2d(x, "coco", seed=s, rot=r, flip=f)
    assert torch.equal(a, training_pose2d(x, "coco", seed=s, rot=r, flip=f))
    # a NaN pose or rotation in one sample leaves the others bitwise as they were
    xn = x.clone()
    xn[5, 3, 0] = float("nan")
    rn = r.clone()
    rn[9] = float("nan")
    an = training_pose2d(xn, "coco", seed=s, rot=rn, flip=f)
    keep = torch.ones(B, dtype=torch.bool, device=dev())
    keep[5] = keep[9] = False
    assert torch.equal(an[keep], a[keep])


def test_graph_capture_launch_counts_and_no_sync():
    B = 32
    args, _ = h36m_inputs(B, seed=77)
    cargs = [cuda(a) for a in args]
    mod = h36m_module("coco")
    seed = seed_t()

    def step(seed):
        f, r = augm_params(B, True, 30.0, seed)
        tg = mod(*cargs, rot=r, flip=f)
        return f, r, tg["lift_pose3d"], training_pose2d(tg["joint_img"], "coco", seed=seed, rot=r, flip=f)

    lib = _lib.load()
    lib.p2m_launch_count_reset()
    augm_params(B, True, 30.0, seed)
    assert lib.p2m_launch_count() == 1
    lib.p2m_launch_count_reset()
    f, r = augm_params(B, True, 30.0, seed)
    lib.p2m_launch_count_reset()
    mod(*cargs, rot=r, flip=f)
    assert lib.p2m_launch_count() == mod.LAUNCHES == 6
    lib.p2m_launch_count_reset()
    x = torch.from_numpy(poses(B, 19, np.random.default_rng(1))).to(dev())
    training_pose2d(x, "coco", seed=seed, rot=r, flip=f)
    assert lib.p2m_launch_count() == 1

    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        step(seed)
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step(seed)
    flips = []
    for new in ((1, 2), (0x1234_5678_9ABC, 99)):
        seed.copy_(seed_t(new))
        g.replay()
        torch.cuda.synchronize()
        for o, e in zip(outs, step(seed_t(new))):
            assert torch.equal(o, e)
        flips.append(outs[0].clone())
    assert not torch.equal(flips[0], flips[1])
    torch.cuda.set_sync_debug_mode("error")
    try:
        step(seed)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_argument_errors():
    lib = _lib.load()
    s = seed_t()
    f = torch.empty(4, dtype=torch.int32, device=dev())
    r = torch.empty(4, device=dev())
    host = np.zeros(4, np.float32)
    lib.p2m_launch_count_reset()
    assert lib.p2m_augm_params(0, 1, 30.0, s.data_ptr(), f.data_ptr(), r.data_ptr(), None) == 1
    assert lib.p2m_augm_params(4, 2, 30.0, s.data_ptr(), f.data_ptr(), r.data_ptr(), None) == 1
    assert lib.p2m_augm_params(4, 1, -1.0, s.data_ptr(), f.data_ptr(), r.data_ptr(), None) == 1
    assert lib.p2m_augm_params(4, 1, float("nan"), s.data_ptr(), f.data_ptr(), r.data_ptr(), None) == 1
    assert lib.p2m_augm_params(4, 1, 30.0, None, f.data_ptr(), r.data_ptr(), None) == 1
    assert lib.p2m_augm_params(4, 1, 30.0, s.data_ptr(), f.data_ptr(), host.ctypes.data, None) == 1
    x = torch.zeros(4, 19, 2, device=dev())
    out = torch.empty_like(x)
    N = _lib.P2M_NOISE_NONE
    base = [x.data_ptr(), 4, 19, None, 0, N, 0, None, None, 384, 288, r.data_ptr(), f.data_ptr(),
            _lib.P2M_JOINTS_COCO, 0, out.data_ptr(), None]
    for what, at, v in (("bad joint set", 13, 5), ("host rot", 11, host.ctypes.data), ("16 joints", 2, 16),
                        ("19 human36 joints", 13, _lib.P2M_JOINTS_HUMAN36)):
        a = list(base)
        a[at] = v
        assert lib.p2m_training_pose2d_augmented(*a) == 1, what
    assert lib.p2m_launch_count() == 0
    assert lib.p2m_training_pose2d_augmented(*base) == 0
    with pytest.raises(ValueError):
        augm_params(0, True, 30.0)
    with pytest.raises(ValueError):
        augm_params(4, True, -3.0)
    with pytest.raises(ValueError):
        training_pose2d(x, "coco", noise=False, rot=torch.zeros(3, device=dev()))
    with pytest.raises(ValueError):
        training_pose2d(x, "coco", noise=False, flip=torch.zeros(4, device=dev()))       # float flips
    with pytest.raises(ValueError):
        training_pose2d(x, "human36", noise=False, flip=f)                              # 19 Human3.6M joints
    with pytest.raises(RuntimeError):
        training_pose2d(x, "coco", noise=False, rot=torch.zeros(4))
    args, _ = h36m_inputs(4, seed=5)
    with pytest.raises(ValueError):
        h36m_module("coco")(*[cuda(a) for a in args], rot=torch.zeros(5, device=dev()))


def test_posenet_step_on_a_flipped_batch():
    """augm_params -> Human36MTargets('coco', rot, flip) -> training_pose2d -> one native PoseNet training step."""
    from pose2mesh_release_b200 import posenet

    B = 16
    args, _ = h36m_inputs(B, seed=91)
    seed = seed_t()
    f, r = augm_params(B, True, 30.0, seed)
    tg = h36m_module("coco")(*[cuda(a) for a in args], rot=r, flip=f)
    pose2d = training_pose2d(tg["joint_img"], "coco", seed=seed, rot=r, flip=f)
    assert int(f.sum()) > 0 and torch.isfinite(pose2d).all()
    torch.manual_seed(0)
    net = posenet.get_model(19, 4096, 2, 0.5).to(dev()).train()
    out = net.forward_train_native(pose2d, seed=seed)
    loss = ((out.reshape(B, 19, 3) - tg["lift_pose3d"] / 1000) * tg["joint_valid"]).abs().mean()
    loss.backward()
    grads = [p.grad for p in net.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g).all() for g in grads)


CLASSES = {"coco": COCOTargets, "muco": MuCoTargets, "amass": AMASSTargets}


def dataset_case(dataset, B, seed):
    """(module call arguments as numpy, oracle keyword arguments, the oracle's camera-frame mesh).  COCO: annotation
    keypoints within 0.1 px of the projected regressed joints on even samples and 60 px off on odd ones (far on either
    side of 3 px), a third of the samples with no visible keypoint; MuCo: trans moved 4 m in front of the camera."""
    pose, betas, trans, R, t = inputs(B, dataset, seed)
    rng = np.random.default_rng(seed)
    if dataset == "muco":
        trans = (trans + np.float32([0, 0, 4.0])).astype(np.float32)
    mesh, _ = oracle(dataset, pose, betas, trans, R, t)
    f = rng.uniform(1100, 1200, (B, 2)).astype(np.float32)
    c = rng.uniform(480, 540, (B, 2)).astype(np.float32)
    if dataset == "coco":
        s = rng.uniform(180, 260, (B, 2) if seed % 2 else B).astype(np.float32)
        tt = rng.uniform(300, 500, (B, 2)).astype(np.float32)
        reg = np.einsum("jv,bvc->bjc", TGOLDEN["reg_coco"], mesh)
        img = reg[..., :2] / 1000 * s.reshape(B, -1)[:, None, :] + tt[:, None, :]
        sd = np.where(np.arange(B) % 2 == 0, 0.1, 60.0)[:, None, None]
        kps = (img + sd * rng.normal(size=img.shape)).astype(np.float32)
        vis = (rng.uniform(size=(B, 17)) < 0.7).astype(np.float32)
        vis[2::3] = 0
        return (pose, betas, s, tt, kps, vis), dict(s=s, t=tt, keypoints=kps, keypoints_valid=vis), mesh
    if dataset == "muco":
        return (pose, betas, trans, f, c), dict(f=f, c=c), mesh
    return (pose, betas, R, t, f, c), dict(f=f, c=c), mesh


@pytest.mark.parametrize("dataset", ["coco", "muco", "amass"])
@pytest.mark.parametrize("joint_set", ["human36", "coco"])
@pytest.mark.parametrize("B", [1, 7, 256])
def test_dataset_targets_vs_oracle(dataset, joint_set, B):
    args, kw, mesh_cam = dataset_case(dataset, B, 500 + B)
    mod = CLASSES[dataset](layer(), TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"], joint_set)
    flip, rot = aug_for(B, np.random.default_rng(B))
    cargs = [cuda(a) for a in args]
    base = mod(*cargs)
    got = mod(*cargs, rot=torch.from_numpy(rot).to(dev()), flip=torch.from_numpy(flip).to(dev()))
    zero = mod(*cargs, rot=torch.zeros(B, device=dev()), flip=torch.zeros(B, dtype=torch.int32, device=dev()))
    bits = lambda x: x.view(torch.int32)  # noqa: E731  (bitwise, so COCO's NaN errors compare equal to themselves)
    for k in base:
        assert torch.equal(bits(base[k]), bits(zero[k])), k
        if k != "lift_pose3d":
            assert torch.equal(bits(base[k]), bits(got[k])), k
    got = {k: v.cpu().numpy().astype(np.float64) for k, v in got.items()}
    want = so.sample_targets(dataset, mesh_cam, TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"], joint_set, **kw)
    scale = np.abs(mesh_cam).max(axis=(1, 2))
    for k, sc in (("mesh", scale / 1000), ("reg_pose3d", scale)):
        assert (np.abs(got[k] - want[k]).max(axis=(1, 2)) <= ORACLE_REL * sc).all(), k
    lift = so.j3d_processing(want["lift_pose3d"], rot, flip, joint_set)
    xy = np.abs(lift[:, :, :2]).max(axis=2, keepdims=True)
    tol = ORACLE_REL * scale[:, None, None] + np.spacing(xy.astype(np.float32)).astype(np.float64)
    assert (np.abs(got["lift_pose3d"] - lift) <= tol).all()
    assert (np.abs(got["joint_img"] - want["joint_img"]).max(axis=(1, 2)) <= ORACLE_REL * (2 * 1200 + scale)).all()
    ge, we = got["fitting_error"], want["fitting_error"]
    np.testing.assert_array_equal(np.isnan(ge), np.isnan(we))
    ok = ~np.isnan(we)
    bound = 1e-3 if dataset == "coco" else ORACLE_REL * scale[ok]        # COCO's error is in pixels of a 64 crop
    assert (np.abs(ge[ok] - we[ok]) <= bound).all(), np.abs(ge[ok] - we[ok]).max()
    for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid", "joint_valid"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    if dataset == "coco" and B >= 7:
        assert got["mesh_valid"][0, 0, 0] == 1 and got["mesh_valid"][1, 0, 0] == 0 and np.isnan(ge[2])
    if dataset == "muco":
        assert (ge > 100).all() and (got["mesh_valid"] == 0).all() and (got["joint_valid"] == 1).all()


def test_dataset_targets_match_reference_fitting():
    m, mi = GOLDEN["fit__mesh"], GOLDEN["coco_fit__mesh_index"]
    reg = (TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"])
    lib = _lib.load()
    for k in range(len(mi)):
        js = "coco" if GOLDEN["coco_fit__set"][k] else "human36"
        mod = COCOTargets(layer(), *reg, js)
        J = mod.num_joints
        e = lambda *sh: torch.empty(sh, device=dev())  # noqa: E731
        out = [e(1, 6890, 3), e(1, J, 3), e(1, 17, 3), e(1, 6890), e(1, J), e(1, 17), e(1, J), e(1, J, 2), e(1)]
        mesh = cuda(m[mi[k]][None])
        a = [cuda(GOLDEN[f"coco_fit__{n}"][k:k + 1]) for n in ("s", "t", "kps", "valid")]
        assert lib.p2m_sample_targets(mod.handle(0), _lib.P2M_DATASET_COCO, 1 if js == "coco" else 0, 3.0, mesh.data_ptr(), None, None, None,
            a[0].data_ptr(), 1, a[1].data_ptr(), a[2].data_ptr(), a[3].data_ptr(), None, None, 1,
            *[o.data_ptr() for o in out], None) == 0
        err = float(out[8].cpu())
        want = GOLDEN["coco_fit__error"][k]
        assert (np.isnan(err) and np.isnan(want)) or abs(err - want) < 1e-3, (k, err, want)
        assert float(out[3][0, 0].cpu()) == (0.0 if want > 3 else 1.0)
    mod = MuCoTargets(layer(), *reg, "coco")
    B = m.shape[0]
    out = [torch.empty(sh, device=dev()) for sh in ((B, 6890, 3), (B, 19, 3), (B, 17, 3), (B, 6890), (B, 19), (B, 17),
                                                     (B, 19), (B, 19, 2), (B,))]
    f, c = cuda(np.full((B, 2), 1000.0)), cuda(np.full((B, 2), 500.0))
    mesh = cuda(m)
    assert lib.p2m_sample_targets(mod.handle(0), _lib.P2M_DATASET_MUCO, 1, 45.0, mesh.data_ptr(), None,
                                  f.data_ptr(), c.data_ptr(), None, 0, None, None, None, None, None, B,
                                  *[o.data_ptr() for o in out], None) == 0
    np.testing.assert_allclose(out[8].cpu().numpy(), GOLDEN["muco_fit__error"], rtol=1e-5)


def test_sample_targets_argument_errors():
    lib = _lib.load()
    mod = COCOTargets(layer(), TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"], "coco")
    B = 2
    x = torch.zeros(B, 6890, 3, device=dev())
    o = torch.zeros(B * 6890 * 3, device=dev())
    lib.p2m_launch_count_reset()
    base = [mod.handle(0), _lib.P2M_DATASET_COCO, 1, 3.0, x.data_ptr(), None, None, None, o.data_ptr(), 1,
            o.data_ptr(), o.data_ptr(), o.data_ptr(), None, None, B] + [o.data_ptr()] * 9 + [None]
    for what, at, v in (("unknown dataset", 1, 7), ("n_s 3", 9, 3), ("no keypoints", 11, None),
                        ("Human36M without joint_cam", 1, _lib.P2M_DATASET_HUMAN36M),
                        ("MuCo without f", 1, _lib.P2M_DATASET_MUCO), ("batch 0", 15, 0),
                        ("host keypoints", 11, np.zeros(34 * B, np.float32).ctypes.data)):
        a = list(base)
        a[at] = v
        assert lib.p2m_sample_targets(*a) == 1, what
    assert lib.p2m_launch_count() == 0
    pose, betas = (cuda(a) for a in inputs(B, "coco", 1)[:2])
    with pytest.raises(ValueError):
        mod(pose, betas, torch.zeros(B, 3, device=dev()), torch.zeros(B, 2, device=dev()),
            torch.zeros(B, 17, 2, device=dev()), torch.zeros(B, 17, device=dev()))        # s [B, 3]
    with pytest.raises(ValueError):
        mod(pose, betas, torch.zeros(B, device=dev()), torch.zeros(B, 2, device=dev()),
            torch.zeros(B, 16, 2, device=dev()), torch.zeros(B, 17, device=dev()))        # 16 keypoints
    lib.p2m_launch_count_reset()
    mod(pose, betas, torch.ones(B, device=dev()), torch.zeros(B, 2, device=dev()), torch.zeros(B, 17, 2, device=dev()),
        torch.ones(B, 17, device=dev()))
    assert lib.p2m_launch_count() == mod.LAUNCHES == 6


def test_mixed_batch_posenet_and_pose2mesh_steps():
    """A flipped Human36M + COCO + MuCo batch built on the device (augm_params, each dataset's targets and inputs, MuCo
    flipping before the noise), then one native PoseNet step and one FlatPose2Mesh step whose losses take the masks."""
    import scipy.sparse as sp
    from helpers import graph_from_fixture
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L
    from pose2mesh_release_b200 import posenet, pose2mesh_net
    from test_gpu_inputs import COCO_FLIP_PAIRS, COCO_SKELETON

    n = 8
    seed = seed_t()
    parts = []
    h_args, _ = h36m_inputs(n, seed=61)
    for k, (dataset, mod_args) in enumerate((("human36m", [cuda(a) for a in h_args]),
                                             ("coco", [cuda(a) for a in dataset_case("coco", n, 62)[0]]),
                                             ("muco", [cuda(a) for a in dataset_case("muco", n, 63)[0]]))):
        s = seed.clone()
        s[1] += k                                                       # one stream per dataset's sub-batch
        f, r = augm_params(n, True, 0.0, s)
        mod = h36m_module("coco") if dataset == "human36m" else CLASSES[dataset](layer(), TGOLDEN["reg_h36m"],
                                                                                  TGOLDEN["reg_coco"], "coco")
        tg = mod(*mod_args, rot=r, flip=f)
        pose2d = training_pose2d(tg["joint_img"], "coco", seed=s, rot=r, flip=f, flip_before_noise=dataset == "muco",
                                 area_box="crop" if dataset == "muco" else "tight")
        parts.append((pose2d, tg))
    pose2d = torch.cat([p for p, _ in parts])
    tg = {k: torch.cat([t[k] for _, t in parts]) for k in parts[0][1]}
    B = pose2d.shape[0]
    assert torch.isfinite(pose2d).all()
    torch.manual_seed(0)
    net = posenet.get_model(19, 4096, 2, 0.5).to(dev()).train()
    out = net.forward_train_native(pose2d, seed=seed)
    loss = ((out.reshape(B, 19, 3) - tg["lift_pose3d"] / 1000) * tg["joint_valid"]).abs().mean()
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)

    mats, _ = graph_from_fixture("smpl_small")
    adj = sp.csr_matrix(pg.build_adj(19, COCO_SKELETON, COCO_FLIP_PAIRS))
    adj.eliminate_zeros()
    mats[-1] = pg.laplacian(adj, normalized=True)
    flat = pose2mesh_net.get_model(19, mats).to(dev()).train()
    mesh, pose3d = flat(pose2d)
    V = mesh.shape[1]
    coord_loss = L.CoordLoss(has_valid=True)
    loss = coord_loss(pose3d.reshape(B, 19, 3), tg["lift_pose3d"], tg["lift_pose3d_valid"]) + \
        coord_loss(mesh, tg["mesh"][:, :V], tg["mesh_valid"][:, :V])
    loss.backward()
    grads = [p.grad for p in flat.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g).all() for g in grads)
