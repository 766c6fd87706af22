"""SURREAL, FreiHAND and 3DPW samples on the GPU (inputs.training_pose2d with the 'smpl' / 'mano' sets,
targets.SURREALTargets / FreiHANDTargets / PW3DTargets) against the float64 oracle (tests/smpl_mano_oracle.py) and
the unmodified reference (tests/golden/smpl_mano_samples.npz).

Bounds.  The crops: atol 1e-5 on the normalised coordinates, as test_gpu_samples.py.  The assemblies are checked on
the device's own camera-frame meshes, so only the assembly's arithmetic is under test: SURREAL's and FreiHAND's float32
rooting and mesh / 1000 are the reference's own float32 steps and match bit for bit, as do unrotated lift targets; a
rotated lift and every fp64 result rounded once are within one float32 ulp (sin / cos of the device and of NumPy may
differ in the last fp64 bit).  3DPW against the reference: test_smpl_mano_samples_cpu.pw3d_bounds, the float32
regression's worst case, plus the device's own half ulp.
"""
import numpy as np
import pytest
import torch

import smpl_mano_oracle as smo
from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200.inputs import augm_params, training_pose2d
from pose2mesh_release_b200.targets import (FreiHANDTargets, PW3DTargets, SURREALTargets, AMASSTargets, COCOTargets,
                                            MuCoTargets, camera_frame_coords)
from test_gpu_samples import CLASSES, aug_for, dataset_case, poses, seed_t
from test_gpu_targets import GOLDEN as TGOLDEN
from test_gpu_targets import cuda, h36m_inputs, h36m_module, inputs, layer
from test_smpl_mano_samples_cpu import GOLDEN, SAMPLES, pw3d_bounds, surreal_img_tol

pytestmark = pytest.mark.gpu
REG = (TGOLDEN["reg_h36m"], TGOLDEN["reg_coco"])
SMPL_SKELETON = ((0, 1), (1, 4), (4, 7), (7, 10), (0, 2), (2, 5), (5, 8), (8, 11), (0, 3), (3, 6), (6, 9), (9, 14),
                 (14, 17), (17, 19), (19, 21), (21, 23), (9, 13), (13, 16), (16, 18), (18, 20), (20, 22), (9, 12),
                 (12, 15))


def dev():
    return torch.device("cuda:0")


def npy(t):
    return t.cpu().numpy().astype(np.float64)


def ulp_close(got, want, atol=1e-9):
    """One float32 ulp, plus atol for fp64 results that cancel to near zero (the device's fma order and sin / cos
    differ from NumPy's in the last fp64 bits: about 1e-12 of a millimetre-scale value)."""
    want = np.asarray(want, np.float64)
    return np.abs(np.asarray(got, np.float64) - want) <= \
        np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + atol


def surreal_args(B, seed):
    """pose, betas, trans (moved 4 m in front of the camera), f, c as float32."""
    pose, betas, trans, _, _ = inputs(B, "surreal", seed)
    rng = np.random.default_rng(seed)
    trans = (trans + np.float32([0, 0, 4.0])).astype(np.float32)
    f = rng.uniform(900, 1600, (B, 2)).astype(np.float32)
    c = rng.uniform(200, 600, (B, 2)).astype(np.float32)
    return pose, betas, trans, f, c


def freihand_args(B, seed):
    pose, betas, _, R, t = inputs(B, "freihand", seed)
    return pose, betas, R, t


# ---------------------------------------------------------------------------------------------------------- crops
@pytest.mark.parametrize("B", [1, 7, 256, 1000])
@pytest.mark.parametrize("flip_before", [False, True])
def test_smpl_crop_matches_oracle(B, flip_before):
    rng = np.random.default_rng(B + 11 * flip_before)
    x = poses(B, 24, rng)
    flip, rot = aug_for(B, rng)
    got = training_pose2d(torch.from_numpy(x).to(dev()), "smpl", noise=False, rot=torch.from_numpy(rot).to(dev()),
                          flip=torch.from_numpy(flip).to(dev()), flip_before_noise=flip_before)
    want, _ = smo.training_pose2d(x, "smpl", rot, flip, flip_before)
    np.testing.assert_allclose(npy(got), want, atol=1e-5, rtol=0)


@pytest.mark.parametrize("B", [1, 7, 256, 1000])
def test_mano_crop_matches_oracle(B):
    x = poses(B, 21, np.random.default_rng(B + 3))
    got = training_pose2d(torch.from_numpy(x).to(dev()), "mano", noise=False)
    want, _ = smo.training_pose2d(x, "mano")
    np.testing.assert_allclose(npy(got), want, atol=1e-5, rtol=0)


@pytest.mark.parametrize("kind", ["det", "gt"])
def test_smpl_crop_matches_reference_fixture(kind):
    """det: float32 detections, flip after the crop; gt: the float64 cam2pixel joints, flip before it is rounded."""
    x = torch.from_numpy(GOLDEN[f"surreal__{kind}"].astype(np.float32)).to(dev())
    C = x.shape[0]
    for a, (fl, rot) in enumerate(GOLDEN["aug_cases"]):
        got = training_pose2d(x, "smpl", noise=False, rot=torch.full((C,), float(np.float32(rot)), device=dev()),
                              flip=torch.full((C,), int(fl), dtype=torch.int32, device=dev()),
                              flip_before_noise=kind == "gt")
        np.testing.assert_allclose(npy(got), GOLDEN[f"surreal__pose2d_{kind}"][:, a], atol=1e-5, rtol=0)


@pytest.mark.parametrize("case,joint_set", [("freihand", "mano"), ("pw3d", "coco")])
def test_unaugmented_crops_match_reference_fixture(case, joint_set):
    x = torch.from_numpy(GOLDEN[f"{case}__det"]).to(dev())
    got = training_pose2d(x, joint_set, noise=False)
    np.testing.assert_allclose(npy(got), GOLDEN[f"{case}__pose2d"], atol=1e-5, rtol=0)


# -------------------------------------------------------------------------------------------------------- targets
def check_surreal(got, mesh_cam, joints, f, c, rot, flip):
    want = smo.surreal_targets(mesh_cam, joints, f, c, rot, flip)
    g = {k: npy(v) for k, v in got.items()}
    np.testing.assert_array_equal(g["mesh"], want["mesh"].astype(np.float32))
    assert torch.equal(got["lift_pose3d"], got["reg_pose3d"])          # the reference's one augmented array
    plain = (np.asarray(rot) == 0)
    np.testing.assert_array_equal(g["lift_pose3d"][plain], want["lift_pose3d"][plain].astype(np.float32))
    assert ulp_close(g["lift_pose3d"], want["lift_pose3d"]).all()
    assert ulp_close(g["joint_img"], want["joint_img"]).all()
    for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid", "joint_valid"):
        assert (g[k] == 1).all(), k
    assert (g["fitting_error"] == 0).all()


@pytest.mark.parametrize("B", [1, 7, 256])
def test_surreal_targets_vs_oracle(B):
    pose, betas, trans, f, c = surreal_args(B, 700 + B)
    flip, rot = aug_for(B, np.random.default_rng(B))
    mod = SURREALTargets(layer())
    got = mod(*[cuda(a) for a in (pose, betas, trans, f, c)], rot=torch.from_numpy(rot).to(dev()),
              flip=torch.from_numpy(flip).to(dev()))
    assert got["lift_pose3d"].shape == (B, 24, 3) and got["joint_img"].shape == (B, 24, 2)
    mesh_cam, joints = camera_frame_coords(layer(), "surreal", cuda(pose), cuda(betas), cuda(trans))
    check_surreal(got, npy(mesh_cam), npy(joints), f, c, rot, flip)


def test_surreal_targets_match_reference_fixture():
    mod = SURREALTargets(layer())
    mesh, joints, f, c = (cuda(GOLDEN[f"surreal__{k}"]) for k in ("mesh_in", "joints_in", "f", "c"))
    C = mesh.shape[0]
    for a, (fl, rot) in enumerate(GOLDEN["aug_cases"]):
        rot32 = np.float32(rot)
        got = mod._assemble(mesh, joints, f, c, torch.full((C,), float(rot32), device=dev()),
                            torch.full((C,), int(fl), dtype=torch.int32, device=dev()))
        np.testing.assert_array_equal(npy(got["mesh"]), GOLDEN["surreal__mesh"])
        want = GOLDEN["surreal__lift"][:, a]
        if rot32 == 0:
            np.testing.assert_array_equal(npy(got["lift_pose3d"]), want)
        assert ulp_close(npy(got["lift_pose3d"]), want).all()
        assert torch.equal(got["lift_pose3d"], got["reg_pose3d"])
        tol = surreal_img_tol(GOLDEN["surreal__joints_in"].astype(np.float64), GOLDEN["surreal__f"])
        assert (np.abs(npy(got["joint_img"]) - GOLDEN["surreal__gt"]) <= tol).all()


@pytest.mark.parametrize("B", [1, 7, 256, 1024])
def test_freihand_targets_vs_oracle(B):
    args = freihand_args(B, 800 + B)
    got = FreiHANDTargets(layer(mano=True))(*[cuda(a) for a in args])
    assert "joint_img" not in got and got["reg_pose3d"].shape == (B, 21, 3)
    mesh_cam, joints = camera_frame_coords(layer(mano=True), "freihand", cuda(args[0]), cuda(args[1]), None,
                                           cuda(args[2]), cuda(args[3]))
    want = smo.freihand_targets(npy(mesh_cam), npy(joints))
    for k in ("mesh", "lift_pose3d", "reg_pose3d"):
        np.testing.assert_array_equal(npy(got[k]), want[k].astype(np.float32), err_msg=k)
    for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid", "joint_valid"):
        assert (npy(got[k]) == 1).all(), k
    assert (npy(got["fitting_error"]) == 0).all()


def test_freihand_targets_match_reference_fixture_bitwise():
    """The reference roots in one float32 subtraction and divides the mesh in float32: the same bits."""
    mod = FreiHANDTargets(layer(mano=True))
    got = mod._assemble(cuda(GOLDEN["freihand__mesh_in"]), cuda(GOLDEN["freihand__joints_in"]))
    np.testing.assert_array_equal(npy(got["mesh"]), GOLDEN["freihand__mesh"])
    np.testing.assert_array_equal(npy(got["lift_pose3d"]), GOLDEN["freihand__joints"])
    np.testing.assert_array_equal(npy(got["reg_pose3d"]), GOLDEN["freihand__joints"])


def pw3d_args(B, seed):
    pose, betas, trans, _, _ = inputs(B, "pw3d", seed)
    rng = np.random.default_rng(seed)
    trans = (trans + np.float32([0, 0, 4.0])).astype(np.float32)
    return pose, betas, trans, rng.uniform(900, 1600, (B, 2)).astype(np.float32), \
        rng.uniform(200, 600, (B, 2)).astype(np.float32)


@pytest.mark.parametrize("B", [1, 7, 256])
def test_pw3d_targets_vs_oracle(B):
    pose, betas, trans, f, c = pw3d_args(B, 900 + B)
    got = PW3DTargets(layer(), *REG)(*[cuda(a) for a in (pose, betas, trans, f, c)])
    mesh_cam, _ = camera_frame_coords(layer(), "pw3d", cuda(pose), cuda(betas), cuda(trans))
    want = smo.pw3d_targets(npy(mesh_cam), *REG, f, c)
    g = {k: npy(v) for k, v in got.items()}
    for k in ("mesh", "lift_pose3d", "reg_pose3d", "joint_img"):
        assert ulp_close(g[k], want[k]).all(), (k, np.abs(g[k] - want[k]).max())
    for k in ("mesh_valid", "lift_pose3d_valid", "reg_pose3d_valid", "joint_valid"):
        np.testing.assert_array_equal(g[k], want[k], err_msg=k)
    assert (g["fitting_error"] == 0).all()


def test_pw3d_targets_match_reference_within_float32_regression():
    mesh = SAMPLES["fit__mesh"][GOLDEN["pw3d__mesh_index"]]
    f, c = GOLDEN["pw3d__f"], GOLDEN["pw3d__c"]
    mod = PW3DTargets(layer(), *REG)
    got = {k: npy(v) for k, v in mod._assemble(cuda(mesh), None, None, f=cuda(f), c=cuda(c)).items()}
    bounds = pw3d_bounds(mesh, *REG, smo.pw3d_targets(mesh, *REG, f, c), f)
    rows = GOLDEN["pw3d__rows"]
    for key, gkey, sl in (("reg_pose3d", "reg", slice(None)), ("lift_pose3d", "lift", slice(None)),
                          ("mesh", "mesh", rows), ("joint_img", "joint_img", slice(None))):
        want = GOLDEN[f"pw3d__{gkey}"].astype(np.float64)
        own = np.spacing(np.abs(got[key][:, sl]).astype(np.float32)).astype(np.float64)
        assert (np.abs(got[key][:, sl] - want) <= bounds[key][:, sl] + own).all(), key


# ----------------------------------------------------------------------------------------------------- invariants
def test_launch_counts_position_independence_and_nan_isolation():
    lib = _lib.load()
    B = 12
    sargs = [cuda(a) for a in surreal_args(B, 41)]
    fargs = [cuda(a) for a in freihand_args(B, 42)]
    pargs = [cuda(a) for a in pw3d_args(B, 43)]
    f, r = augm_params(B, True, 30.0, seed_t())
    mods = ((SURREALTargets(layer()), sargs, dict(rot=r, flip=f)), (FreiHANDTargets(layer(mano=True)), fargs, {}),
            (PW3DTargets(layer(), *REG), pargs, {}))
    for mod, args, kw in mods:
        lib.p2m_launch_count_reset()
        full = mod(*args, **kw)
        assert lib.p2m_launch_count() == mod.LAUNCHES == 6
        # samples 3..7 alone give the same bits as inside the batch
        part = mod(*[a[3:8] for a in args], **{k: v[3:8] for k, v in kw.items()})
        for k in full:
            assert torch.equal(full[k][3:8], part[k]), k
        # a NaN pose in sample 5 leaves the others bitwise as they were
        bad = [a.clone() for a in args]
        bad[0][5, 4] = float("nan")
        nan = mod(*bad, **kw)
        keep = torch.ones(B, dtype=torch.bool, device=dev())
        keep[5] = False
        for k in full:
            assert torch.equal(full[k][keep], nan[k][keep]), k
    x = torch.from_numpy(poses(B, 24, np.random.default_rng(5))).to(dev())
    lib.p2m_launch_count_reset()
    training_pose2d(x, "smpl", noise=False, rot=r, flip=f)
    assert lib.p2m_launch_count() == 1


def test_graph_capture_and_replay():
    B = 16
    sargs = [cuda(a) for a in surreal_args(B, 51)]
    fargs = [cuda(a) for a in freihand_args(B, 52)]
    sm, fm = SURREALTargets(layer()), FreiHANDTargets(layer(mano=True))
    seed = seed_t()

    def step(seed):
        f, r = augm_params(B, True, 30.0, seed)
        st = sm(*sargs, rot=r, flip=f)
        ft = fm(*fargs)
        return (st["lift_pose3d"], st["mesh"], training_pose2d(st["joint_img"], "smpl", noise=False, rot=r, flip=f),
                ft["mesh"], ft["reg_pose3d"])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(seed)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step(seed)
    for new in ((1, 2), (0x1234_5678_9ABC, 99)):
        seed.copy_(seed_t(new))
        g.replay()
        torch.cuda.synchronize()
        for o, e in zip(outs, step(seed_t(new))):
            assert torch.equal(o, e)
    torch.cuda.set_sync_debug_mode("error")
    try:
        step(seed)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def centred_layers():
    """The test suite's SMPL and MANO layers rebuilt with center_idx = 0."""
    from test_gpu_targets import MANO, SMPL
    from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer

    m, h = SMPL, MANO
    return (SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                      m["betas"], center_idx=0),
            ManoLayer(h["v_template"], h["shapedirs"], h["posedirs"], h["J_regressor"], h["weights"], h["betas"],
                      h["hands_mean"], center_idx=0, flat_hand_mean=False, side="right"))


def test_argument_errors():
    lib = _lib.load()
    B = 3
    z = lambda *sh: torch.zeros(sh, device=dev())  # noqa: E731
    zi = torch.zeros(B, dtype=torch.int32, device=dev())
    with pytest.raises(ValueError):
        training_pose2d(z(B, 24, 2), "smpl")                                  # noise on 'smpl'
    with pytest.raises(ValueError):
        training_pose2d(z(B, 21, 2), "mano")                                  # noise on 'mano'
    with pytest.raises(ValueError):
        training_pose2d(z(B, 23, 2), "smpl", noise=False)
    with pytest.raises(ValueError):
        training_pose2d(z(B, 24, 2), "mano", noise=False)
    with pytest.raises(ValueError):
        training_pose2d(z(B, 21, 2), "mano", noise=False, flip=zi)            # no MANO flip pairs
    with pytest.raises(ValueError):
        training_pose2d(z(B, 24, 2), "hand", noise=False)
    # the C entry points refuse the same, before any launch
    x, o = z(B, 24, 2), z(B, 24, 2)
    lib.p2m_launch_count_reset()
    call = lambda n, js, noise, flip: lib.p2m_training_pose2d_augmented(  # noqa: E731
        x.data_ptr(), B, n, None, 0, noise, 0, None, seed_t().data_ptr(), 384, 288, None, flip, js, 0, o.data_ptr(),
        None)
    assert call(24, _lib.P2M_JOINTS_SMPL, _lib.P2M_NOISE_COCO, None) == 1
    assert call(23, _lib.P2M_JOINTS_SMPL, 0, None) == 1
    assert call(21, _lib.P2M_JOINTS_MANO, 0, zi.data_ptr()) == 1
    assert call(21, 4, 0, None) == 1
    assert lib.p2m_launch_count() == 0
    # targets: layers of the wrong kind, shapes, devices
    with pytest.raises(ValueError):
        SURREALTargets(layer(mano=True))
    with pytest.raises(ValueError):
        FreiHANDTargets(layer())
    with pytest.raises(ValueError):
        PW3DTargets(layer(), *REG, "human36")
    with pytest.raises(ValueError):
        PW3DTargets(layer(mano=True), *REG)                                   # a ManoLayer
    # a layer with center_idx set: the datasets never centre the layer's output
    sm_c, mano_c = centred_layers()
    with pytest.raises(ValueError):
        SURREALTargets(sm_c)
    with pytest.raises(ValueError):
        FreiHANDTargets(mano_c)
    pose, betas, trans, f, c = (cuda(a) for a in surreal_args(B, 3))
    with pytest.raises(ValueError):
        PW3DTargets(sm_c, *REG)(pose, betas, trans, f, c)
    sm = SURREALTargets(layer())
    pose, betas, trans, f, c = (cuda(a) for a in surreal_args(B, 3))
    with pytest.raises(ValueError):
        sm(pose, betas, trans, z(B, 3), c)                                    # f [B, 3]
    with pytest.raises(ValueError):
        sm(pose, betas, trans, f, c, rot=z(B + 1))
    with pytest.raises(ValueError):
        sm(pose, betas, trans, f, c, flip=z(B))                               # float flips
    with pytest.raises(ValueError):
        sm._assemble(z(B, 10, 3), z(B, 23, 3), f, c)                          # 23 joints
    for bad in (torch.zeros((), device=dev()), z(B, 10), z(0, 10, 3), z(B, 0, 3)):
        with pytest.raises(ValueError):
            sm._assemble(bad, z(B, 24, 3), f, c)
    with pytest.raises(RuntimeError):
        sm(pose, betas, trans, f.cpu(), c)
    lib.p2m_launch_count_reset()
    mc, jc, out = z(B, 10, 3), z(B, 24, 3), z(B * 10 * 3)
    base = [_lib.P2M_DATASET_SURREAL, mc.data_ptr(), jc.data_ptr(), 10, 24, f.data_ptr(), c.data_ptr(), None, None, B] + \
        [out.data_ptr()] * 9 + [None]
    for what, at, v in (("unknown dataset", 0, _lib.P2M_DATASET_AMASS), ("SURREAL 21 joints", 4, 21),
                        ("SURREAL without f", 5, None), ("SURREAL without joint_img", 17, None),
                        ("FreiHAND with f", 0, _lib.P2M_DATASET_FREIHAND), ("batch 0", 9, 0), ("0 vertices", 3, 0),
                        ("host mesh", 1, np.zeros(30 * B, np.float32).ctypes.data)):
        a = list(base)
        a[at] = v
        assert lib.p2m_layer_joint_targets(*a) == 1, what
    # 3DPW in p2m_sample_targets: the coco set only, no augmentation
    pm = PW3DTargets(layer(), *REG)
    mesh6890 = z(B, 6890, 3)
    po = z(B * 6890 * 3)
    for js, rot in ((_lib.P2M_JOINTS_HUMAN36, None), (_lib.P2M_JOINTS_COCO, z(B).data_ptr())):
        assert lib.p2m_sample_targets(pm.handle(0), _lib.P2M_DATASET_PW3D, js, 0.0, mesh6890.data_ptr(), None,
                                      f.data_ptr(), c.data_ptr(), None, 0, None, None, None, rot, None, B,
                                      *[po.data_ptr()] * 9, None) == 1
    assert lib.p2m_launch_count() == 0


# ---------------------------------------------------------------------------------------------- unchanged paths
def test_existing_paths_null_and_zero_augmentation_are_bitwise():
    """The coco / human36 crops and the Human36M, COCO, MuCo and AMASS targets with rot / flip None and all zero."""
    from inputs_cases import error_table
    from pose2mesh_release_b200.inputs import Human36MErrorModel

    B = 40
    rng = np.random.default_rng(8)
    zr, zf = torch.zeros(B, device=dev()), torch.zeros(B, dtype=torch.int32, device=dev())
    model = Human36MErrorModel(*error_table())
    for js, J, noise in (("coco", 19, True), ("human36", 17, True), ("coco", 19, False), ("human36", 17, False)):
        x = torch.from_numpy(poses(B, J, rng)).to(dev())
        kw = dict(noise=noise, error_model=model, seed=seed_t())
        assert torch.equal(training_pose2d(x, js, **kw), training_pose2d(x, js, rot=zr, flip=zf, **kw))
    bits = lambda t: t.view(torch.int32)  # noqa: E731
    args, _ = h36m_inputs(B, seed=12)
    for js in ("human36", "coco"):
        mod = h36m_module(js)
        cargs = [cuda(a) for a in args]
        a, b = mod(*cargs), mod(*cargs, rot=zr, flip=zf)
        assert all(torch.equal(bits(a[k]), bits(b[k])) for k in a)
        for dataset in ("coco", "muco", "amass"):
            dargs = [cuda(v) for v in dataset_case(dataset, B, 30)[0]]
            dm = CLASSES[dataset](layer(), *REG, js)
            a, b = dm(*dargs), dm(*dargs, rot=zr, flip=zf)
            assert all(torch.equal(bits(a[k]), bits(b[k])) for k in a), (dataset, js)
    assert CLASSES == {"coco": COCOTargets, "muco": MuCoTargets, "amass": AMASSTargets}


# ----------------------------------------------------------------------------------------------------- end to end
def _steps(pose2d, tg, J, graph_name, skeleton, pairs):
    import scipy.sparse as sp
    from helpers import graph_from_fixture
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L
    from pose2mesh_release_b200 import posenet, pose2mesh_net

    B = pose2d.shape[0]
    assert torch.isfinite(pose2d).all()
    torch.manual_seed(0)
    net = posenet.get_model(J, 4096, 2, 0.5).to(dev()).train()
    out = net.forward_train_native(pose2d, seed=seed_t())
    loss = ((out.reshape(B, J, 3) - tg["lift_pose3d"] / 1000) * tg["joint_valid"]).abs().mean()
    loss.backward()
    assert torch.isfinite(loss) and all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)

    mats, _ = graph_from_fixture(graph_name)
    adj = sp.csr_matrix(pg.build_adj(J, skeleton, pairs))
    adj.eliminate_zeros()
    mats[-1] = pg.laplacian(adj, normalized=True)
    flat = pose2mesh_net.get_model(J, mats).to(dev()).train()
    mesh, pose3d = flat(pose2d)
    V = min(mesh.shape[1], tg["mesh"].shape[1])                         # the padded graph against the real mesh
    coord_loss = L.CoordLoss(has_valid=True)
    loss = coord_loss(pose3d.reshape(B, J, 3), tg["lift_pose3d"], tg["lift_pose3d_valid"]) + \
        coord_loss(mesh[:, :V], tg["mesh"][:, :V], tg["mesh_valid"][:, :V])
    loss.backward()
    grads = [p.grad for p in flat.parameters() if p.grad is not None]
    assert torch.isfinite(loss) and grads and all(torch.isfinite(g).all() for g in grads)


def test_freihand_batch_posenet_and_pose2mesh_steps():
    """FreiHAND targets and crop built on the device, then one native PoseNet step (21 joints) and one FlatPose2Mesh
    step on the mano_like hierarchy with the joint graph build_adj(21, MANO skeleton, joint_hori_conn)."""
    from pose2mesh_release_b200 import graph as pg

    B = 16
    pose, betas, R, t = (cuda(a) for a in freihand_args(B, 61))
    tg = FreiHANDTargets(layer(mano=True))(pose, betas, R, t)
    _, joints = camera_frame_coords(layer(mano=True), "freihand", pose, betas, None, R, t)
    det = joints[..., :2] / joints[..., 2:] * 1000.0 + 300.0          # a pinhole projection stands in for detections
    pose2d = training_pose2d(det, "mano", noise=False)
    _steps(pose2d, tg, 21, "mano_like", pg.MANO_SKELETON, pg.MANO_HORI_CONN)


def test_surreal_flipped_batch_posenet_and_pose2mesh_steps():
    """posenet_smplJ_train_surreal's batch (24 joints) on smpl_small: augm_params(flip=True, rotate_factor=0), the same
    flips for SURREALTargets and for the float32 detections' crop (flipped after it is rounded)."""
    B = 16
    f, r = augm_params(B, True, 0.0, seed_t())
    assert int(f.sum()) > 0 and not r.any()
    tg = SURREALTargets(layer())(*[cuda(a) for a in surreal_args(B, 62)], rot=r, flip=f)
    gen = torch.Generator(device=dev()).manual_seed(62)
    det = tg["joint_img"] + 6.0 * torch.randn(tg["joint_img"].shape, device=dev(), generator=gen)   # detections
    pose2d = training_pose2d(det, "smpl", noise=False, rot=r, flip=f)
    _steps(pose2d, tg, 24, "smpl_small", SMPL_SKELETON, smo.SMPL_FLIP_PAIRS)
    # use_gt_input: the float64 cam2pixel joints flip before the crop is rounded; the same crop to a float32 ulp
    gt = training_pose2d(tg["joint_img"], "smpl", noise=False, rot=r, flip=f, flip_before_noise=True)
    assert (gt - training_pose2d(tg["joint_img"], "smpl", noise=False, rot=r, flip=f)).abs().max() < 1e-5
