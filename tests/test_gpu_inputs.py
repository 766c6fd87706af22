"""The training inputs on the GPU (pose2mesh_release_b200/inputs.py): the device against oracle/inputs_oracle.py on the
same seeds (outcomes identical, coordinates to a float32 ulp), the device's own samples against the reference's
statistics (tests/golden/inputs.npz), the noise-free path against normalize_pose2d, determinism, CUDA-graph replay
with fresh seeds, argument checks and one end-to-end training step."""
import ctypes as C

import numpy as np
import pytest
import torch

from inputs_cases import CASES, GOLDEN, P_FAIL, SEEDS, case, error_table, fixture_pvalues, ordered_table
from oracle import inputs_oracle as io
from pose2mesh_release_b200 import _lib, postprocess
from pose2mesh_release_b200.inputs import Human36MErrorModel, synthesize_pose, training_pose2d

pytestmark = pytest.mark.gpu
M = int(GOLDEN["M"])


def dev():
    return torch.device("cuda:0")


def seed_t(seed=SEEDS):
    return torch.tensor([np.int64(np.uint64(seed[0])), np.int64(np.uint64(seed[1]))], dtype=torch.int64,
                        device=dev())


def random_poses(B, rng, vis_p=0.8):
    xy = rng.uniform(0, [288, 384], (B, 17, 2))
    v = (rng.uniform(size=(B, 17, 1)) < vis_p).astype(np.float64)
    return np.concatenate([xy, v], 2).astype(np.float32), rng.uniform(300, 6000, B)


def batch(B):
    """The fixture cases, then seeded random poses; area as float32."""
    rng = np.random.default_rng(B)
    joints, area = random_poses(B, rng)
    for i, name in enumerate(CASES[:B]):
        j, a, _ = case(name)
        joints[i], area[i] = j, a
    return joints, area.astype(np.float32)


def within_ulp(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float64).astype(np.float32)
    tol = np.spacing(np.maximum(np.abs(got), np.abs(want)))
    return np.abs(got.astype(np.float64) - want.astype(np.float64)) <= tol


@pytest.mark.parametrize("B", [1, 7, 256, 4096])
def test_synthesize_pose_matches_oracle(B):
    joints, area = batch(B)
    got = synthesize_pose(torch.from_numpy(joints).to(dev()), torch.from_numpy(area).to(dev()), seed_t()).cpu().numpy()
    rows = np.arange(B) if B <= 256 else np.unique(np.r_[0:8, B - 8:B, 0:B:61])
    want = io.synthesize_pose(joints[rows].astype(np.float64), area[rows].astype(np.float64), SEEDS, sample_index=rows)
    g = got[rows]
    np.testing.assert_array_equal(g[:, :, 2], want[:, :, 2])            # the same rows are zeroed
    for r in range(len(rows)):                                           # the same outcome class
        j, a = joints[rows[r]].astype(np.float64), float(area[rows[r]])
        np.testing.assert_array_equal(io.outcome_cells(g[r:r + 1], j, a), io.outcome_cells(want[r:r + 1], j, a))
    ok = within_ulp(g[:, :, :2], want[:, :, :2])
    assert ok.all(), (np.argwhere(~ok)[:5], g[~ok][:5], want[:, :, :2][~ok][:5])


@pytest.mark.parametrize("name", CASES)
def test_device_samples_match_reference_fixture(name):
    joints, area, _ = case(name)
    j = torch.from_numpy(np.repeat(joints[None], M, 0).astype(np.float32)).to(dev())
    a = torch.full((M,), area, dtype=torch.float32, device=dev())
    out = synthesize_pose(j, a, seed_t((0xC0FFEE, 17))).cpu().numpy().astype(np.float64)
    ps = fixture_pvalues(name, out)
    p, where = min(ps)
    print(f"{name}: smallest p = {p:.3g} ({where}) over {len(ps)} tests")
    assert p > P_FAIL, (p, where)


def test_h36m_noise_matches_oracle():
    table, names = error_table()
    model = Human36MErrorModel(table, names)
    for B in (1, 7, 4096):
        got = model.generate_syn_error(B, seed_t()).cpu().numpy()
        want = io.generate_syn_error(ordered_table(), B, SEEDS)
        assert (got == want).mean() > 0.999 and within_ulp(got, want).all()


def h36m_like(B, J, rng):
    """Image-pixel poses of a person about 300 x 500 px somewhere in a 1000 x 1000 image."""
    base = rng.uniform(200, 600, (B, 1, 2))
    return (base + rng.uniform(0, [300, 500], (B, J, 2))).astype(np.float32)


@pytest.mark.parametrize("joint_set,J", [("coco", 19), ("human36", 17)])
@pytest.mark.parametrize("area_box", ["tight", "crop"])
@pytest.mark.parametrize("B", [1, 7, 256])
def test_training_pose2d_matches_oracle(joint_set, J, area_box, B):
    rng = np.random.default_rng(B + J)
    px = h36m_like(B, J, rng)
    table, names = error_table()
    model = Human36MErrorModel(table, names)
    got = training_pose2d(torch.from_numpy(px).to(dev()), joint_set, error_model=model, area_box=area_box,
                          seed=seed_t()).cpu().numpy()
    noise = "coco" if joint_set == "coco" else "h36m"
    want, _ = io.training_pose2d(px, noise, SEEDS, ordered_table(), area_box)
    np.testing.assert_allclose(got, want, atol=1e-5, rtol=0)
    # the eval branch: detections mapped through the box of the ground-truth joints
    det = px + rng.normal(0, 3, px.shape).astype(np.float32)
    got = training_pose2d(torch.from_numpy(det).to(dev()), joint_set, noise=False,
                          box_joints=torch.from_numpy(px).to(dev())).cpu().numpy()
    want, _ = io.training_pose2d(det, "none", box_joints=px)
    np.testing.assert_allclose(got, want, atol=1e-5, rtol=0)


def test_noise_free_is_normalize_pose2d_bitwise():
    rng = np.random.default_rng(9)
    for J in (17, 19, 32):
        x = torch.from_numpy(h36m_like(300, J, rng)).to(dev())
        for js in ("coco", "human36"):
            assert torch.equal(training_pose2d(x, js, noise=False), postprocess.normalize_pose2d(x))


def test_determinism_seeds_graph_replay_and_no_sync():
    rng = np.random.default_rng(11)
    B = 64
    px = torch.from_numpy(h36m_like(B, 19, rng)).to(dev())
    s = seed_t()
    a = training_pose2d(px, "coco", seed=s)
    assert torch.equal(a, training_pose2d(px, "coco", seed=s.clone()))
    for k in (0, 1):
        s2 = s.clone()
        s2[k] += 1
        assert not torch.equal(a, training_pose2d(px, "coco", seed=s2))
    j, ar = batch(B)
    jt, at = torch.from_numpy(j).to(dev()), torch.from_numpy(ar).to(dev())
    model = Human36MErrorModel(*error_table())
    px17 = px[:, :17].contiguous()

    def step(seed):
        return (training_pose2d(px, "coco", seed=seed), synthesize_pose(jt, at, seed),
                training_pose2d(px17, "human36", error_model=model, seed=seed))

    seed = s.clone()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        step(seed)
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step(seed)
    for new in ((1, 2), (0x1234_5678_9ABC, 99)):
        seed.copy_(seed_t(new))
        g.replay()
        torch.cuda.synchronize()
        for o, e in zip(outs, step(seed_t(new))):
            assert torch.equal(o, e)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step(s)
        training_pose2d(px, "coco", noise=False, box_joints=px)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _lib.load().p2m_launch_count_reset()
    step(s)
    assert _lib.load().p2m_launch_count() == 3


def test_argument_errors_launch_nothing():
    lib = _lib.load()
    x = torch.zeros(4, 19, 2, device=dev())
    out = torch.empty_like(x)
    s = seed_t()
    host = np.zeros((4, 19, 2), np.float32)
    table = Human36MErrorModel(*error_table()).table
    N, COCO, H36M = _lib.P2M_NOISE_NONE, _lib.P2M_NOISE_COCO, _lib.P2M_NOISE_H36M
    x17 = torch.zeros(4, 17, 2, device=dev())
    bad = {
        "host array": (host.ctypes.data, 4, 19, None, 0, N, 0, None, None, 384, 288, out.data_ptr()),
        "mixed host and device": (x.data_ptr(), 4, 19, host.ctypes.data, 19, N, 0, None, None, 384, 288,
                                  out.data_ptr()),
        "B = 0": (x.data_ptr(), 0, 19, None, 0, N, 0, None, None, 384, 288, out.data_ptr()),
        "J > 32": (x.data_ptr(), 1, 33, None, 0, N, 0, None, None, 384, 288, out.data_ptr()),
        "no error model": (x17.data_ptr(), 4, 17, None, 0, H36M, 0, None, s.data_ptr(), 384, 288, out.data_ptr()),
        "no seed": (x.data_ptr(), 4, 19, None, 0, COCO, 0, None, None, 384, 288, out.data_ptr()),
        "COCO noise on 16 joints": (x.data_ptr(), 4, 16, None, 0, COCO, 0, None, s.data_ptr(), 384, 288,
                                    out.data_ptr()),
        "bad noise": (x.data_ptr(), 4, 19, None, 0, 7, 0, None, s.data_ptr(), 384, 288, out.data_ptr()),
        "bad area box": (x.data_ptr(), 4, 19, None, 0, COCO, 2, None, s.data_ptr(), 384, 288, out.data_ptr()),
    }
    for what, args in bad.items():
        lib.p2m_launch_count_reset()
        assert lib.p2m_training_pose2d(*args, None) == 1, what
        assert lib.p2m_launch_count() == 0, what
    j, a = torch.zeros(2, 17, 3, device=dev()), torch.zeros(2, device=dev())
    lib.p2m_launch_count_reset()
    assert lib.p2m_synthesize_pose(j.data_ptr(), a.data_ptr(), s.data_ptr(), 0, j.data_ptr(), None) == 1
    assert lib.p2m_synthesize_pose(j.data_ptr(), np.zeros(2, np.float32).ctypes.data, s.data_ptr(), 2, j.data_ptr(),
                                   None) == 1
    broken = (_lib.H36MError * 17)()
    C.memmove(broken, table, C.sizeof(broken))
    broken[4].weight = 2.0
    assert lib.p2m_h36m_syn_error(broken, s.data_ptr(), 2, x.data_ptr(), None) == 1
    assert b"entry 4" in lib.p2m_last_error()
    assert lib.p2m_h36m_syn_error(None, s.data_ptr(), 2, x.data_ptr(), None) == 1
    assert lib.p2m_launch_count() == 0
    # the Python layer's own checks
    with pytest.raises(ValueError):
        training_pose2d(x17, "human36")                                   # no error model
    with pytest.raises(ValueError):
        training_pose2d(torch.zeros(0, 19, 2, device=dev()), "coco")
    with pytest.raises(ValueError):
        training_pose2d(torch.zeros(2, 33, 2, device=dev()), "coco", noise=False)
    with pytest.raises(ValueError):
        training_pose2d(x.requires_grad_(), "coco")
    with pytest.raises(ValueError):
        training_pose2d(x17, "mpii")
    with pytest.raises(ValueError):
        training_pose2d(x17, "coco", area_box="loose")
    with pytest.raises(ValueError):
        synthesize_pose(torch.zeros(2, 17, 2, device=dev()), a)
    with pytest.raises(ValueError):
        synthesize_pose(j, a, torch.zeros(2, dtype=torch.int32, device=dev()))
    with pytest.raises(RuntimeError):
        synthesize_pose(j.cpu(), a)


# a COCO skeleton with the pelvis (17) and the neck (18) attached; data/COCO/dataset.py's flip pairs
COCO_SKELETON = ((1, 2), (0, 1), (0, 2), (2, 4), (1, 3), (6, 8), (8, 10), (5, 7), (7, 9), (12, 14), (14, 16),
                 (11, 13), (13, 15), (5, 6), (11, 12), (5, 18), (6, 18), (11, 17), (12, 17), (0, 18), (17, 18))
COCO_FLIP_PAIRS = ((1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))


def test_targets_to_inputs_to_a_training_step():
    """Human36MTargets('coco') -> training_pose2d -> FlatPose2Mesh in train mode -> losses -> backward, all on the
    device."""
    import scipy.sparse as sp
    from helpers import graph_from_fixture
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L
    from pose2mesh_release_b200 import pose2mesh_net
    from test_gpu_targets import cuda, h36m_inputs, h36m_module

    B = 8
    args, _ = h36m_inputs(B, seed=41)
    tg = h36m_module("coco")(*[cuda(a) for a in args])
    torch.manual_seed(3)
    pose2d = training_pose2d(tg["joint_img"], "coco")
    assert pose2d.shape == (B, 19, 2) and torch.isfinite(pose2d).all()
    mats, _ = graph_from_fixture("smpl_small")
    adj = sp.csr_matrix(pg.build_adj(19, COCO_SKELETON, COCO_FLIP_PAIRS))   # the 19-joint input graph
    adj.eliminate_zeros()
    mats[-1] = pg.laplacian(adj, normalized=True)
    flat = pose2mesh_net.get_model(19, mats).to(dev()).train()
    mesh, pose3d = flat(pose2d)
    coord_loss = L.CoordLoss(has_valid=True)
    V = mesh.shape[1]
    loss = coord_loss(pose3d.reshape(B, 19, 3), tg["lift_pose3d"], tg["lift_pose3d_valid"]) + \
        coord_loss(mesh, tg["mesh"][:, :V], tg["mesh_valid"][:, :V])
    loss.backward()
    grads = [p.grad for p in flat.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g).all() for g in grads)
    assert float(flat.pose_lifter.w1.weight.grad.abs().max()) > 0
