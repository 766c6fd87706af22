"""The Trainer's objective on the GPU (loss.Pose2MeshLoss, p2m_pose2mesh_loss and its backward) and the differentiable
joint regression (postprocess.regress_joints), against float64 (tests/pose2mesh_loss_oracle.py).

Every check is element-wise against a bound built from the float64 values (tests/fp64_ref.py style): the fp32 rounding
of each product, normalisation and sum the kernels perform, with eps = 2^-24.  Where a term's argument (a regressed
joint's residual, a face's cos or edge residual) lies within its forward bound of zero the kernel may take either sign
of |.|'s gradient, so that term's whole gradient is allowed as well.  The vertex and lift residuals of 0/1 masks are
exact fp32 differences, whose sign the rounding cannot change."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pose2mesh_loss_cases import INPUTS, make_case

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
WEIGHTS = (0.1, 20.0, 1e-3)
# (n_vertex, n_padded, batch, regressor joints, lifted joints): SMPL's 6890 rows in MeshNet's 12288, MANO's 778 in 1088
SIZES = {"smpl_b1": (6890, 12288, 1, 17, 17), "smpl_b64": (6890, 12288, 64, 19, 17),
         "smpl_b256": (6890, 12288, 256, 24, 17), "mano_b1024": (778, 1088, 1024, 21, 21)}


def dev():
    return torch.device("cuda:0")


def _criterion(c):
    from pose2mesh_release_b200 import loss as L

    return L.Pose2MeshLoss(c["face"], c["joint_regressor"], c["perm_reverse"], *WEIGHTS)


def _run(crit, c, edge, grad=True):
    x = {k: c[k].to(dev()) for k in INPUTS}
    x["cam_mesh"].requires_grad_(grad)
    x["lift_pose"].requires_grad_(grad)
    loss, terms = crit(*(x[k] for k in INPUTS), edge=edge)
    if grad:
        loss.backward()
    return loss.detach(), terms, x["cam_mesh"].grad, x["lift_pose"].grad


def _reference_and_bounds(c, edge):
    """float64 loss, terms, d cam_mesh (real rows, vertex order), d lift_pose, and the bounds of each."""
    import pose2mesh_loss_oracle as lo

    d64 = {k: c[k].to(dev()).double() for k in INPUTS}
    face, perm = c["face"], c["perm_reverse"]
    nv = int(face.max()) + 1
    B, nj, nl = d64["cam_mesh"].shape[0], c["joint_regressor"].shape[0], d64["lift_pose"].shape[1]
    jr = c["joint_regressor"].to(dev()).double()
    rows = torch.as_tensor(perm[:nv], dtype=torch.long, device=dev())
    d64["cam_mesh"].requires_grad_(True)
    d64["lift_pose"].requires_grad_(True)
    loss, terms = lo.pose2mesh_loss(*(d64[k] for k in INPUTS), face, jr, perm, WEIGHTS, edge)
    loss.backward()
    gx, gl = d64["cam_mesh"].grad[:, rows], d64["lift_pose"].grad
    wn, we, wj = WEIGHTS
    x, g, m = d64["cam_mesh"].detach()[:, rows], d64["gt_mesh"], d64["mesh_valid"]
    lp, glp, ml = d64["lift_pose"].detach(), d64["gt_lift3dpose"], d64["lift3dpose_valid"]
    gr, mr = d64["gt_reg3dpose"], d64["reg3dpose_valid"]
    n1, n4, n5, nfs = 3.0 * B * nv, 3.0 * B * nj, 3.0 * B * nl, 3.0 * B * len(face)
    chunks = -(-nv // 256)
    # ---- forward
    b1 = (3 * chunks + 10) * EPS * float(((x * m).abs() + (g * m).abs()).sum()) / n1
    pp = 1000 * torch.matmul(jr, x)
    err_pp = (chunks + 14) * EPS * 1000 * torch.matmul(jr.abs(), x.abs()) + EPS * pp.abs()
    d4 = pp * mr - gr * mr
    err_d4 = (err_pp + 2 * EPS * (pp.abs() + gr.abs())) * mr.abs()
    b4 = wj * float(err_d4.sum() + (-(-3 * nj // 32) + 6) * EPS * d4.abs().sum()) / n4
    b5 = wj * (-(-3 * nl // 32) + 8) * EPS * float(((lp * ml).abs() + (glp * ml).abs()).sum()) / n5
    f = torch.as_tensor(face, dtype=torch.long, device=dev())
    o, t = x[:, f], g[:, f]                                              # [B, nf, 3 corners, 3]
    ends = ((0, 1), (0, 2), (1, 2))
    e = torch.stack([o[:, :, q] - o[:, :, p] for p, q in ends], 2)      # [B, nf, 3 edges, 3]
    le = e.norm(dim=3)
    lg = torch.stack([(t[:, :, q] - t[:, :, p]).norm(dim=2) for p, q in ends], 2)
    cr = torch.cross(F.normalize(t[:, :, 1] - t[:, :, 0], dim=2), F.normalize(t[:, :, 2] - t[:, :, 0], dim=2), dim=2)
    sin_gt = cr.norm(dim=2, keepdim=True)                               # conditioning of the gt normal
    cos = (e / le[..., None] * F.normalize(cr, dim=2)[:, :, None]).sum(3)
    res = le - lg
    err_cos = 32 * EPS * (1 + 1 / sin_gt)                                # [B, nf, 1]
    err_res = 8 * EPS * (le + lg)
    b2 = wn * float(3 * err_cos.sum() + 16 * EPS * cos.abs().sum()) / nfs
    b3 = we * float(err_res.sum() + 16 * EPS * res.abs().sum()) / nfs if edge else 0.0
    bt = torch.tensor([b1, b2, b3, b4, b5], dtype=torch.float64) + EPS * terms.detach().abs().cpu()
    bl = float(bt.sum()) + 4 * EPS * abs(float(loss.detach()))
    # ---- d cam_mesh
    s1, s4, sn, se = 1 / n1, wj / n4, wn / nfs, (we / nfs if edge else 0.0)
    g4 = s4 * torch.sign(d4) * mr
    mag_j = 1000 * torch.matmul(jr.abs().t(), g4.abs())
    amb_j = 2000 * s4 * torch.matmul(jr.abs().t(), (d4.abs() <= err_d4).double() * mr.abs())
    face_mag, face_err, face_amb = (torch.zeros(B, nv, device=dev(), dtype=torch.float64) for _ in range(3))
    for i, (p, q) in enumerate(ends):
        mag = sn / le[:, :, i] + se
        err = 32 * EPS * (1 + 1 / sin_gt[:, :, 0]) * sn / le[:, :, i] + 8 * EPS * se
        amb = 2 * (sn / le[:, :, i] * (cos[:, :, i].abs() <= err_cos[:, :, 0]) + se * (res[:, :, i].abs() <= err_res[:, :, i]))
        for corner in (p, q):
            for acc, val in ((face_mag, mag), (face_err, err), (face_amb, amb)):
                acc.index_add_(1, f[:, corner], val)
    vert = s1 * m.abs()
    bx = (2 * EPS * vert + (nj + 4) * EPS * mag_j + amb_j + (face_err + face_amb + 32 * EPS * face_mag)[..., None]
          + 4 * EPS * (vert + mag_j + face_mag[..., None]))
    blift = 2 * EPS * (wj / n5) * ml.abs().expand_as(lp)
    return (float(loss), terms.detach().cpu(), gx, gl), (bl, bt, bx, blift)


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    worst = float((err / bound.clamp_min(1e-300)).max())
    assert bool((err <= bound).all()), f"{what}: max |err| / bound = {worst:.3g}"


@pytest.mark.parametrize("edge", (True, False))
@pytest.mark.parametrize("size", list(SIZES))
def test_objective_and_gradients_within_float64_bound(size, edge):
    nv, n_padded, B, nj, nl = SIZES[size]
    c = make_case(nv, n_padded, B, nj, nl, seed=100 + B + nj)
    loss, terms, gx, gl = _run(_criterion(c), c, edge)
    (rl, rt, rgx, rgl), (bl, bt, bx, blift) = _reference_and_bounds(c, edge)
    assert terms.dtype == torch.float32 and terms.shape == (5,) and not terms.requires_grad
    assert loss.dtype == torch.float32 and loss.dim() == 0
    _within(terms.cpu(), rt, bt, "terms")
    assert abs(float(loss) - rl) <= bl, (float(loss), rl, bl)
    if not edge:
        assert float(terms[2]) == 0.0
    rows = np.asarray(c["perm_reverse"][:nv])
    pad = np.ones(n_padded, bool)
    pad[rows] = False
    assert gx.shape == (B, n_padded, 3)
    assert int(torch.count_nonzero(gx[:, torch.from_numpy(pad).to(dev())])) == 0    # padding rows exactly zero
    _within(gx[:, torch.from_numpy(rows).long().to(dev())], rgx, bx, "d cam_mesh")
    _within(gl, rgl, blift, "d lift_pose")


def test_fixed_order_terms_are_bitwise_reproducible():
    c = make_case(6890, 12288, 64, 17, 17, seed=7)
    crit = _criterion(c)
    a, b = _run(crit, c, True), _run(crit, c, True)
    assert torch.equal(a[1][[0, 3, 4]], b[1][[0, 3, 4]])
    assert torch.equal(a[3], b[3])                           # d lift_pose has no atomics


def test_launch_counts():
    from pose2mesh_release_b200 import _lib

    c = make_case(778, 1088, 8, 21, 21, seed=3)
    crit = _criterion(c)
    _run(crit, c, True)                                       # tables uploaded
    lib = _lib.load()
    x = {k: c[k].to(dev()) for k in INPUTS}
    x["cam_mesh"].requires_grad_(True)
    torch.cuda.synchronize()
    lib.p2m_launch_count_reset()
    loss, _ = crit(*(x[k] for k in INPUTS), edge=True)
    assert lib.p2m_launch_count() == 2                         # the face kernel and the vertex / joint kernel
    with torch.autograd.set_multithreading_enabled(False):   # the counter is per thread: backward on this one
        lib.p2m_launch_count_reset()
        loss.backward()
        assert lib.p2m_launch_count() == 3


def test_cuda_graph_replay_matches_eager_and_follows_the_edge_flag():
    c = make_case(6890, 12288, 16, 17, 17, seed=5)
    crit = _criterion(c)
    x = {k: c[k].to(dev()) for k in INPUTS}
    x["cam_mesh"].requires_grad_(True)
    x["lift_pose"].requires_grad_(True)
    edge = torch.zeros(1, device=dev())

    def step():
        loss, terms = crit(*(x[k] for k in INPUTS), edge=edge)
        return (loss.detach(), terms) + torch.autograd.grad(loss, [x["cam_mesh"], x["lift_pose"]])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for flag in (0.0, 1.0, 0.0):
        edge.fill_(flag)
        graph.replay()
        torch.cuda.synchronize()
        ref = _run(crit, c, bool(flag))
        assert torch.equal(out[1][[0, 3, 4]], ref[1][[0, 3, 4]]) and torch.equal(out[3], ref[3])
        assert (float(out[1][2]) == 0.0) == (flag == 0.0)
        torch.testing.assert_close(out[1], ref[1], rtol=1e-6, atol=0)
        torch.testing.assert_close(out[0], ref[0], rtol=1e-6, atol=0)
        scale = float(ref[2].abs().max())
        assert float((out[2] - ref[2]).abs().max()) <= 1e-6 * scale   # fp32 atomics of the face kernel


def test_regress_joints_no_grad_is_the_forward_kernel_and_gradient_within_bound():
    from pose2mesh_release_b200 import _lib, postprocess

    g = torch.Generator().manual_seed(8)
    verts = torch.randn(7, 6890, 3, generator=g).to(dev())
    jr = (torch.rand(24, 6890, generator=g) * (torch.rand(24, 6890, generator=g) < 0.03)).to(dev())
    direct = torch.empty(7, 24, 3, device=dev())
    _lib.call("p2m_regress_joints", dev(), jr, verts, direct, 7, 24, 6890, 3)
    assert torch.equal(postprocess.regress_joints(verts, jr), direct)
    v = verts.clone().requires_grad_(True)
    joints = postprocess.regress_joints(v, jr)
    assert torch.equal(joints.detach(), direct)
    dj = torch.randn(7, 24, 3, generator=g).to(dev())
    joints.backward(dj)
    ref = torch.matmul(jr.double().t(), dj.double())
    bound = (24 + 2) * EPS * torch.matmul(jr.double().abs().t(), dj.double().abs())
    _within(v.grad, ref, bound, "d vertices")
    with pytest.raises(ValueError, match="joint_regressor"):
        postprocess.regress_joints(v, jr.clone().requires_grad_(True))


def test_rejects_bad_shapes():
    from pose2mesh_release_b200 import loss as L

    c = make_case(778, 1088, 2, 21, 21, seed=1)
    with pytest.raises(ValueError, match="joint_regressor"):
        L.Pose2MeshLoss(c["face"], torch.zeros(25, 778), c["perm_reverse"])
    with pytest.raises(ValueError, match="perm_reverse"):
        L.Pose2MeshLoss(c["face"], c["joint_regressor"], np.zeros(1088, np.int64))
    crit = _criterion(c)
    x = [c[k].to(dev()) for k in INPUTS]
    with pytest.raises(ValueError, match="cam_mesh"):
        crit(x[0][:, :700], *x[1:])


def test_flat_pose2mesh_train_step_matches_torch_composition():
    """One FlatPose2Mesh training step at SMPL size, B = 64 (native PoseNet and MeshNet), with the objective as one op
    and as the torch composition a user writes without it: same seed, inputs and BatchNorm state."""
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L
    from pose2mesh_release_b200 import pose2mesh_net

    face = pg.synthetic_sphere_faces(6890, 2)
    _, graph_L, _, perm_rev = pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=9)
    torch.manual_seed(123)
    flat = pose2mesh_net.get_model(17, graph_L).to(dev()).train()
    state = {k: v.detach().clone() for k, v in flat.state_dict().items()}
    n_padded = graph_L[0].shape[0]
    c = make_case(6890, n_padded, 64, 17, 17, seed=11)
    rows = torch.as_tensor(np.asarray(perm_rev)[:6890], dtype=torch.long, device=dev())
    jr = c["joint_regressor"].to(dev())
    t = {k: c[k].to(dev()) for k in INPUTS[2:]}
    pose2d = torch.randn(64, 17, 2, generator=torch.Generator().manual_seed(4)).to(dev())
    crit = L.Pose2MeshLoss(face, c["joint_regressor"], perm_rev, *WEIGHTS)
    coord, mesh_losses = L.CoordLoss(has_valid=True), L.MeshLosses(face)

    def step(native):
        flat.load_state_dict(state)
        flat.zero_grad(set_to_none=True)
        torch.manual_seed(7)
        cam_mesh, lift_pose = flat(pose2d)
        if native:
            loss, _ = crit(cam_mesh, lift_pose, t["gt_mesh"], t["gt_reg3dpose"], t["gt_lift3dpose"], t["mesh_valid"],
                           t["reg3dpose_valid"], t["lift3dpose_valid"], edge=True)
        else:
            pred_mesh = cam_mesh[:, rows]
            pred_pose = torch.matmul(jr[None], pred_mesh * 1000)
            normal, edge = mesh_losses(pred_mesh, t["gt_mesh"])
            loss = (coord(pred_mesh, t["gt_mesh"], t["mesh_valid"]) + WEIGHTS[0] * normal
                    + WEIGHTS[2] * coord(pred_pose, t["gt_reg3dpose"], t["reg3dpose_valid"])
                    + WEIGHTS[2] * coord(lift_pose, t["gt_lift3dpose"], t["lift3dpose_valid"]) + WEIGHTS[1] * edge)
        loss.backward()
        return float(loss), {k: p.grad.detach().clone() for k, p in flat.named_parameters() if p.grad is not None}

    la, ga = step(True)
    lb, gb = step(False)
    assert abs(la - lb) <= 1e-3 * abs(lb)
    assert ga.keys() == gb.keys() and len(ga) > 0
    # test_gpu_at_size.py's bound: 1e-3 of the tensor's largest entry, and at least 1e-6 of the model's largest gradient
    # (the biases in front of a train-mode BatchNorm have an exact gradient of zero and hold rounding noise only)
    floor = 1e-3 * max(float(v.abs().max()) for v in gb.values())
    for k in gb:
        scale = max(float(gb[k].abs().max()), floor)
        assert float((ga[k] - gb[k]).abs().max()) <= 1e-3 * scale, k
