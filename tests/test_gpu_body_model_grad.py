"""The body-model backward (p2m_body_model_backward through a differentiable=True SMPLLayer / ManoLayer) on the GPU:

  * accuracy: every case of tests/golden/body_model_grad.npz (the unmodified reference layers' autograd, float64) and
    the float64 restatement at SMPL B in {1, 15, 16, 17, 256, 1000} and MANO B in {1, 1024}, cotangents on the
    vertices, the joints or both, within GRAD_BOUND (derived in tests/test_body_model_grad_cpu.py) per sample and per
    gradient tensor;
  * bitwise determinism, batch-position invariance, NaN isolation, CUDA-graph replay, five launches;
  * argument and workspace errors in Python and the C ABI;
  * autograd end to end: the mesh and coordinate losses through the layer, and 20 Adam steps.
"""
import numpy as np
import pytest
import torch

import body_model_grad_ref as gr
from golden.make_golden_body_model_grad import MODES
from test_body_model_cpu import MODELS
from test_body_model_grad_cpu import CASES, GRAD_BOUND, case, case_cotangents, grad_ratio

from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200.body_model import ManoLayer, SMPLLayer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def note(key, ratio):
    """Print the error-to-bound ratio (shown with -s) and return the error."""
    print(f"{key}: error / bound = {ratio / GRAD_BOUND:.3f}")
    return ratio


def layer_for(key, center_idx=None, differentiable=True):
    m = MODELS[key]
    if key == "smpl":
        return SMPLLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["parents"],
                         m["betas"], center_idx=center_idx, differentiable=differentiable)
    return ManoLayer(m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["weights"], m["betas"],
                     m["hands_mean"], center_idx=center_idx, flat_hand_mean=key.endswith("_flat"), side=m["side"],
                     differentiable=differentiable)


def cuda(a, grad=False):
    if a is None:
        return None
    return torch.as_tensor(np.asarray(a, np.float32)).to(DEV).requires_grad_(grad)


def gpu_vjp(layer, pose, betas, trans, gv, gj):
    """Through autograd: -> (grad_pose, grad_betas, grad_trans) as float64 numpy (None where no gradient)."""
    p, b, t = cuda(pose, True), cuda(betas, True), cuda(trans, True)
    kw = {}
    if b is not None:
        kw["th_betas"] = b
    if t is not None:
        kw["th_trans"] = t
    v, j = layer(p, **kw)
    outs, cots = [], []
    if gv is not None:
        outs.append(v), cots.append(cuda(gv))
    if gj is not None:
        outs.append(j), cots.append(cuda(gj))
    torch.autograd.backward(outs, cots)
    torch.cuda.synchronize()
    f = lambda x: None if x is None or x.grad is None else x.grad.cpu().numpy().astype(np.float64)  # noqa: E731
    return f(p), f(b), f(t)


def random_inputs(key, B, seed):
    rng = np.random.RandomState(seed)
    width = 72 if key == "smpl" else 48
    pose = rng.normal(0.0, 0.6, (B, width)).astype(np.float32)
    betas = rng.normal(0.0, 1.5, (B, 10)).astype(np.float32)
    trans = rng.normal(0.0, 0.5 if key == "smpl" else 0.1, (B, 3)).astype(np.float32)
    return pose, betas, trans


def random_cotangents(key, B, seed, mode):
    rng = np.random.RandomState(seed)
    nv, nj = (6890, 24) if key == "smpl" else (778, 21)
    gv = rng.normal(0.0, 1.0, (B, nv, 3)).astype(np.float32)
    gj = rng.normal(0.0, 1.0, (B, nj, 3)).astype(np.float32)
    return (None if mode == "joints" else gv), (None if mode == "verts" else gj)


def restated(key, pose, betas, trans, gv, gj, center=None, rows=None):
    """The restatement on the samples `rows` (all by default); every batch-wide flag here is set by any sample."""
    rows = np.arange(len(pose)) if rows is None else rows
    s = lambda a: None if a is None else a[rows]  # noqa: E731
    return gr.vjp("smpl" if key == "smpl" else "mano", MODELS[key], s(pose), s(betas), s(trans), center, s(gv),
                  s(gj))[2:]


# ------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_golden_case(name, mode):
    c = case(name)
    gv, gj = case_cotangents(c, mode)
    got = gpu_vjp(layer_for(c["model"], c["center"]), c["pose"], c["betas"], c["trans"], gv, gj)
    assert note(f"golden {name} {mode}", grad_ratio(got, c["grads"][mode])) <= GRAD_BOUND


def _sample_rows(B):
    return np.unique(np.array([0, 1, B // 2, B - 2, B - 1]).clip(0, B - 1))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [1, 15, 16, 17, 256, 1000])
def test_smpl_batch_sizes(B, mode):
    pose, betas, trans = random_inputs("smpl", B, seed=B)
    gv, gj = random_cotangents("smpl", B, B + 1, mode)
    got = gpu_vjp(layer_for("smpl"), pose, betas, trans, gv, gj)
    rows = _sample_rows(B)
    ref = restated("smpl", pose, betas, trans, gv, gj, rows=rows)
    assert note(f"smpl B={B} {mode}", grad_ratio([g[rows] for g in got], ref)) <= GRAD_BOUND


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [1, 1024])
@pytest.mark.parametrize("key", ["mano_right", "mano_left_flat"])
def test_mano_batch_sizes(key, B, mode):
    pose, betas, trans = random_inputs(key, B, seed=B + 7)
    gv, gj = random_cotangents(key, B, B + 8, mode)
    got = gpu_vjp(layer_for(key), pose, betas, trans, gv, gj)
    rows = _sample_rows(B)
    ref = restated(key, pose, betas, trans, gv, gj, rows=rows)
    assert note(f"{key} B={B} {mode}", grad_ratio([g[rows] for g in got], ref)) <= GRAD_BOUND


@pytest.mark.parametrize("key,center", [("smpl", 0), ("smpl", 7), ("mano_right", 9), ("mano_left", 4)])
def test_centring_against_restatement(key, center):
    pose, betas, _ = random_inputs(key, 20, seed=30)
    gv, gj = random_cotangents(key, 20, 31, "both")
    for trans in (None, np.zeros((20, 3), np.float32)):
        got = gpu_vjp(layer_for(key, center), pose, betas, trans, gv, gj)
        ref = restated(key, pose, betas, trans, gv, gj, center=center)
        assert note(f"centre {key} {center}", grad_ratio(got, ref)) <= GRAD_BOUND


def test_betas_gradient_rules():
    smpl = layer_for("smpl")
    pose, betas, trans = random_inputs("smpl", 4, seed=40)
    gv, gj = random_cotangents("smpl", 4, 41, "both")
    _, gb, _ = gpu_vjp(smpl, pose, np.zeros_like(betas), trans, gv, gj)
    assert np.array_equal(gb, np.zeros_like(betas))  # the all-zero batch is replaced by the model's betas
    assert gpu_vjp(smpl, pose, None, trans, gv, gj)[1] is None
    p, one = cuda(pose, True), torch.zeros(1, requires_grad=True)
    v, _ = smpl(p, one)  # the reference's default argument counts as absent
    v.sum().backward()
    assert one.grad is None and p.grad is not None
    mano = layer_for("mano_right")
    mp, mb, mt = random_inputs("mano_right", 3, seed=42)
    mgv, mgj = random_cotangents("mano_right", 3, 43, "both")
    got = gpu_vjp(mano, mp, np.zeros_like(mb), mt, mgv, mgj)  # an explicit zero MANO batch is used as given
    ref = restated("mano_right", mp, np.zeros_like(mb), mt, mgv, mgj)
    assert np.abs(got[1]).max() > 0 and note("mano zero betas", grad_ratio(got, ref)) <= GRAD_BOUND


def test_trans_gradient_rules():
    layer = layer_for("smpl", center_idx=0)
    pose, betas, trans = random_inputs("smpl", 3, seed=44)
    gv, gj = random_cotangents("smpl", 3, 45, "both")
    assert np.array_equal(gpu_vjp(layer, pose, betas, np.zeros_like(trans), gv, gj)[2], np.zeros_like(trans))
    # a scalar trans is expanded by torch before the layer's Function: autograd reduces its gradient
    p, s = cuda(pose, True), torch.tensor(0.3, device=DEV, requires_grad=True)
    v, j = layer(p, cuda(betas), s)
    torch.autograd.backward([v, j], [cuda(gv), cuda(gj)])
    full = gpu_vjp(layer, pose, betas, np.full_like(trans, 0.3), gv, gj)[2]
    assert abs(s.grad.item() - full.sum()) <= 1e-5 * np.abs(full).sum()


def test_outputs_bitwise_equal_to_default_layer():
    pose, betas, trans = (cuda(a) for a in random_inputs("smpl", 33, seed=46))
    a = layer_for("smpl", differentiable=False)(pose, betas, trans)
    b = layer_for("smpl")(pose.clone().requires_grad_(True), betas, trans)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_second_backward_raises():
    layer = layer_for("smpl")
    p = cuda(random_inputs("smpl", 2, seed=47)[0], True)
    v, _ = layer(p)
    loss = v.square().sum()
    loss.backward()
    with pytest.raises(RuntimeError):
        loss.backward()
    v, _ = layer(p)
    g = torch.autograd.grad(v.square().sum(), p, create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()


# ------------------------------------------------------------------------------------------------ the C ABI
def abi_backward(layer, pose, betas, trans, gv, gj, want_betas=True, want_trans=True, ws_bytes=None, rule=None,
                 center=-1):
    lib = _lib.load()
    h = layer.handle(0)
    B = pose.shape[0]
    gp = torch.empty_like(pose)
    gb = torch.empty_like(betas) if want_betas and betas is not None else None
    gt = torch.empty_like(trans) if want_trans and trans is not None else None
    need = lib.p2m_body_model_backward_workspace_bytes(h, B)
    ws = torch.empty(need, device=DEV, dtype=torch.uint8)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    rule = _lib.P2M_BETAS_ZERO_MEANS_MODEL if rule is None else rule
    st = lib.p2m_body_model_backward(h, pose.data_ptr(), ptr(betas), rule, ptr(trans), center, ptr(gv), ptr(gj),
                                     ptr(gp), ptr(gb), ptr(gt), B, ws.data_ptr(),
                                     need if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return st, gp, gb, gt


def test_null_betas_and_trans_outputs():
    layer = layer_for("smpl")
    pose, betas, trans = (cuda(a) for a in random_inputs("smpl", 40, seed=50))
    gv, gj = (cuda(a) for a in random_cotangents("smpl", 40, 51, "both"))
    st, gp, gb, gt = abi_backward(layer, pose, betas, trans, gv, gj)
    assert st == 0
    for wb, wt in ((False, True), (True, False), (False, False)):
        st, gp2, gb2, gt2 = abi_backward(layer, pose, betas, trans, gv, gj, wb, wt)
        assert st == 0 and torch.equal(gp, gp2)
        assert (gb2 is None) == (not wb) and (gt2 is None) == (not wt)
        assert gb2 is None or torch.equal(gb, gb2)
        assert gt2 is None or torch.equal(gt, gt2)
    # NULL cotangents are zeros
    st, gp_v, _, _ = abi_backward(layer, pose, betas, trans, gv, None)
    st2, gp_v2, _, _ = abi_backward(layer, pose, betas, trans, gv, torch.zeros_like(gj))
    assert st == st2 == 0 and torch.equal(gp_v, gp_v2)


def test_abi_errors():
    lib = _lib.load()
    layer = layer_for("smpl")
    pose, betas, trans = (cuda(a) for a in random_inputs("smpl", 4, seed=52))
    gv, gj = (cuda(a) for a in random_cotangents("smpl", 4, 53, "both"))
    h = layer.handle(0)
    need = lib.p2m_body_model_backward_workspace_bytes(h, 4)
    assert need > 0 and lib.p2m_body_model_backward_workspace_bytes(h, 0) == 0
    assert lib.p2m_body_model_backward_workspace_bytes(None, 4) == 0
    assert abi_backward(layer, pose, betas, trans, gv, gj, ws_bytes=need - 1)[0] == 3  # P2M_ERR_WORKSPACE
    assert "workspace" in lib.p2m_last_error().decode()
    assert abi_backward(layer, pose, betas, trans, gv, gj, rule=7)[0] == 1  # P2M_ERR_INVALID
    assert "bad argument" in lib.p2m_last_error().decode()
    assert abi_backward(layer, pose, betas, trans, gv, gj, center=24)[0] == 1
    ws = torch.empty(need, device=DEV, dtype=torch.uint8)
    st = lib.p2m_body_model_backward(h, pose.data_ptr(), None, 0, None, -1, gv.data_ptr(), None, None, None, None, 4,
                                     ws.data_ptr(), need, None)
    assert st != 0 and "grad_pose" in lib.p2m_last_error().decode()
    assert lib.p2m_body_model_backward(h, pose.data_ptr(), None, 0, None, -1, None, None, pose.data_ptr(), None, None,
                                       0, ws.data_ptr(), need, None) != 0


def test_python_argument_errors():
    layer = layer_for("smpl")
    pose, betas, trans = (cuda(a, True) for a in random_inputs("smpl", 4, seed=54))
    with pytest.raises(ValueError):
        layer(pose, betas[:3])
    with pytest.raises(ValueError):
        layer(pose[:, :69], betas)
    with pytest.raises(ValueError):
        layer(pose, betas, trans[:2])
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(pose.detach().cpu().requires_grad_(True))


# ------------------------------------------------------------------------------------------------ determinism
def test_bitwise_deterministic_and_batch_position_invariant():
    layer = layer_for("smpl")
    pose, betas, trans = random_inputs("smpl", 64, seed=60)
    gv, gj = random_cotangents("smpl", 64, 61, "both")
    a = gpu_vjp(layer, pose, betas, trans, gv, gj)
    b = gpu_vjp(layer, pose, betas, trans, gv, gj)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    ref = [g[:1] for g in a]
    for pos in (15, 16, 17, 63):
        sw = lambda x: np.concatenate([x[1:pos + 1], x[:1], x[pos + 1:]])  # noqa: E731  sample 0 moved to pos
        got = gpu_vjp(layer, sw(pose), sw(betas), sw(trans), sw(gv), sw(gj))
        assert all(np.array_equal(g[pos:pos + 1], r) for g, r in zip(got, ref)), pos
    for B in (1, 17, 40):
        got = gpu_vjp(layer, pose[:B], betas[:B], trans[:B], gv[:B], gj[:B])
        assert all(np.array_equal(g[:1], r) for g, r in zip(got, ref)), B


def test_mano_batch_position_invariant():
    layer = layer_for("mano_right", center_idx=4)
    pose, betas, _ = random_inputs("mano_right", 40, seed=62)
    gv, gj = random_cotangents("mano_right", 40, 63, "both")
    full = gpu_vjp(layer, pose, betas, None, gv, gj)
    one = gpu_vjp(layer, pose[33:34], betas[33:34], None, gv[33:34], gj[33:34])
    assert all(np.array_equal(f[33:34], o) for f, o in zip(full, one) if o is not None)


def test_nan_isolation():
    layer = layer_for("smpl")
    pose, betas, trans = random_inputs("smpl", 40, seed=64)
    gv, gj = random_cotangents("smpl", 40, 65, "both")
    ref = gpu_vjp(layer, pose, betas, trans, gv, gj)
    keep = np.arange(40) != 17
    for what in ("pose", "grad_verts"):
        p, g = pose.copy(), gv.copy()
        if what == "pose":
            p[17, 5] = np.nan
        else:
            g[17, 100, 1] = np.nan
        got = gpu_vjp(layer, p, betas, trans, g, gj)
        assert all(np.array_equal(x[keep], r[keep]) for x, r in zip(got, ref)), what
        assert not np.isfinite(got[0][17]).all(), what


def test_zero_pose_and_large_angles_are_finite():
    layer = layer_for("smpl")
    pose = np.zeros((3, 72), np.float32)
    pose[1, 3:6] = [0, 0, 3 * np.pi]
    pose[2, 6:9] = [1e-7, 0, 0]
    _, betas, trans = random_inputs("smpl", 3, seed=66)
    gv, gj = random_cotangents("smpl", 3, 67, "both")
    got = gpu_vjp(layer, pose, betas, trans, gv, gj)
    assert all(np.isfinite(g).all() for g in got)
    assert note("zero / large angles", grad_ratio(got, restated("smpl", pose, betas, trans, gv, gj))) <= GRAD_BOUND


def test_cuda_graph_replay_matches_eager():
    layer = layer_for("smpl", center_idx=0)
    pose, betas, trans = (cuda(a) for a in random_inputs("smpl", 32, seed=70))
    gv, gj = (cuda(a) for a in random_cotangents("smpl", 32, 71, "both"))

    def step(p, b, t):
        p, b, t = (x.detach().requires_grad_(True) for x in (p, b, t))
        v, j = layer(p, b, t)
        torch.autograd.backward([v, j], [gv, gj])
        return v.detach(), j.detach(), p.grad, b.grad, t.grad

    zero = torch.zeros_like(trans)
    eager = {k: [x.clone() for x in step(pose, betas, t)] for k, t in (("zero", zero), ("trans", trans))}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(pose, betas, trans)
    torch.cuda.current_stream().wait_stream(s)
    p_in, b_in, t_in = pose.clone(), betas.clone(), trans.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step(p_in, b_in, t_in)
    for k, t in (("zero", zero), ("trans", trans)):
        t_in.copy_(t)
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(o, e) for o, e in zip(out, eager[k])), k


@pytest.mark.parametrize("key", ["smpl", "mano_right"])
def test_five_launches(key):
    """The launch counter is per host thread, and autograd runs backward on its own thread: count the C call."""
    layer = layer_for(key)
    pose, betas, trans = (cuda(a) for a in random_inputs(key, 8, seed=72))
    gv, gj = (cuda(a) for a in random_cotangents(key, 8, 73, "both"))
    lib = _lib.load()
    abi_backward(layer, pose, betas, trans, gv, gj)
    lib.p2m_launch_count_reset()
    assert abi_backward(layer, pose, betas, trans, gv, gj)[0] == 0
    assert lib.p2m_launch_count() == 5


# ------------------------------------------------------------------------------------------------ autograd chains
def ref_verts(pose, betas, trans):
    with torch.no_grad():
        return gr.outputs("smpl", MODELS["smpl"], gr._t(pose), gr._t(betas), gr._t(trans), None)[0].numpy()


def test_losses_through_the_layer():
    from oracle import loss_oracle as lo
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200 import loss as L

    B = 8
    pose, betas, trans = random_inputs("smpl", B, seed=80)
    rng = np.random.RandomState(81)
    tgt_v = (ref_verts(pose, betas, trans) + rng.normal(0.0, 0.05, (B, 6890, 3))).astype(np.float32)
    tgt_j = rng.normal(0.0, 0.5, (B, 24, 3)).astype(np.float32)
    face = pg.synthetic_sphere_faces(6890, 2)
    layer = layer_for("smpl")
    p, b, t = cuda(pose, True), cuda(betas, True), cuda(trans, True)
    v, j = layer(p, b, t)
    ln, le = L.MeshLosses(face)(v, cuda(tgt_v))
    loss = L.CoordLoss()(v, cuda(tgt_v)) + L.CoordLoss()(j, cuda(tgt_j)) + ln + le
    loss.backward()
    got = [x.grad.cpu().numpy().astype(np.float64) for x in (p, b, t)]

    pt, bt, tt = (gr._t(a).requires_grad_(True) for a in (pose, betas, trans))
    rv, rj = gr.outputs("smpl", MODELS["smpl"], pt, bt, tt, None)
    ft = torch.as_tensor(np.asarray(face, np.int64))
    tv, tj = gr._t(tgt_v), gr._t(tgt_j)
    rloss = (lo.coord_loss(rv, tv) + lo.coord_loss(rj, tj) + lo.normal_vector_loss(rv, tv, ft)
             + lo.edge_length_loss(rv, tv, ft))
    rloss.backward()
    assert abs(loss.item() - rloss.item()) <= 1e-5 * abs(rloss.item())
    ref = [x.grad.numpy() for x in (pt, bt, tt)]
    assert note("losses through the layer", grad_ratio(got, ref)) <= GRAD_BOUND


def test_adam_loop_tracks_float64():
    """20 Adam steps on pose, betas and trans at B=64 (lr 0.01, mean squared vertex distance to a target), on the GPU
    layer and on the float64 restatement from the same start.  Each step's gradient agrees to GRAD_BOUND of its
    largest entry; Adam divides by sqrt(v), so a step moves each parameter by at most ~lr whatever the gradient's
    scale, and an fp32 difference of relative size e in the gradient moves a step by about lr e.  Over 20 steps the
    parameters may drift apart by about 20 lr GRAD_BOUND (5e-5) plus the fp32 rounding of the parameters themselves
    (~1e-7); entries whose gradient is near zero may flip Adam's direction for a step, so the bound is 10 lr per
    parameter at worst and 20 lr GRAD_BOUND x 10 on the median."""
    B, lr, steps = 64, 0.01, 20
    pose, betas, trans = random_inputs("smpl", B, seed=90)
    rng = np.random.RandomState(91)
    tp, tb, tt = (pose + rng.normal(0, 0.2, pose.shape), betas + rng.normal(0, 0.5, betas.shape),
                  trans + rng.normal(0, 0.1, trans.shape))
    target = ref_verts(tp, tb, tt)
    layer = layer_for("smpl")
    gpu = [cuda(a, True) for a in (pose, betas, trans)]
    ref = [gr._t(a).requires_grad_(True) for a in (pose, betas, trans)]
    opt_g, opt_r = torch.optim.Adam(gpu, lr=lr), torch.optim.Adam(ref, lr=lr)
    tgt_g, tgt_r = cuda(target), gr._t(target)
    for _ in range(steps):
        opt_g.zero_grad(), opt_r.zero_grad()
        v, _ = layer(*gpu)
        ((v - tgt_g) ** 2).sum(-1).mean().backward()
        rv, _ = gr.outputs("smpl", MODELS["smpl"], *ref, None)
        ((rv - tgt_r) ** 2).sum(-1).mean().backward()
        opt_g.step(), opt_r.step()
    for g, r in zip(gpu, ref):
        d = np.abs(g.detach().cpu().numpy().astype(np.float64) - r.detach().numpy())
        moved = np.abs(r.detach().numpy() - np.asarray(pose if r is ref[0] else betas if r is ref[1] else trans))
        assert moved.max() > 5 * lr  # the loop did move the parameters
        assert d.max() <= 10 * lr and np.median(d) <= 20 * lr * GRAD_BOUND * 10

