"""The single-pass mixed precision (P2M_PREC_FP16_MIXED_TC, "fp16_mixed") on the device: training.

1. One layer against float64: p2m_cheb_conv_fwd with batch-statistics BatchNorm, and p2m_cheb_conv_fwd / _bwd over
   every width of the three conv configurations, the graph families of tests/graphs.py and the persistent CTA loop.
   y, dX, dW and db lie within fp64_ref's bounds at "fp16_mixed", and at least one element of y, dX and dW of each
   tensor-core case lies beyond the fp16x3 bound: the single pass is what ran.
2. The training step layer by layer on test_gpu_network_fp64's TRAIN_CASES and its shifted-channel case: every layer
   from its own captured inputs, the convs held to their single-pass bounds and the fc (an fp16x3 dense GEMM at every
   tensor-core precision) to its fp16x3 bound.  Every conv and dW launch of the step is single-pass, the fc's dense
   GEMM is not, and every layer's route equals fp16x3's.
3. At size: the SMPL B = 256 and MANO B = 1024 training steps layer by layer (test_gpu_at_size_fp64.run_train_case).
4. Eval: bitwise fp16's outputs at full SMPL size, also from a CUDA-graph replay; a model switched back to fp16x3 gives
   bitwise the results of one that never left it.
5. A short seeded Adam fit converges as at fp16x3.
Every test ends with kernel_status == 0."""
import numpy as np
import pytest
import torch

import fp64_ref as R
import graphs as G
from helpers import CASES, graph_from_fixture

pytestmark = pytest.mark.gpu

MIXED = "fp16_mixed"


def dev():
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def clear_conv_log():
    """The launch log (p2m_debug_conv_log) is process-wide and holds 32768 launches; the training steps here, the
    Adam fit most of all, log far more than that.  Each test starts and ends with it empty, so that no later reader in
    the same process finds it overflowed."""
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    lib.p2m_debug_conv_log_reset()
    yield
    lib.p2m_debug_conv_log_reset()


# ------------------------------------------------------------------------------------------------------ 1. one layer
def run_layer(L, x, W, b, dz, sm_cap=0):
    import test_gpu_kernels_fp64 as K

    return K.run(L, x, W, b, MIXED, dz, sm_cap)


def check_layer(tag, L, x, W, b, dz, y, dx, dW, db, p):
    """p: the conv path (p2m_debug_conv_path); y, dX and dW must lie beyond the fp16x3 bound somewhere where their
    pass ran on the tensor cores (dX: the dT GEMMs)."""
    on_tc = {"y": p["conv"], "dx": p["dt"], "dW": p["dw"], "db": 0}
    L = L.tocsr().astype(np.float32).astype(np.float64)
    y64 = R.cheb_conv_fwd(x, L, W, b)
    dx64, dW64, db64 = R.cheb_conv_bwd(x, L, W, dz)
    b16 = (R.cheb_conv_fwd_bound(x, L, W, b, MIXED),) + R.cheb_conv_bwd_bound(x, L, W, dz, MIXED)
    b3 = (R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3"),) + R.cheb_conv_bwd_bound(x, L, W, dz, "fp16x3")
    for i, (what, got, ref) in enumerate((("y", y, y64), ("dx", dx, dx64), ("dW", dW, dW64), ("db", db, db64))):
        err = np.abs(got - ref)
        r = float((err / b16[i]).max())
        assert r <= 1.0, f"{tag} {what}: max |err| / single-pass bound = {r:.3g}"
        if on_tc[what]:
            r3 = float((err / b3[i]).max())
            assert r3 > 1.0, f"{tag} {what}: within the fp16x3 bound ({r3:.3g}): the single pass did not run"


def make_layer(V, B, fin, fout, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    dz = rng.standard_normal((B, V, fout)).astype(np.float32)
    return x, W, b, dz


def level(name):
    fx, i = {"tma": ("smpl_small", 1), "ragged": ("mano_like", 0)}[name]
    return graph_from_fixture(fx)[0][i]


WIDTHS = [(fin, fout) for fin in (32, 64, 128, 160, 256) for fout in (64, 128, 256)]


@pytest.mark.parametrize("lvl", ["tma", "ragged"])
@pytest.mark.parametrize("fin,fout", WIDTHS, ids=lambda v: str(v))
def test_single_layer_width_grid(fin, fout, lvl):
    from pose2mesh_release_b200 import _lib

    L = level(lvl)
    x, W, b, dz = make_layer(L.shape[0], 1, fin, fout, seed=fin * 1000 + fout)
    _lib.conv_log(reset=True)
    y, dx, dW, db, p = run_layer(L, x, W, b, dz)
    log = _lib.conv_log(reset=True)
    assert p["conv"] == 1 and p["dw"] == 1 and p["dt"] == (fin in (64, 128, 256)), p
    # forward conv, dW and (where dX runs on the tensor cores) the three dT GEMMs: all single pass
    kinds = [e["kind"] for e in log]
    assert kinds.count("dw") == -(-fout // 64) * (fin // 32) and all(e["f16"] == 1 for e in log), log
    assert kinds.count("conv") == 1 + 3 * p["dt"], kinds
    check_layer(f"width {fin}->{fout} {lvl}", L, x, W, b, dz, y, dx, dW, db, p)


SYMMETRIC_FAMILIES = ["V1", "V64", "V127", "V128", "V129", "V1088", "band8", "band16", "band20", "h1_256", "h1_257",
                      "far", "hub", "empty_rows", "iso_uniform", "dense"]


@pytest.mark.parametrize("fin,fout", [(64, 64), (128, 128), (256, 256)], ids=lambda v: str(v))
@pytest.mark.parametrize("name", SYMMETRIC_FAMILIES)
def test_single_layer_graph_family(name, fin, fout):
    L = G.get(name)
    x, W, b, dz = make_layer(L.shape[0], 2, fin, fout, seed=L.shape[0] + fin)
    y, dx, dW, db, p = run_layer(L, x, W, b, dz)
    check_layer(f"{name} {fin}->{fout}", L, x, W, b, dz, y, dx, dW, db, p)


@pytest.mark.parametrize("fin,fout", [(64, 64), (128, 128), (256, 256)], ids=lambda v: str(v))
def test_single_layer_persistent_cta_loop(fin, fout):
    """V = 128 on a grid capped at 8 SMs: B = 1, 7, 9 and 29 make each CTA of the conv, the dT GEMMs and the dW run
    from 1 to several tiles."""
    from pose2mesh_release_b200 import _lib

    L = G.get("V128")
    most = {"conv": 0, "dw": 0}
    for B in (1, 7, 9, 29):
        x, W, b, dz = make_layer(128, B, fin, fout, seed=B)
        _lib.conv_log(reset=True)
        y, dx, dW, db, p = run_layer(L, x, W, b, dz, sm_cap=8)
        log = _lib.conv_log(reset=True)
        for e in log:
            assert e["f16"] == 1 and e["grid_x"] == min(e["n_tiles"], max(1, 8 // e["grid_y"])), e
            most[e["kind"]] = max(most[e["kind"]], e["tiles_per_cta"])
        check_layer(f"persistent B={B} {fin}->{fout}", L, x, W, b, dz, y, dx, dW, db, p)
    assert most["conv"] >= 4 and most["dw"] >= 4, most


@pytest.mark.parametrize("fin,fout", [(64, 64), (128, 256), (256, 256)], ids=lambda v: str(v))
@pytest.mark.parametrize("lvl", ["tma", "ragged"])
def test_single_layer_batch_statistics_batchnorm(fin, fout, lvl):
    """p2m_cheb_conv_fwd with bn_mode 2 (refused at fp16) runs at fp16_mixed: y, save_mean / save_invstd and the
    running statistics against float64 with the conv error held to the single-pass bound."""
    import test_gpu_batchnorm_fp64 as BN

    L = level(lvl)
    x, W, b, bn = BN.make_layer(L, 2, fin, fout, seed=fin + fout)
    for relu in (False, True):
        got, p = BN.run_bn_layer(L, x, W, b, bn, 2, relu, MIXED)
        assert p["conv"] == 1 and got["nbt"] == 8, (p, got["nbt"])
        BN.check_train(f"bn2 {fin}->{fout} {lvl} relu={relu}", MIXED, L.tocsr(), x, W, b, bn, got, relu)


# ------------------------------------------------------------------------------------------- 2. network, layer by layer
def routes_at(net, B, need_dx, precision):
    from pose2mesh_release_b200 import _lib

    own = net.hier.precision
    net.hier.set_precision(_lib.PRECISIONS[precision])
    try:
        return [net.route(li, B, need_dx) for li in range(net.n_layers)]
    finally:
        net.hier.set_precision(own)


def train_and_check(net, tag, x, tgt, need_dx):
    import test_gpu_network_fp64 as N
    from pose2mesh_release_b200 import _lib

    B = x.shape[0]
    assert routes_at(net, B, need_dx, MIXED) == routes_at(net, B, need_dx, "fp16x3"), tag
    _lib.conv_log(reset=True)
    cap, grads, bufs, y = N.forward_train_backward(net, x, tgt, need_dx)
    log = _lib.conv_log(reset=True)
    tc = [e for e in log if e["kind"] in ("conv", "dw")]
    assert tc and all(e["f16"] == 1 for e in tc), (tag, [e for e in tc if e["f16"] != 1])
    assert all(e["f16"] == 0 for e in log if e["kind"] == "gemm"), tag
    assert len(tc) + sum(e["kind"] == "gemm" for e in log) == len(log), (tag, log)
    N.check_train(net, tag, x, y, cap, grads, bufs, need_dx)
    assert net.hier.kernel_status(0) == 0


def _train_cases():
    import test_gpu_network_fp64 as N

    return N.TRAIN_CASES


@pytest.mark.parametrize("name,elide,B,need_dx", _train_cases(), ids=lambda v: str(v))
def test_train_step_layer_by_layer(name, elide, B, need_dx):
    import test_gpu_network_fp64 as N

    net = N.Net(name, MIXED, seed=100 * elide + B, open_relus=True)
    net.hier.set_debug(0, elide_padding=elide)
    x, tgt = N.train_inputs(net, B, seed=B + elide)
    train_and_check(net, f"{name} fp16_mixed elide={elide} B={B} dx={need_dx}", x, tgt, need_dx)


def test_train_step_with_shifted_channels():
    import test_gpu_network_fp64 as N

    net = N.Net("custom", MIXED, seed=7, open_relus=True, bias_shift=1000.0)
    x, tgt = N.train_inputs(net, 3, seed=9)
    train_and_check(net, "custom shifted fp16_mixed", x, tgt, True)


# ------------------------------------------------------------------------------------------------------ 3. at size
@pytest.mark.parametrize("name,B", [("smpl_like", 256), ("mano_like", 1024)])
def test_train_at_size(name, B):
    """test_gpu_at_size_fp64.run_train_case at fp16_mixed: its launch check expects the single-pass bit on every conv
    and dW launch, its bounds are the single-pass ones and its routes fp16x3's."""
    import test_gpu_at_size_fp64 as A

    torch.cuda.reset_peak_memory_stats()
    net = A.run_train_case(name, B, MIXED)
    assert net.hier.kernel_status(0) == 0


# ------------------------------------------------------------------------------------------------- 4. eval and back
def test_eval_bitwise_fp16_at_full_size():
    import test_gpu_fp16_inference as F

    m16 = F.smpl_model("fp16")[0]
    mm = F.smpl_model(MIXED)[0]
    x = torch.randn(256, 17, 5, generator=torch.Generator().manual_seed(0)).to(dev())
    with torch.no_grad():
        y16 = m16(x)
        ym = mm(x)
    assert torch.equal(ym, y16), "fp16_mixed's eval forward differs from fp16's"
    xs = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        mm(xs)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        yg = mm(xs)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y16), "CUDA-graph replay at fp16_mixed differs from fp16's eager forward"
    assert mm._hier.kernel_status(0) == 0


def test_switched_back_to_fp16x3_is_bitwise_unchanged():
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats, _ = graph_from_fixture("smpl_small")
    torch.manual_seed(5)
    ref = Pose2Mesh(5, 3, mats, joint_set="human36").to(dev()).set_precision("fp16x3")
    torch.manual_seed(5)
    model = Pose2Mesh(5, 3, mats, joint_set="human36").to(dev()).set_precision(MIXED)
    x = torch.randn(4, 17, 5, generator=torch.Generator().manual_seed(1)).to(dev())
    before = {k: v.clone() for k, v in model.state_dict().items()}
    model.train()
    model(x).abs().mean().backward()             # a training step's forward and backward at fp16_mixed
    model.zero_grad(set_to_none=True)
    with torch.no_grad():
        for k, v in model.state_dict().items():
            v.copy_(before[k])
    model.set_precision("fp16x3")

    def step(m):
        m.train()
        y = m(x)
        y.abs().mean().backward()
        grads = [p.grad.clone() for p in m.parameters()]
        m.eval()
        with torch.no_grad():
            ye = m(x)
        return y.detach(), grads, ye, {k: v.clone() for k, v in m.state_dict().items()}

    with torch.no_grad():
        model.eval()
        ref.eval()
        assert torch.equal(model(x), ref(x)), "eval forward after the switch back"
    a, b = step(model), step(ref)
    # the eval forward bit for bit; the training step to fp16x3's accuracy (the dW partial sums of the CTAs meet in
    # atomic adds, whose order is not fixed from run to run)
    assert torch.equal(a[2], b[2])
    for u, v in [(a[0], b[0])] + list(zip(a[1], b[1])) + [(a[3][k], b[3][k]) for k in b[3] if b[3][k].is_floating_point()]:
        assert float((u - v).abs().max()) <= 1e-5 * float(v.abs().max()) + 1e-30
    assert model._hier.kernel_status(0) == 0


# ------------------------------------------------------------------------------------------------ 5. convergence
# The fit: Pose2Mesh on the smpl_small hierarchy, B = 16 fixed inputs, L1 loss to the eval outputs of a teacher of the
# same architecture (another seed, so the targets are reachable), Adam (lr 1e-3),
# 60 steps from one initialisation at each precision.  The two trajectories start equal and drift apart only through
# rounding (about 2^-11 relative per product at fp16_mixed, 2^-21 at fp16x3), which Adam's normalised steps do not
# amplify over 60 steps.  MARGIN: the final losses must agree to 5 % of the loss the fp16x3 fit removed.  That band is
# a chosen limit: wide against rounding drift, narrow against a wrong gradient (a dW or dX that is off by a scale or a
# transposition leaves the fit far behind, or makes it diverge).
STEPS, MARGIN = 60, 0.05


def fit(precision):
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats, _ = graph_from_fixture("smpl_small")
    torch.manual_seed(11)
    model = Pose2Mesh(5, 3, mats, joint_set="human36").to(dev()).set_precision(precision).train()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(16, 17, 5, generator=g).to(dev())
    torch.manual_seed(12)
    teacher = Pose2Mesh(5, 3, mats, joint_set="human36").to(dev()).set_precision("fp16x3").eval()
    with torch.no_grad():
        tgt = teacher(x)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    losses = []
    for _ in range(STEPS):
        opt.zero_grad(set_to_none=True)
        loss = (model(x) - tgt).abs().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert model._hier.kernel_status(0) == 0
    return np.array(losses)


def test_short_fit_converges_as_fp16x3():
    l3, lm = fit("fp16x3"), fit(MIXED)
    assert np.isfinite(lm).all()
    assert lm[0] == pytest.approx(l3[0], rel=1e-2)
    drop = l3[0] - l3[-1]
    assert drop > 0.2 * l3[0], l3
    assert lm[-1] < 0.8 * lm[0], lm
    assert abs(lm[-1] - l3[-1]) <= MARGIN * drop, (lm[-1], l3[-1], drop)
