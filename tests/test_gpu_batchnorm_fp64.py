"""MeshNet's BatchNorm kernels element-wise against float64 (tests/fp64_ref.py), at both precisions.

Single layer: p2m_cheb_conv_fwd with bn_mode 1 (eval affine folded into the conv epilogue: k_bn_fold_eval) and
bn_mode 2 (batch statistics: k_col_stats, k_bn_finalize, k_affine_act / k_affine_act4) over every BatchNorm layer
shape of the shipped channel plans, statistics blocks below / at / above 512 rows, Fout > 256, widths and a y pointer
that take the scalar k_affine_act, channels shifted through the conv bias to mean / sigma up to 1000 and a constant
channel; save_mean / save_invstd, the running statistics and num_batches_tracked against float64.

Network: on small custom channel plans, the train-mode BN backward and the residual / unpool epilogue (only reachable
through p2m_meshnet_forward / _backward): invariance to a constant added to every conv bias in front of a BatchNorm,
and the scalar BN paths against float64 autograd over the oracle.

The worst error-to-bound ratio per precision is written to the JSON file named by P2M_BN_FP64_REPORT (if set)."""
import ctypes as C
import json
import os
import time

import numpy as np
import pytest
import torch

import fp64_ref as R
from helpers import graph_from_fixture

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16x3"]
_WORST = {}
RATIOS = [0, 10, 100, 1000]   # mean / sigma of the channels, cyclically; channel 1 is constant


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    out = os.environ.get("P2M_BN_FP64_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump({"wall_s": time.time() - t0, "worst_ratio": _WORST}, f, indent=1)


def dev():
    return torch.device("cuda:0")


def check(what, precision, got, ref, bound):
    r = R.bound_ratio(got, ref, bound)
    if r > _WORST.setdefault(precision, [0.0, ""])[0]:
        _WORST[precision] = [r, what]
    assert r <= 1.0, f"{what}: max |err| / bound = {r:.3g}"


def cuda(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a)).to(dtype=dtype, device=dev()).contiguous()


def conv_path(h, fin, fout):
    from pose2mesh_release_b200 import _lib

    out = (C.c_int32 * 9)()
    _lib.check(_lib.load().p2m_debug_conv_path(h, 0, fin, fout, out), "p2m_debug_conv_path")
    return dict(zip(("conv", "conv_xs", "dw", "dw_xs", "dt", "dt_xs", "tma", "max_h1", "n_iso"), list(out)))


# ------------------------------------------------------------------------------------------------------ single layer
def make_layer(L, B, fin, fout, seed, ratios=RATIOS):
    """x, W, b (conv bias carrying mean / sigma = ratios[f % len]; channel 1 constant: zero weights, bias 3) and BN
    parameters."""
    V = L.shape[0]
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2 / (3 * fin + fout))
         * 2.0 ** rng.uniform(-4, 1, (fout, 1))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    sig = R.cheb_conv_fwd(x, L, W, b).reshape(-1, fout).std(axis=0)
    b = (b + np.resize(np.asarray(ratios, np.float64), fout) * sig).astype(np.float32)
    if fout > 1:
        W[1] = 0.0
        b[1] = 3.0
    bn = dict(gamma=((rng.random(fout) + 0.5) * rng.choice([-1, 1], fout)).astype(np.float32),
              beta=(rng.standard_normal(fout) * 0.5).astype(np.float32),
              rm=rng.standard_normal(fout).astype(np.float32), rv=(rng.random(fout) + 0.5).astype(np.float32))
    return x, W, b, bn


def run_bn_layer(L, x, W, b, bn, mode, relu, precision, y_offset=0, null_running=False, null_nbt=False):
    """p2m_cheb_conv_fwd with bn_mode `mode`; returns dict of float64 numpy results and the conv path."""
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200 import cheby_graph_conv as cgc

    lib = _lib.load()
    B, V, fin = x.shape
    fout = W.shape[0]
    cgc.set_default_precision(precision)
    try:
        gh = cgc.graph_handle(L)
        h = gh.handle(0)
        xg, Wg, bg = cuda(x), cuda(W), cuda(b)
        gam, bet = cuda(bn["gamma"]), cuda(bn["beta"])
        rm, rv = cuda(bn["rm"]), cuda(bn["rv"])
        nbt = torch.full((1,), 7, dtype=torch.int64, device=dev())
        smean = torch.full((fout,), float("nan"), device=dev())
        sinv = torch.full((fout,), float("nan"), device=dev())
        ybuf = torch.full((B * V * fout + y_offset,), float("nan"), device=dev())
        nbytes = lib.p2m_cheb_conv_workspace_bytes(h, 0, B, fin, fout)
        ws = torch.empty(nbytes, device=dev(), dtype=torch.uint8)
        a = _lib.ConvFwdArgs(level=0, batch=B, fin=fin, fout=fout, x=xg.data_ptr(), weight=Wg.data_ptr(),
                             bias=bg.data_ptr(), bn_mode=mode, bn_weight=gam.data_ptr(), bn_bias=bet.data_ptr(),
                             bn_running_mean=None if null_running else rm.data_ptr(),
                             bn_running_var=None if null_running else rv.data_ptr(),
                             bn_num_batches_tracked=None if null_nbt else nbt.data_ptr(),
                             save_mean=smean.data_ptr(), save_invstd=sinv.data_ptr(), relu=int(relu),
                             y=ybuf.data_ptr() + 4 * y_offset)
        with torch.cuda.device(dev()):
            _lib.check(lib.p2m_cheb_conv_fwd(h, C.byref(a), ws.data_ptr(), nbytes,
                                             torch.cuda.current_stream(dev()).cuda_stream), "p2m_cheb_conv_fwd")
        torch.cuda.synchronize()
        assert gh.kernel_status(0) == 0
        p = conv_path(h, fin, fout)
    finally:
        cgc.set_default_precision("fp32")
    out = dict(y=ybuf[y_offset:].view(B, V, fout), rm=rm, rv=rv, mean=smean, invstd=sinv)
    out = {k: v.double().cpu().numpy() for k, v in out.items()}
    out["nbt"] = int(nbt.item())
    return out, p


def check_train(tag, precision, L, x, W, b, bn, got, relu, running=True):
    z64 = R.cheb_conv_fwd(x, L, W, b)
    E = R.cheb_conv_fwd_bound(x, L, W, b, precision)
    y64, mean, var, rm64, rv64 = R.bn_train_fwd(z64, bn["gamma"], bn["beta"], bn["rm"], bn["rv"], relu)
    bd = R.bn_train_fwd_bound(z64, E, bn["gamma"], bn["beta"], bn["rm"], bn["rv"])
    check(tag + "/y", precision, got["y"], y64, bd["y"])
    check(tag + "/save_mean", precision, got["mean"], mean, bd["mean"])
    check(tag + "/save_invstd", precision, got["invstd"], 1 / np.sqrt(var + R.BN_EPS), bd["invstd"])
    if running:
        check(tag + "/running_mean", precision, got["rm"], rm64, bd["rm"])
        check(tag + "/running_var", precision, got["rv"], rv64, bd["rv"])


def check_eval(tag, precision, L, x, W, b, bn, got, relu):
    z64 = R.cheb_conv_fwd(x, L, W, b)
    E = R.cheb_conv_fwd_bound(x, L, W, b, precision)
    y64 = R.bn_eval_fwd(z64, bn["gamma"], bn["beta"], bn["rm"], bn["rv"], relu)
    check(tag + "/y_eval", precision, got["y"], y64, R.bn_eval_fwd_bound(z64, E, bn["gamma"], bn["beta"], bn["rm"],
                                                                           bn["rv"], b))


def plan_bn_shapes():
    """(plan, level size, Fin, Fout) of every BatchNorm layer of the shipped plans (meshnet.py's block -> level map:
    block i on laps[-(i + 1)], the last block on the finest level)."""
    from pose2mesh_release_b200.meshnet import channel_plan

    out = set()
    for name, mano in (("smpl_small", False), ("mano_like", True)):
        mats = list(graph_from_fixture(name)[0])
        del mats[-2]
        plan = channel_plan(5, 3, mano)
        for i, chans in enumerate(plan):
            lap = mats[-(i + 1) + (1 if i == len(plan) - 1 else 0)]
            for j in range(len(chans) - 1):
                if not (i == len(plan) - 1 and j == len(chans) - 2):
                    out.add((name, lap.shape[0], chans[j], chans[j + 1]))
    return sorted(out)


def level_of(name, V):
    return next(m for m in graph_from_fixture(name)[0] if m.shape[0] == V)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,V,fin,fout", plan_bn_shapes(), ids=lambda v: str(v))
def test_plan_layer_batchnorm(name, V, fin, fout, precision):
    L = level_of(name, V)
    for B in (1, 2, 3):
        x, W, b, bn = make_layer(L, B, fin, fout, seed=V + fin + fout + B)
        relu = B != 2
        tag = f"{name} V={V} {fin}->{fout} B={B}"
        got, p = run_bn_layer(L, x, W, b, bn, 2, relu, precision)
        assert p["conv"] == (precision == "fp16x3" and fin % 32 == 0), p
        check_train(tag, precision, L, x, W, b, bn, got, relu)
        assert got["nbt"] == 8
        bn_e = dict(bn, rm=(R.cheb_conv_fwd(x, L, W, b).reshape(-1, fout).mean(axis=0)).astype(np.float32))
        got, _ = run_bn_layer(L, x, W, b, bn_e, 1, relu, precision)
        check_eval(tag, precision, L, x, W, b, bn_e, got, relu)
        assert got["nbt"] == 7 and np.array_equal(got["rm"], bn_e["rm"]) and np.array_equal(got["rv"], bn_e["rv"])


# rows = B * V around the 512-row statistics block; Fout > 256 (more channels than lanes); Fout 12 / 36 (scalar path)
EDGE = [(511, 1, 64, 64), (512, 1, 64, 64), (513, 1, 64, 64), (256, 2, 32, 128), (257, 2, 64, 64),
        (1088, 2, 64, 320), (1088, 1, 32, 512), (136, 3, 20, 12), (1088, 1, 64, 36), (17, 1, 64, 36)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("V,B,fin,fout", EDGE, ids=lambda v: str(v))
def test_edge_layer_batchnorm(V, B, fin, fout, precision):
    import graphs as G

    L = G.sized(V)
    x, W, b, bn = make_layer(L, B, fin, fout, seed=V * 7 + fout)
    for relu in (False, True):
        tag = f"edge V={V} B={B} {fin}->{fout} relu={relu}"
        got, _ = run_bn_layer(L, x, W, b, bn, 2, relu, precision)
        check_train(tag, precision, L, x, W, b, bn, got, relu)
        got, _ = run_bn_layer(L, x, W, b, bn, 1, relu, precision)
        check_eval(tag, precision, L, x, W, b, bn, got, relu)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_misaligned_output_and_null_state(precision):
    """y one float off 16-byte alignment (scalar k_affine_act), NULL running statistics and NULL num_batches_tracked
    (both optional in mode 2: y, save_mean and save_invstd still right, nothing else written)."""
    L = level_of("mano_like", 1088)
    x, W, b, bn = make_layer(L, 2, 64, 64, seed=21)
    got, _ = run_bn_layer(L, x, W, b, bn, 2, True, precision, y_offset=1)
    check_train("misaligned y", precision, L, x, W, b, bn, got, True)
    got, _ = run_bn_layer(L, x, W, b, bn, 1, True, precision, y_offset=1)
    check_eval("misaligned y", precision, L, x, W, b, bn, got, True)
    got, _ = run_bn_layer(L, x, W, b, bn, 2, False, precision, null_running=True, null_nbt=True)
    check_train("null running", precision, L, x, W, b, bn, got, False, running=False)
    assert got["nbt"] == 7
    assert np.array_equal(got["rm"], bn["rm"].astype(np.float64)) and np.array_equal(got["rv"], bn["rv"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_eval_running_variance_extremes(precision):
    """Eval mode with running_var from 1e-8 (scale ~ 316 gamma) to 1e4, and a large running mean against the bias."""
    L = level_of("smpl_small", 1024)
    x, W, b, bn = make_layer(L, 1, 64, 128, seed=31)
    rng = np.random.default_rng(32)
    bn["rv"] = (np.resize([1e-8, 1e-4, 1.0, 1e4], 128) * (rng.random(128) + 0.5)).astype(np.float32)
    bn["rm"] = (R.cheb_conv_fwd(x, L, W, b).reshape(-1, 128).mean(axis=0) + rng.standard_normal(128)).astype(np.float32)
    for relu in (False, True):
        got, _ = run_bn_layer(L, x, W, b, bn, 1, relu, precision)
        check_eval(f"rv extremes relu={relu}", precision, L, x, W, b, bn, got, relu)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("ratio", [100, 1000])
def test_shifted_channels_in_every_channel(ratio, precision):
    """Every channel at mean / sigma = ratio (the one-pass variance loses ~(ratio^2 sqrt(m) u) of it)."""
    L = level_of("mano_like", 1088)
    x, W, b, bn = make_layer(L, 2, 64, 64, seed=ratio, ratios=[ratio])
    got, _ = run_bn_layer(L, x, W, b, bn, 2, False, precision)
    check_train(f"all channels at {ratio}", precision, L, x, W, b, bn, got, False)


# ------------------------------------------------------------------------------------------------------------ network
def small_net(levels, plan, precision, seed, open_relus=True, bias_shift=0.0):
    """A MeshNet of `plan` over the given Laplacians (fine -> coarse, joint graph last; len(plan) - 1 of them) through
    BakedHierarchy and _MeshNetFunction directly; reference-layout state dict with the oracle's initialiser, BN bias 6
    (open ReLUs: no pre-activation near zero) and `bias_shift` added to every conv bias in front of a BatchNorm."""
    from oracle import meshnet_oracle as mo
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200.meshnet import BakedHierarchy

    torch.manual_seed(seed)
    n_layers = sum(len(p) - 1 for p in plan)
    sd = {}
    fc = torch.nn.Linear(levels[-1].shape[0] * plan[0][-1], levels[-2].shape[0] * plan[1][0])
    sd["fc.weight"], sd["fc.bias"] = fc.weight.detach().clone(), fc.bias.detach().clone() * 0.1
    idx = 0
    for chans in plan:
        for fin, fout in zip(chans[:-1], chans[1:]):
            bound = float(np.sqrt(2.0 / (3 * fin + fout)))
            sd[f"cl.{idx}.weight"] = (torch.rand(fout, 3 * fin) * 2 - 1) * bound
            sd[f"cl.{idx}.bias"] = torch.randn(fout) * 0.1
            if idx != n_layers - 1:
                sd[f"cl.{idx}.bias"] += bias_shift
                sd[f"bn.{idx}.weight"] = torch.rand(fout) + 0.5
                sd[f"bn.{idx}.bias"] = torch.full((fout,), 6.0) if open_relus else torch.randn(fout) * 0.1
                sd[f"bn.{idx}.running_mean"] = torch.randn(fout) * 0.1
                sd[f"bn.{idx}.running_var"] = torch.rand(fout) + 0.5
                sd[f"bn.{idx}.num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
            idx += 1
    hier = BakedHierarchy(levels, plan)
    hier.set_precision(_lib.PRECISIONS[precision])
    return hier, sd, n_layers, mo


def net_train_step(hier, sd, n_layers, x, tgt):
    """One train-mode forward + L1 loss + backward through the native library.  Returns (y, loss, grads by name,
    new running stats by name, dx)."""
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    n_bn = n_layers - 1
    p = {k: cuda(v).requires_grad_(True) for k, v in sd.items() if "running" not in k and "num_batches" not in k}
    buf = {k: cuda(v) if v.is_floating_point() else v.to(dev()) for k, v in sd.items()
           if "running" in k or "num_batches" in k}
    names = (["fc.weight", "fc.bias"] + [f"cl.{i}.weight" for i in range(n_layers)]
             + [f"cl.{i}.bias" for i in range(n_layers)] + [f"bn.{i}.weight" for i in range(n_bn)]
             + [f"bn.{i}.bias" for i in range(n_bn)])
    buffers = ([buf[f"bn.{i}.running_mean"] for i in range(n_bn)] + [None],
               [buf[f"bn.{i}.running_var"] for i in range(n_bn)] + [None],
               [buf[f"bn.{i}.num_batches_tracked"] for i in range(n_bn)] + [None])
    xg = x.to(dev()).requires_grad_(True)
    y = _MeshNetFunction.apply(xg, hier, True, buffers, n_layers, *[p[k] for k in names])
    loss = (y - tgt.to(dev())).abs().mean()
    loss.backward()
    torch.cuda.synchronize()
    assert hier.kernel_status(0) == 0
    return (y.detach().cpu(), float(loss), {k: p[k].grad.cpu() for k in names},
            {k: v.cpu() for k, v in buf.items()}, xg.grad.cpu())


def oracle_train_step(mo, sd, levels, plan, x, tgt):
    """The same step in float64 autograd over oracle.meshnet_oracle.forward (the fp32 Laplacians cast up)."""
    laps = [m.to(torch.float64) for m in mo.laplacians_to_torch(levels, drop_second_coarsest=False)]
    s = {k: (v.double().clone().requires_grad_(True) if v.is_floating_point() and "running" not in k
             else (v.double().clone() if v.is_floating_point() else v.clone())) for k, v in sd.items()}
    xo = x.double().clone().requires_grad_(True)
    yo = mo.forward(s, laps, xo, training=True, plan=plan)
    lo = (yo - tgt.double()).abs().mean()
    lo.backward()
    return yo.detach(), float(lo.detach()), {k: v.grad for k, v in s.items() if v.requires_grad}, s, xo.grad


def per_mesh_rel_err(y, ref):
    d = (y.double() - ref.double()).abs().flatten(1).max(dim=1).values
    return float((d / ref.double().abs().flatten(1).max(dim=1).values.clamp_min(1e-30)).max())


def grad_err(got, ref, scale=0.0):
    """max |got - ref| / max(max |ref|, scale) (the strict gradient parity of test_gpu_parity.grad_close)."""
    got, ref = got.double(), ref.double()
    return float((got - ref).abs().max()) / max(float(ref.abs().max()), scale, 1e-30)


def smpl_small_levels(*sizes):
    return [level_of("smpl_small", V) for V in sizes]


# levels {128, 64, joint 17}: block 1 ends in a residual + unpool, block 2 in an identity residual, block 3 is the head
NET_PLAN = [(5, 32, 64), (64, 128), (128, 128), (128, 64, 3)]


@pytest.mark.parametrize("precision", PRECISIONS)
def test_network_bias_shift_invariance(precision):
    """Train mode: a constant c added to every conv bias in front of a BatchNorm cancels in the normalisation.  y, the
    loss and every gradient except those biases' equal the c = 0 run, running_var is unchanged and running_mean moves
    by exactly momentum * c."""
    levels = smpl_small_levels(128, 64, 17)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 17, 5, generator=g)
    tgt = torch.randn(2, 128, 3, generator=g)
    hier, sd0, n_layers, _ = small_net(levels, NET_PLAN, precision, seed=11)
    y0, l0, g0, b0, dx0 = net_train_step(hier, sd0, n_layers, x, tgt)
    for c in (10.0, 100.0, 1000.0):
        _, sd, _, _ = small_net(levels, NET_PLAN, precision, seed=11, bias_shift=c)
        y, l, gr, bf, dx = net_train_step(hier, sd, n_layers, x, tgt)
        # (PyTorch's own fp32 BatchNorm on this net: ~7e-6 at c = 1000, from z's fp32 storage)
        assert per_mesh_rel_err(y, y0) < 2e-5, (c, per_mesh_rel_err(y, y0))
        assert abs(l - l0) <= 2e-5 * abs(l0), (c, l, l0)
        assert grad_err(dx, dx0) < 1e-3, (c, "dx", grad_err(dx, dx0))
        scale = max(float(v.abs().max()) for v in g0.values())
        for k in g0:
            if k.startswith("cl.") and k.endswith(".bias") and int(k.split(".")[1]) != n_layers - 1:
                assert torch.count_nonzero(gr[k]) == 0, k          # zeroed by the backward: exactly 0
                continue
            assert grad_err(gr[k], g0[k], 1e-3 * scale) < 1e-3, (c, k, grad_err(gr[k], g0[k], 1e-3 * scale))
        for k in b0:
            if k.endswith("running_var"):
                assert torch.allclose(bf[k], b0[k], rtol=1e-5, atol=1e-6), (c, k)
            elif k.endswith("running_mean"):
                d = (bf[k].double() - b0[k].double() - 0.1 * c).abs().max()
                assert d <= 1e-5 + 8 * R.U32 * c, (c, k, float(d))
            else:
                assert int(bf[k]) == int(b0[k]) == 1, k


# block 0 on the 17-row joint level at B = 1 with BN widths = 2 (mod 4): k_affine_act and k_bn_bwd_apply, and 1/n of 17
NET_PLAN_SCALAR = [(5, 18, 34), (34, 64), (64, 64), (64, 32, 3)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("plan_name", ["NET_PLAN", "NET_PLAN_SCALAR"])
def test_network_train_step_matches_float64(plan_name, precision):
    """A whole train step (forward, L1 loss, backward) against float64 autograd over the oracle with the same plan,
    under the strict open-ReLU tolerances: y 1e-4 of each mesh's largest entry, every gradient 1e-3 of its tensor's
    largest entry (conv biases in front of a BN, mathematically zero, on the global scale), running statistics."""
    plan = NET_PLAN if plan_name == "NET_PLAN" else NET_PLAN_SCALAR
    levels = smpl_small_levels(128, 64, 17)
    g = torch.Generator().manual_seed(4)
    B = 1 if plan_name == "NET_PLAN_SCALAR" else 3
    x = torch.randn(B, 17, 5, generator=g)
    tgt = torch.randn(B, 128, 3, generator=g)
    hier, sd, n_layers, mo = small_net(levels, plan, precision, seed=12)
    y, l, gr, bf, dx = net_train_step(hier, sd, n_layers, x, tgt)
    yo, lo, go, so, dxo = oracle_train_step(mo, sd, levels, plan, x, tgt)
    assert per_mesh_rel_err(y, yo) < 1e-4, per_mesh_rel_err(y, yo)
    assert abs(l - lo) < 1e-5 * max(1.0, abs(lo))
    assert grad_err(dx, dxo) < 1e-3, ("dx", grad_err(dx, dxo))
    scale = max(float(v.abs().max()) for v in go.values())
    for k in go:
        zero_bias = k.startswith("cl.") and k.endswith(".bias") and int(k.split(".")[1]) != n_layers - 1
        if zero_bias:
            assert torch.count_nonzero(gr[k]) == 0, k
        e = grad_err(gr[k], go[k], 1e-3 * scale if zero_bias else 0.0)
        assert e < 1e-3, (k, e)
    for k in bf:
        if "num_batches" in k:
            assert int(bf[k]) == 1
        else:
            assert torch.allclose(bf[k].double(), so[k], rtol=1e-5, atol=1e-6), k
