"""Per-BatchNorm modes on the GPU: Pose2Mesh and LinearModel honour each BatchNorm's training flag,
track_running_stats, momentum (None: cumulative) and eps, and each PoseNet stage's Dropout, checked against float64
(bn_modes_ref) with every parameter, gradient and buffer.  Default options stay bitwise what the calls without options
compute."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import bn_modes_ref as R
import posenet_train_ref as T
from helpers import graph_from_fixture

pytestmark = pytest.mark.gpu

# outputs: max |err| <= TOL * max |ref| (fp32 storage against float64); gradients: bn_modes_ref.grad_ok, the parity
# the project holds its gradients to
TOL = {"y": 2e-5}


def dev():
    return torch.device("cuda:0")


def _meshnet(name, precision, seed=11):
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats = graph_from_fixture(name)[0]
    torch.manual_seed(seed)
    model = Pose2Mesh(5, 3, [m.copy() for m in mats])
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for i, m in enumerate(model.bn):
            model.cl[i].bias.copy_(torch.randn(model.cl[i].bias.shape, generator=g) * 0.1)
            if m is None:
                continue
            m.weight.copy_(torch.rand(m.num_features, generator=g) + 0.5)
            m.bias.copy_(torch.full((m.num_features,), 6.0))  # open ReLUs: no pre-activation near zero
    model.set_precision(precision)
    model = model.to(dev())
    # running statistics of the inputs the tests use (one batch-statistics pass with momentum 1): frozen BatchNorms
    # then normalise like batch statistics do, and the ReLUs stay open
    for m in model.bn:
        if m is not None:
            m.momentum = 1.0
    with torch.no_grad():
        model.train()(_inputs(model, 4)[0].to(dev()))
    for m in model.bn:
        if m is not None:
            m.momentum = 0.1
            m.num_batches_tracked.zero_()
    return model, R.laplacians64(mats)


def _inputs(model, B, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, model.graph_L[-1].shape[0], 5, generator=g) * 0.5
    tgt = torch.randn(B, model.num_vertices, 3, generator=g)
    return x, tgt


def _buffers(model):
    return {k: v.detach().clone() for k, v in model.named_buffers()}


def _native_step(model, x, tgt):
    """Forward + L1 loss + backward: (y, dx, grads by name)."""
    model.zero_grad(set_to_none=True)
    xg = x.to(dev()).requires_grad_(True)
    y = model(xg)
    (y - tgt.to(dev())).abs().mean().backward()
    torch.cuda.synchronize()
    return y.detach(), xg.grad, {k: p.grad.detach().clone() for k, p in model.named_parameters()}


def _ref_step(m, laps, x, tgt):
    """The same step in float64 on m, a module64 copy of the module taken before the native step: (y, dx, grads, m)."""
    xg = x.double().requires_grad_(True)
    y = R.meshnet_forward(m, laps, xg)
    (y - tgt.double()).abs().mean().backward()
    return y.detach(), xg.grad, {k: p.grad for k, p in m.named_parameters()}, m


def _check_step(model, laps, x, tgt):
    before = _buffers(model)
    m64 = R.module64(model)
    y, dx, grads = _native_step(model, x, tgt)
    y64, dx64, g64, m64 = _ref_step(m64, laps, x, tgt)
    assert R.close(y, y64, TOL["y"]) <= 1
    assert R.grad_ok(dx, dx64)[0], R.grad_ok(dx, dx64)
    for k, g in grads.items():
        i = int(k.split(".")[1]) if k.startswith("cl.") and k.endswith(".bias") else -1
        if 0 <= i < len(model.cl) - 1 and model.bn[i].training:
            # in front of a batch-statistics BatchNorm the bias gradient is mathematically zero: written as exactly 0
            assert not g.any(), k
            continue
        assert R.grad_ok(g, g64[k])[0], (k, R.grad_ok(g, g64[k]))
    after = dict(model.named_buffers())
    for k, v in m64.named_buffers():
        if k.endswith("num_batches_tracked"):
            assert int(after[k]) == int(v), k
        else:
            assert R.close(after[k], v, 1e-5) <= 1, k
    return before, y, grads


@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["smpl_small", "mano_like"])
@pytest.mark.parametrize("training", [True, False])
def test_default_options_bitwise_equal_to_calls_without_options(name, precision, training):
    """The module's default option arrays and a NULL array (the calls without options) give bitwise the same y, dx,
    running statistics and num_batches_tracked, and the same gradients up to the last bits by which two runs of one
    build differ (the CUDA-core dW accumulates with atomics)."""
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    model, _ = _meshnet(name, precision)
    model.train(training)
    x, tgt = _inputs(model, 4)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    outs = []
    for explicit in (True, False):
        model.load_state_dict(sd)
        model.zero_grad(set_to_none=True)
        xg = x.to(dev()).requires_grad_(training)
        n, params = model._flat_params()
        buffers = model._bn_buffers() + ((model._bn_opts(),) if explicit else ())
        with torch.set_grad_enabled(training):
            y = _MeshNetFunction.apply(xg, model._hier, training, buffers, n, *params)
            if training:
                (y - tgt.to(dev())).abs().mean().backward()
        torch.cuda.synchronize()
        grads = [p.grad.clone() for p in params] if training else []
        outs.append((y.detach().clone(), xg.grad, grads, {k: v.clone() for k, v in model.named_buffers()}))
    (y0, dx0, g0, b0), (y1, dx1, g1, b1) = outs
    assert torch.equal(y0, y1)
    if training:
        assert torch.equal(dx0, dx1) and all(R.close(a, b, 1e-6) <= 1 for a, b in zip(g0, g1))
    assert all(torch.equal(b0[k], b1[k]) for k in b0)


@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["smpl_small", "mano_like"])
def test_frozen_batchnorms_in_train_mode(name, precision):
    """Every BatchNorm in eval mode inside a train-mode MeshNet: y, dx and every gradient (the conv biases in front of
    the BatchNorms now nonzero) against float64; running statistics and num_batches_tracked bitwise untouched; y equal
    to the eval forward's within both bounds."""
    model, laps = _meshnet(name, precision)
    model.train()
    for m in model.bn:
        if m is not None:
            m.eval()
    x, tgt = _inputs(model, 4)
    before, y, grads = _check_step(model, laps, x, tgt)
    for k, v in model.named_buffers():
        assert torch.equal(v, before[k]), k
    assert all(float(grads[f"cl.{i}.bias"].abs().max()) > 0 for i in range(len(model.cl) - 1))
    model.eval()
    with torch.no_grad():
        ye = model(x.to(dev()))
    y64 = R.meshnet_forward(R.module64(model), laps, x.double())
    assert R.close(ye, y64, TOL["y"]) <= 1 and R.close(y, ye, 2 * TOL["y"]) <= 1


@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
def test_mixed_layers(precision):
    """Frozen / batch statistics with update / batch statistics without update, alternating over the layers."""
    model, laps = _meshnet("mano_like", precision)
    model.train()
    for i, m in enumerate(model.bn):
        if m is None:
            continue
        if i % 3 == 0:
            m.eval()
        elif i % 3 == 2:
            m.track_running_stats = False
    x, tgt = _inputs(model, 3)
    before, _, _ = _check_step(model, laps, x, tgt)
    for i, m in enumerate(model.bn):
        if m is not None and i % 3 != 1:
            assert torch.equal(m.running_mean, before[f"bn.{i}.running_mean"])
            assert int(m.num_batches_tracked) == 0


def test_momentum_none_eps_and_stats_less_eval():
    """momentum=None over three steps gives the cumulative averages and num_batches_tracked == 3; momentum=0.01 and
    eps=1e-3 in train and eval; an eval forward whose BatchNorm has no running buffers uses batch statistics."""
    model, laps = _meshnet("mano_like", "fp16x3")
    model.train()
    for m in model.bn:
        if m is not None:
            m.momentum = None
    for step in range(3):
        x, tgt = _inputs(model, 3, seed=10 + step)
        _check_step(model, laps, x, tgt)
    assert all(int(m.num_batches_tracked) == 3 for m in model.bn if m is not None)

    model, laps = _meshnet("smpl_small", "fp32")
    for m in model.bn:
        if m is not None:
            m.momentum, m.eps = 0.01, 1e-3
    model.train()
    x, tgt = _inputs(model, 3)
    _check_step(model, laps, x, tgt)
    model.eval()
    model.bn[1] = nn.BatchNorm1d(model.bn[1].num_features, track_running_stats=False).to(dev()).eval()
    with torch.no_grad():
        y = model(x.to(dev()))
    y64 = R.meshnet_forward(R.module64(model), laps, x.double())
    assert R.close(y, y64, TOL["y"]) <= 1


# ---------------------------------------------------------------------------------------------------------- PoseNet
def _posenet(J, H, S, p, seed=7):
    from pose2mesh_release_b200 import posenet

    torch.manual_seed(seed)
    net = posenet.LinearModel(J, H, S, p)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, t in net.state_dict().items():
            if "batch_norm" in name and t.dtype.is_floating_point:
                t.copy_(torch.rand(t.shape, generator=g) + 0.5 if name.endswith(("weight", "running_var"))
                        else torch.randn(t.shape, generator=g) * 0.3)
            if "batch_norm" in name and name.endswith("bias"):
                t.add_(2.0)  # open ReLUs: a pre-activation within rounding of zero would flip against float64
    return net.to(dev()).train()


def _posenet_check(net, B, seed_vals=(1234, 99)):
    J, H = net.num_joint, net.linear_size
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 2 * J, generator=g)
    d_out = torch.randn(B, 3 * J, generator=g)
    seed = torch.tensor(seed_vals, dtype=torch.int64, device=dev())
    _, p = net._native_modes()
    masks = []
    for s in range(net.num_stage):
        for d in (2 * s, 2 * s + 1):
            masks.append(torch.as_tensor(T.dropout_multiplier(np.array(seed_vals), d, B * H, p[s])).reshape(B, H))
    m64 = R.module64(net)
    before = {k: v.clone() for k, v in net.named_buffers()}
    xg = x.to(dev()).requires_grad_(True)
    net.zero_grad(set_to_none=True)
    out = net.forward_train_native(xg, seed=seed)
    out.backward(d_out.to(dev()))
    x64 = x.double().requires_grad_(True)
    out64 = R.posenet_forward(m64, x64, masks)
    out64.backward(d_out.double())
    assert R.close(out, out64, 1e-4) <= 1
    assert R.grad_ok(xg.grad, x64.grad)[0], R.grad_ok(xg.grad, x64.grad)
    p64 = dict(m64.named_parameters())
    bn_after = {f"linear_stages.{s}.w1.bias": st.batch_norm2 for s, st in enumerate(net.linear_stages)}
    for k, prm in net.named_parameters():
        if prm.grad is None:
            continue
        if k in bn_after and bn_after[k].training:   # mathematically zero: column sums of rounding noise
            assert float(prm.grad.abs().max()) <= 1e-3 * float(p64[k.replace("bias", "weight")].grad.abs().max()), k
            continue
        assert R.grad_ok(prm.grad, p64[k].grad)[0], (k, R.grad_ok(prm.grad, p64[k].grad))
    b64 = dict(m64.named_buffers())
    for k, v in net.named_buffers():
        if k.startswith("linear_stages"):
            assert R.close(v, b64[k], 1e-5) <= 1, k
    return before


@pytest.mark.parametrize("H", [1024, 96])
def test_posenet_frozen_dropout_eval_and_per_stage_p(H):
    """Frozen BatchNorms, Dropout in eval mode, and per-stage p (0.2, 0.7), against float64 with the seed's masks."""
    net = _posenet(17, H, 2, 0.5)
    for st in net.linear_stages:
        st.batch_norm1.eval()
        st.batch_norm2.eval()
        st.dropout.eval()
    before = _posenet_check(net, 48)
    for k, v in net.named_buffers():
        assert torch.equal(v, before[k]), k
    net = _posenet(17, H, 2, 0.5)
    net.linear_stages[0].dropout.p, net.linear_stages[1].dropout.p = 0.2, 0.7
    net.linear_stages[1].batch_norm1.eval()
    _posenet_check(net, 48)


def test_posenet_default_p_keeps_masks_and_batch_of_one():
    """A default p gives bitwise the output of the call without options; B = 1 runs with every BatchNorm frozen and is
    refused while one uses batch statistics."""
    from pose2mesh_release_b200 import _lib

    import ctypes as C

    net = _posenet(17, 1024, 2, 0.5)
    x = torch.randn(32, 34, device=dev())
    seed = torch.tensor([5, 6], dtype=torch.int64, device=dev())
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        out = net.forward_train_native(x, seed=seed)
    net.load_state_dict(sd)
    lib = _lib.load()
    dims = (32, 17, 1024, 2)
    saved = torch.empty(lib.p2m_posenet_train_saved_bytes(*dims), dtype=torch.uint8, device=dev())
    ws = torch.empty(lib.p2m_posenet_train_workspace_bytes(*dims), dtype=torch.uint8, device=dev())
    legacy = torch.empty_like(out)
    native, extra = net._native_params(), net._native_train_extra()
    _lib.call("p2m_posenet_train_forward", dev(), C.byref(native), C.byref(extra), x, 32, 0.5, seed, legacy, None,
              saved, saved.numel(), ws, ws.numel())
    torch.cuda.synchronize()
    assert torch.equal(out, legacy)

    for st in net.linear_stages:
        st.batch_norm1.eval()
        st.batch_norm2.eval()
    _posenet_check(net, 1)
    net.linear_stages[1].batch_norm2.train()
    with pytest.raises(ValueError, match="more than 1 value"):
        net.forward_train_native(torch.randn(1, 34, device=dev()))


def test_flat_pose2mesh_frozen_data_parallel_step():
    """FlatPose2Mesh in train() with every BatchNorm frozen: one DataParallelStep step whose gradients match float64."""
    from pose2mesh_release_b200.dist import DataParallelStep
    from pose2mesh_release_b200.pose2mesh_net import FlatPose2Mesh

    mats = graph_from_fixture("smpl_small")[0]
    torch.manual_seed(4)
    model = FlatPose2Mesh(17, [m.copy() for m in mats]).to(dev()).train()
    for m in model.modules():
        if isinstance(m, nn.BatchNorm1d):
            m.eval()
    step = DataParallelStep(model)
    g = torch.Generator().manual_seed(2)
    pose2d = torch.randn(4, 17, 2, generator=g)
    tgt = torch.randn(4, model.pose2mesh.num_vertices, 3, generator=g)
    for st in model.pose_lifter.linear_stages:   # the float64 side cannot draw the native masks
        st.dropout.eval()
    m64 = R.module64(model)
    step.zero_grad()
    mesh, pose3d = model(pose2d.to(dev()))
    ((mesh - tgt.to(dev())).abs().mean() + pose3d.abs().mean()).backward()
    step.reduce_gradients()
    torch.cuda.synchronize()
    p2 = pose2d.double().reshape(4, -1)
    pose3d64 = R.posenet_forward(m64.pose_lifter, p2, [torch.ones(4, 4096, dtype=torch.float64)] * 4).reshape(4, 17, 3)
    comb = torch.cat((pose2d.double(), pose3d64.detach() / 1000), dim=2)
    mesh64 = R.meshnet_forward(m64.pose2mesh, R.laplacians64(mats), comb)
    ((mesh64 - tgt.double()).abs().mean() + pose3d64.abs().mean()).backward()
    p64 = dict(m64.named_parameters())
    for k, p in model.named_parameters():
        if p64[k].grad is not None:
            assert R.grad_ok(p.grad, p64[k].grad)[0], (k, R.grad_ok(p.grad, p64[k].grad))


def test_frozen_step_replays_in_a_cuda_graph():
    """A frozen-BatchNorm training step with momentum=None in the batch-statistics layers, captured in a CUDA graph,
    replays bitwise the eager step's y, running statistics and num_batches_tracked, and its gradients up to the last
    bits by which two eager runs differ (the dW accumulations use atomics)."""
    model, _ = _meshnet("mano_like", "fp16x3")
    model.train()
    for i, m in enumerate(model.bn):
        if m is not None:
            m.momentum = None
            if i % 2 == 0:
                m.eval()
    x, tgt = _inputs(model, 4)
    xs, ts = x.to(dev()), tgt.to(dev())
    sd = {k: v.clone() for k, v in model.state_dict().items()}

    def step():
        y = model(xs)
        (y - ts).abs().mean().backward()
        return y

    model.zero_grad(set_to_none=False)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):  # warm-up
            for p in model.parameters():
                p.grad = torch.zeros_like(p) if p.grad is None else p.grad.zero_()
            step()
    torch.cuda.current_stream().wait_stream(s)
    model.load_state_dict(sd)
    for p in model.parameters():
        p.grad.zero_()
    eager_y = step().detach().clone()
    eager = ([p.grad.clone() for p in model.parameters()], {k: v.clone() for k, v in model.named_buffers()})
    model.load_state_dict(sd)
    graph = torch.cuda.CUDAGraph()
    for p in model.parameters():
        p.grad.zero_()
    with torch.cuda.graph(graph):
        y_g = step()
    model.load_state_dict(sd)
    for p in model.parameters():
        p.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y_g, eager_y)
    assert all(R.close(p.grad, g, 1e-6) <= 1 for p, g in zip(model.parameters(), eager[0]))
    assert all(torch.equal(v, eager[1][k]) for k, v in model.named_buffers())
