"""Per-BatchNorm modes without a GPU: the float64 restatement of torch's rules (bn_modes_ref) against nn.BatchNorm1d,
the option records Pose2Mesh and LinearModel build from their submodules, the ctypes layout of p2m_bn_opts_t, and the
states the native kernels refuse."""
import ctypes as C
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

import bn_modes_ref as R

F_ = 6
MODES = {  # name: (module setup, number of steps)
    "train": (lambda bn: bn.train(), 1),
    "eval": (lambda bn: bn.eval(), 1),
    "frozen_in_train": (lambda bn: bn.eval(), 1),
    "no_stats_train": (lambda bn: bn.train(), 1),
    "no_stats_eval": (lambda bn: bn.eval(), 1),
    "momentum_none": (lambda bn: bn.train(), 3),
    "eps_momentum": (lambda bn: bn.train(), 2),
    "eps_momentum_eval": (lambda bn: bn.eval(), 1),
}


def _bn(name):
    kw = {}
    if name.startswith("no_stats"):
        kw["track_running_stats"] = False
    if name == "momentum_none":
        kw["momentum"] = None
    if name.startswith("eps_momentum"):
        kw.update(momentum=0.01, eps=1e-3)
    bn = nn.BatchNorm1d(F_, **kw).double()
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(F_, generator=g, dtype=torch.float64) + 0.5)
        bn.bias.copy_(torch.randn(F_, generator=g, dtype=torch.float64))
        if bn.running_mean is not None:
            bn.running_mean.copy_(torch.randn(F_, generator=g, dtype=torch.float64))
            bn.running_var.copy_(torch.rand(F_, generator=g, dtype=torch.float64) + 0.5)
    return bn


@pytest.mark.parametrize("name", sorted(MODES))
def test_restatement_matches_batchnorm1d(name):
    """The rules as bn_modes_ref states them reproduce nn.BatchNorm1d in float64: outputs, running statistics,
    num_batches_tracked, and the gradients of the input, gamma, beta and the bias of a Linear in front."""
    setup, steps = MODES[name]
    bn = _bn(name)
    setup(bn)
    stats, cumulative, momentum, eps = R.expected_opts(bn)
    state = {"rm": None if bn.running_mean is None else bn.running_mean.clone(),
             "rv": None if bn.running_var is None else bn.running_var.clone(),
             "nbt": None if bn.num_batches_tracked is None else bn.num_batches_tracked.clone()}
    gamma = bn.weight.detach().clone().requires_grad_(True)
    beta = bn.bias.detach().clone().requires_grad_(True)
    g = torch.Generator().manual_seed(5)
    for step in range(steps):
        x = torch.randn(9, F_, generator=g, dtype=torch.float64) * 2 + 1
        bias = torch.randn(F_, generator=g, dtype=torch.float64)
        w = torch.randn(9, F_, generator=g, dtype=torch.float64)
        x1, b1 = x.clone().requires_grad_(True), bias.clone().requires_grad_(True)
        bn.zero_grad()
        y1 = bn(x1 + b1)
        (y1 * w).sum().backward()
        x2, b2 = x.clone().requires_grad_(True), bias.clone().requires_grad_(True)
        gamma.grad = beta.grad = None
        y2 = R.batch_norm(x2 + b2, gamma, beta, state, stats, cumulative, momentum, eps)
        (y2 * w).sum().backward()
        torch.testing.assert_close(y2, y1, rtol=1e-12, atol=1e-12)
        for a, b in ((x2.grad, x1.grad), (b2.grad, b1.grad), (gamma.grad, bn.weight.grad), (beta.grad, bn.bias.grad)):
            torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
        if stats == R.P2M_BN_RUNNING:   # frozen: the bias in front gets sum_rows g_z, not 0
            assert b1.grad.abs().max() > 1e-3
        else:
            assert b1.grad.abs().max() < 1e-9
        if bn.running_mean is not None:
            torch.testing.assert_close(state["rm"], bn.running_mean, rtol=1e-12, atol=1e-12)
            torch.testing.assert_close(state["rv"], bn.running_var, rtol=1e-12, atol=1e-12)
            assert int(state["nbt"]) == int(bn.num_batches_tracked)
    if name == "momentum_none":
        assert int(bn.num_batches_tracked) == 3


def _opts_tuple(o):
    return o.stats, o.cumulative, o.momentum, o.eps


def _small_meshnet():
    from helpers import graph_from_fixture
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    return Pose2Mesh(5, 3, graph_from_fixture("mano_like")[0])


def test_meshnet_option_arrays_follow_the_submodules():
    model = _small_meshnet()
    n = len(model.cl)
    bns = [m for m in model.bn if m is not None]
    assert len(bns) == n - 1
    model.train()
    bns[0].eval()
    bns[1].momentum = None
    bns[2].eps, bns[2].momentum = 1e-3, 0.01
    bns[3].track_running_stats = False
    model.bn[4] = nn.BatchNorm1d(bns[4].num_features, track_running_stats=False)
    model.bn[4].eval()
    for training in (True, False):
        model.train(training)
        if training:
            bns[0].eval()
        opts = model._bn_opts()
        assert len(opts) == n
        for i in range(n - 1):
            assert _opts_tuple(opts[i]) == pytest.approx(R.expected_opts(model.bn[i])), (training, i)
    model.train()
    bns[0].eval()
    opts = model._bn_opts()
    assert opts[0].stats == R.P2M_BN_RUNNING and opts[1].stats == R.P2M_BN_BATCH_UPDATE and opts[1].cumulative == 1
    assert opts[3].stats == R.P2M_BN_BATCH and opts[4].stats == R.P2M_BN_BATCH
    assert (opts[2].eps, opts[2].momentum) == (1e-3, 0.01)


def test_posenet_option_arrays_follow_the_submodules():
    from pose2mesh_release_b200.posenet import LinearModel

    net = LinearModel(4, 32, 3, 0.5)
    net.train()
    net.linear_stages[0].batch_norm2.eval()
    net.linear_stages[1].dropout.eval()
    net.linear_stages[2].dropout.p = 0.7
    net.linear_stages[2].batch_norm1.momentum = None
    bn, p = net._native_modes()
    assert len(bn) == 6 and len(p) == 3
    for s, st in enumerate(net.linear_stages):
        assert _opts_tuple(bn[2 * s]) == pytest.approx(R.expected_opts(st.batch_norm1))
        assert _opts_tuple(bn[2 * s + 1]) == pytest.approx(R.expected_opts(st.batch_norm2))
    assert list(p) == pytest.approx([0.5, 0.0, 0.7])
    net.eval()
    bn, p = net._native_modes()
    assert all(o.stats == R.P2M_BN_RUNNING for o in bn) and list(p) == [0.0, 0.0, 0.0]


def test_ctypes_record_matches_header():
    from pose2mesh_release_b200 import _lib

    hdr = open(__file__.replace("tests/test_bn_modes_cpu.py", "include/p2m_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} p2m_bn_opts_t;", hdr).group(1)
    fields = re.findall(r"^\s*(int32_t|double|float)\s+(\w+);", body, re.M)
    ctype = {"int32_t": C.c_int32, "double": C.c_double, "float": C.c_float}
    assert [(n, ctype[t]) for t, n in fields] == list(_lib.BnOpts._fields_)
    assert C.sizeof(_lib.BnOpts) == 24
    for name in ("P2M_BN_BATCH_UPDATE", "P2M_BN_BATCH", "P2M_BN_RUNNING"):
        assert int(re.search(rf"#define {name} (\d+)", hdr).group(1)) == getattr(_lib, name) == getattr(R, name)


def test_unsupported_states_raise_value_error():
    from pose2mesh_release_b200.posenet import LinearModel

    model = _small_meshnet()
    model.bn[0] = nn.BatchNorm1d(model.bn[0].num_features, affine=False)
    with pytest.raises(ValueError, match="affine"):
        model(torch.zeros(2, 21, 5))
    model = _small_meshnet()
    model.bn[1] = nn.LayerNorm(model.bn[1].num_features)
    with pytest.raises(ValueError, match="BatchNorm1d"):
        model(torch.zeros(2, 21, 5))

    net = LinearModel(4, 32, 2, 0.5)
    net.linear_stages[1].batch_norm2 = nn.BatchNorm1d(32, affine=False)
    with pytest.raises(ValueError, match="affine"):
        net.forward_train_native(torch.zeros(2, 8))
    net = LinearModel(4, 32, 2, 0.5)
    net.linear_stages[0].dropout = nn.Identity()
    with pytest.raises(ValueError, match="Dropout"):
        net.forward_native(torch.zeros(2, 8))
    net = LinearModel(4, 32, 2, 0.5)
    net.linear_stages[0].batch_norm1 = nn.Identity()
    with pytest.raises(ValueError, match="BatchNorm1d"):
        net.forward_train_native(torch.zeros(2, 8))
