"""PoseNet's train step layer by layer against float64 (tests/posenet_layers_ref.py): every operation of the native
training forward and backward from the fp32 tensors the device produced (`saved`, and the backward's intermediates
from p2m_debug_posenet_backward_capture), with the device's own ReLU masks, each held element-wise to its own bound
with no quantile and no slack.  The grid covers every branch posenet.cu takes: tensor cores or fp32 CUDA cores, the
padded dW (K = B rounded up to 32), the output layer on either path, several statistics blocks, F % 4 != 0, no stages,
every dropout mode, every BatchNorm mode, channels far from zero and operands far from 1.  Capturing changes no result.

The worst ratio per quantity class, the near-zero pre-activation count and the wall time are written to the JSON file
named by P2M_POSENET_FP64_REPORT (if set)."""
import json
import os
import time

import numpy as np
import pytest
import torch

import fp64_ref as R
import posenet_layers_ref as PL

pytestmark = pytest.mark.gpu

SEED = [0x5DEECE66D1234567, -987654321]
_WORST = {}
_NEAR_ZERO = {"grid": 0}        # per case, and summed over the natural grid (the constructed case not included)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    out = os.environ.get("P2M_POSENET_FP64_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump({"wall_s": time.time() - t0, "worst_ratio": _WORST, "near_zero": _NEAR_ZERO}, f, indent=1)


def dev():
    return torch.device("cuda:0")


def _net(J, H, S, p, init="random", seed=7):
    """LinearModel in train(); p: one dropout p for all stages or one per stage.  init='random' gives the BatchNorms
    random affine parameters and running statistics, 'default' keeps torch's (gamma 1, beta 0, mean 0, var 1)."""
    from pose2mesh_release_b200 import posenet

    torch.manual_seed(seed)
    ps = list(p) if isinstance(p, (list, tuple)) else [p] * S
    net = posenet.LinearModel(J, H, S, ps[0] if ps else 0.5)
    for st, q in zip(net.linear_stages, ps):
        st.dropout.p = q
    if init == "random":
        g = torch.Generator().manual_seed(seed + 1)
        with torch.no_grad():
            for name, t in net.state_dict().items():
                if "batch_norm" in name and t.dtype.is_floating_point:
                    t.copy_(torch.rand(t.shape, generator=g) + 0.5 if name.endswith(("weight", "running_var"))
                            else torch.randn(t.shape, generator=g) * 0.3)
    return net.to(dev()).train()


def _bns(net):
    return [bn for st in net.linear_stages for bn in (st.batch_norm1, st.batch_norm2)]


def _state(net):
    return {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}


def _run(net, x, d_out, capture=None):
    from pose2mesh_release_b200 import posenet

    seed = torch.tensor(SEED, dtype=torch.int64, device=dev())
    fields = posenet.CAPTURE_FIELDS if capture == "all" else capture
    with torch.no_grad():
        res = posenet.debug_train_step_capture(net, x.to(dev()), seed, d_out.to(dev()), fields)
    torch.cuda.synchronize()
    return res


def _numpy(res):
    out = {}
    for k, v in res.items():
        if isinstance(v, torch.Tensor):
            out[k] = v.cpu().numpy()
        elif isinstance(v, list):
            out[k] = [t.cpu().numpy() for t in v]
        else:
            out[k] = v
    return out


def _modes(net):
    return [dict(stats=o.stats, cumulative=o.cumulative, momentum=o.momentum, eps=o.eps)
            for o in net._native_modes()[0]]


def check_layers(net, x, d_out, tag, constructed=False):
    """One captured train step of `net` from its current state, every layer within its float64 bound."""
    from pose2mesh_release_b200 import _lib

    J, H, S, B = net.num_joint, net.linear_size, net.num_stage, x.shape[0]
    sd, modes, p_stage = _state(net), _modes(net), list(net._native_modes()[1])
    res = _numpy(_run(net, x, d_out, "all"))
    for k, v in res.items():
        vs = v if isinstance(v, list) else [v]
        if k != "scale" or H % 64 == 0:              # the fp32 path leaves the scales unwritten (NaN)
            assert all(np.isfinite(t).all() for t in vs if t.dtype.kind == "f"), (tag, k)
    chk, near = PL.check_step(sd, _state(net), x.numpy(), d_out.numpy(), SEED, modes, p_stage, res, J, H, S,
                              _lib.load().p2m_posenet_train_saved_bytes(B, J, H, S))
    assert not chk.bitwise, (tag, chk.bitwise)
    for cls, r in chk.ratio.items():
        if r > _WORST.get(cls, [0.0])[0]:
            _WORST[cls] = [r, tag]
    _NEAR_ZERO[tag] = near
    if not constructed:
        _NEAR_ZERO["grid"] += near
    worst = max(chk.ratio, key=chk.ratio.get)
    assert chk.ratio[worst] <= 1.0, (tag, worst, chk.ratio[worst], {k: round(v, 3) for k, v in chk.ratio.items()})
    return chk, near


def _inputs(B, J, seed, gscale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 2 * J, generator=g), torch.randn(B, 3 * J, generator=g) * gscale


SHAPES = [  # H, B, J, S, p, BatchNorm init
    (4096, 256, 17, 2, 0.5, "default"),    # the reference's PoseNet: tensor cores everywhere, also the output
    (1024, 50, 21, 2, 0.5, "random"),      # dW's K = 50 padded to Bp = 64; 3J = 63 on the tensor cores
    (128, 600, 17, 1, 0.5, "random"),      # two STAT_ROWS = 512 blocks in every column reduction; a ragged M tile
    (128, 65, 22, 1, 0.5, "random"),       # 3J = 66: the fp32 output GEMM; Bp = 96
    (96, 50, 17, 2, 0.5, "random"),        # H % 64 != 0: fp32 CUDA-core GEMMs and the transposed gradient
    (90, 33, 5, 1, 0.5, "random"),         # F % 4 != 0: scalar k_bn_bwd_apply, dropout groups straddling rows
    (128, 2, 17, 1, 0.5, "random"),        # the smallest batch
    (128, 64, 17, 0, 0.5, "random"),       # no stages
    (256, 128, 17, 3, (0.0, 0.3, 1.0), "random"),   # dropout modes 0 / 1 / 2
]


@pytest.mark.parametrize("H,B,J,S,p,init", SHAPES, ids=lambda v: str(v))
def test_train_step_layers_within_float64_bound(H, B, J, S, p, init):
    net = _net(J, H, S, p, init)
    x, d_out = _inputs(B, J, B + H)
    check_layers(net, x, d_out, f"H={H} B={B} J={J} S={S} p={p} {init}")


BN_MODES = {
    "all_frozen": lambda bns: [bn.eval() for bn in bns],
    "bn1_frozen_bn2_batch": lambda bns: [(bn.eval() if i % 2 == 0 else setattr(bn, "track_running_stats", False))
                                         for i, bn in enumerate(bns)],
    "cumulative_nbt5": lambda bns: [(setattr(bn, "momentum", None), bn.num_batches_tracked.fill_(5)) for bn in bns],
    "eps_1e-3_momentum_0.01": lambda bns: [(setattr(bn, "eps", 1e-3), setattr(bn, "momentum", 0.01)) for bn in bns],
}


@pytest.mark.parametrize("mode", sorted(BN_MODES))
def test_train_step_layers_in_every_batchnorm_mode(mode):
    """Frozen statistics (k_bn_fold_eval and the backward without batch-mean terms), batch statistics without an
    update (buffers bitwise unchanged), momentum None after 5 batches (1 / 6), and custom eps and momentum."""
    net = _net(17, 1024, 2, 0.5)
    with torch.no_grad():
        BN_MODES[mode](_bns(net))
    x, d_out = _inputs(64, 17, 11)
    check_layers(net, x, d_out, mode)


def test_train_step_layers_with_channels_far_from_zero():
    """Biases giving both BatchNorms channels at mean / sigma ~ 1000: the shifted statistics, the fma(z, scale, shift)
    with shift ~ -1000 gamma, and the affine coefficients of the BatchNorm backward (b z + c cancelling)."""
    J, H, B = 17, 128, 256
    net = _net(J, H, 1, 0.5)
    x, d_out = _inputs(B, J, 5)
    st = net.linear_stages[0]
    with torch.no_grad():
        y0 = x.to(dev()) @ net.w1.weight.T + net.w1.bias
        net.w1.bias += 1000 * y0.std(dim=0)
        state = {k: v.clone() for k, v in net.state_dict().items()}
        z2 = torch.from_numpy(PL.parse_saved(_run(net, x, d_out)["saved"].cpu().numpy(), B, H, 1)[1][0].copy())
        net.load_state_dict(state)
        st.w1.bias += 1000 * z2.std(dim=0).to(dev())
    check_layers(net, x, d_out, "mean/sigma 1000")


RANGE_CASES = {  # BatchNorm affine exponent, upstream gradient scale, single extreme entry
    "bn_affine_2^-12": (-12, 1.0, None),
    "bn_affine_2^8": (8, 1.0, None),
    "gradient_1e-6": (0, 1e-6, None),
    "single_1e30": (0, 1.0, 1e30),
    "single_1e-30": (0, 1.0, 1e-30),
}


@pytest.mark.parametrize("case", sorted(RANGE_CASES))
@pytest.mark.parametrize("H", [128, 4096])
def test_train_step_layers_across_operand_ranges(case, H):
    """The tensor-core GEMMs' range normalisation: activations scaled by 2^-12 / 2^8 with the BatchNorm affine,
    gradients far below fp16's range, and a gradient that is one entry at either end of fp32's range."""
    e, gscale, single = RANGE_CASES[case]
    J, B = 17, 64
    net = _net(J, H, 1, 0.5)
    with torch.no_grad():
        for bn in _bns(net):
            bn.weight.mul_(2.0 ** e)
            bn.bias.mul_(2.0 ** e)
    x, d_out = _inputs(B, J, 9, gscale)
    if single is not None:
        d_out = torch.zeros_like(d_out)
        d_out[37, 20] = single
    check_layers(net, x, d_out, f"{case} H={H}")


def test_a_pre_activation_within_rounding_of_zero():
    """One bn1 entry's pre-activation made rounding noise: beta set from the first run's saved mean and scale so that
    fmaf(z, scale, shift) cancels to within an ulp of z scale (B <= 512: one statistics block, so the second run's
    statistics are bitwise the first's).  The float64 reference cannot tell which side of the ReLU it is on; the
    per-layer check, which takes the device's mask, still holds every layer to its bound."""
    J, H, B, r, c = 17, 128, 64, 7, 5
    net = _net(J, H, 1, 0.0)
    x, d_out = _inputs(B, J, 3)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    y, _, stats, _ = PL.parse_saved(_run(net, x, d_out)["saved"].cpu().numpy(), B, H, 1)
    mean, _, scale, _ = stats[0][0]
    f32 = np.float32
    t = f32(f32(mean[c]) * scale[c])
    beta = f32(t - f32(y[0][r, c] * scale[c]))
    net.load_state_dict(state)
    with torch.no_grad():
        net.linear_stages[0].batch_norm1.bias[c] = float(beta)
    _, near = check_layers(net, x, d_out, "constructed near-zero", constructed=True)
    assert near >= 1


def test_the_grid_meets_pre_activations_near_zero():
    """The natural cases above (not the constructed one) must include pre-activations whose float64 value lies within
    its bound of zero: the situation a chained float64 reference has to tolerate, and the per-layer check must not.
    Run alone, this takes the mean / sigma ~ 1000 case, whose shifts of ~ -1000 gamma leave such entries."""
    if _NEAR_ZERO["grid"] == 0:
        test_train_step_layers_with_channels_far_from_zero()
    assert _NEAR_ZERO["grid"] >= 1, _NEAR_ZERO


@pytest.mark.parametrize("H,B,S", [(1024, 50, 2), (96, 33, 1)])
def test_capture_changes_no_result(H, B, S):
    """The capture backward, with every field, with some fields, and the plain p2m_posenet_backward_opts give bitwise
    the same output, gradients, dx and running buffers from the same state."""
    J = 17
    net = _net(J, H, S, 0.5)
    x, d_out = _inputs(B, J, 4)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    runs = []
    for capture in (None, "all", ("g_z2", "scale"), ("g_y0",), ()):
        net.load_state_dict(state)
        res = _run(net, x, d_out, capture)
        runs.append((res, {k: v.clone() for k, v in net.state_dict().items()}))
    (ref, ref_state), rest = runs[0], runs[1:]
    for res, st in rest:
        for k in ("out", "combine", "dx"):
            assert torch.equal(res[k], ref[k]), k
        parsed = [PL.parse_saved(r["saved"].cpu().numpy(), B, H, S) for r in (res, ref)]
        for a, b in zip(parsed[0][:2], parsed[1][:2]):          # y, z2 (the alignment padding is not written)
            assert all(np.array_equal(u, v) for u, v in zip(a, b))
        assert all(np.array_equal(u, v) for s0, s1 in zip(parsed[0][2], parsed[1][2]) for a, b in zip(s0, s1)
                   for u, v in zip(a, b))
        assert all(torch.equal(a, b) for a, b in zip(res["grads"], ref["grads"]))
        assert all(torch.equal(st[k], ref_state[k]) for k in st)
    full = runs[1][0]
    part = runs[2][0]
    assert all(torch.equal(a, b) for a, b in zip(part["g_z2"], full["g_z2"]))
    if H % 64 == 0:
        assert torch.equal(part["scale"], full["scale"]) and torch.isfinite(full["scale"]).all()
    else:
        assert torch.isnan(full["scale"]).all()      # no tensor-core GEMM: the scales are not written
