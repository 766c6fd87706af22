"""PoseNet's dense tensor-core GEMMs away from O(1) activations and at the edges of their padded paths: the eval
forward (p2m_posenet_forward) and the train forward + backward (p2m_posenet_train_forward / p2m_posenet_backward)
element-wise against the float64 references of fp64_ref and posenet_train_ref, with BatchNorm affine parameters or
the whole residual stream scaled by powers of two from 2^-20 to 2^16; the eval forward's exact equivariance under
power-of-two scaling; batches and output widths around the GEMMs' K-block, M-tile and N = 64 boundaries; and upstream
gradients that are all zero or a single entry at either end of fp32's range.  Every result must also be finite."""
import numpy as np
import pytest
import torch

import fp64_ref as R
from test_gpu_kernels_fp64 import _posenet
from test_gpu_posenet_train import _net, check_train_step, dev

pytestmark = pytest.mark.gpu

SEED = [0x5DEECE66D1234567, -987654321]


def _stage_bns(m):
    return [bn for st in m.linear_stages for bn in (st.batch_norm1, st.batch_norm2)]


def _scale_bn_affine(m, f):
    """gamma and beta of every stage BatchNorm times f: every activation operand of the H x H GEMMs scales by f."""
    with torch.no_grad():
        for bn in _stage_bns(m):
            bn.weight.mul_(f)
            bn.bias.mul_(f)


def _scale_stream(m, f):
    """Every Linear bias, running mean and BatchNorm beta times f: with the input also times f, every activation and
    output of the eval forward is exactly f times what it was."""
    with torch.no_grad():
        for lin in [m.w1, m.w2] + [l for st in m.linear_stages for l in (st.w1, st.w2)]:
            lin.bias.mul_(f)
        for bn in _stage_bns(m):
            bn.running_mean.mul_(f)
            bn.bias.mul_(f)


def _eval(m, x):
    with torch.no_grad():
        y, comb = m.forward_native(x.to(dev()), with_combine=True)
    return y.double().cpu().numpy(), comb.double().cpu().numpy()


# ------------------------------------------------------------------------------------------------------- eval forward
EVAL_SHAPES = [(128, 129, 17), (128, 129, 24), (4096, 33, 17), (4096, 33, 24)]   # H, B, J (3J = 51: tensor-core output)


@pytest.mark.parametrize("what", ["bn_affine", "stream"])
@pytest.mark.parametrize("e", [-20, -12, -6, 0, 6, 12, 16])
@pytest.mark.parametrize("H,B,J", EVAL_SHAPES, ids=lambda v: str(v))
def test_eval_forward_at_activation_scale(H, B, J, e, what):
    m = _posenet(J, H, seed=H + J)
    x = torch.randn(B, 2 * J, generator=torch.Generator().manual_seed(B))
    if what == "bn_affine":
        _scale_bn_affine(m, 2.0 ** e)
    else:
        _scale_stream(m, 2.0 ** e)
        x = x * 2.0 ** e
    y, _ = _eval(m, x)
    assert np.isfinite(y).all()
    sd = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items() if v.is_floating_point()}
    ref, bound = R.posenet_forward(sd, x.numpy(), 2, precision="fp16x3",
                                   last_precision="fp16x3" if 3 * J <= 64 else "fp32")
    r = R.bound_ratio(y, ref, bound)
    assert r <= 1.0, r


@pytest.mark.parametrize("H,B,J", EVAL_SHAPES[:3], ids=lambda v: str(v))
def test_eval_forward_power_of_two_scaling_is_exact(H, B, J):
    """Scaling the input, every bias, running mean and BatchNorm beta by 2^e scales pose3d by exactly 2^e, and
    pose_combine too (its pose3d / 1000 is a correctly rounded division): the fp16 split of a range-normalised operand
    does not depend on its scale."""
    x = torch.randn(B, 2 * J, generator=torch.Generator().manual_seed(B))
    y, comb = _eval(_posenet(J, H, seed=H + J), x)
    assert np.isfinite(y).all() and np.isfinite(comb).all()
    for e in (-20, -10, -3, 3, 10, 20):
        m = _posenet(J, H, seed=H + J)
        _scale_stream(m, 2.0 ** e)
        ys, combs = _eval(m, x * 2.0 ** e)
        assert np.array_equal(ys, y * 2.0 ** e), e
        assert np.array_equal(combs, comb * 2.0 ** e), e


# ------------------------------------------------------------------------------------------ train forward + backward
def _train_case(J, H, S, p, B, d_out=None, bn_exp=0):
    net = _net(J, H, S, p)
    if bn_exp:
        _scale_bn_affine(net, 2.0 ** bn_exp)
    g = torch.Generator().manual_seed(B + H)
    x = torch.randn(B, 2 * J, generator=g).to(dev())
    if d_out is None:
        d_out = torch.randn(B, 3 * J, generator=g)
    seed = torch.tensor(SEED, dtype=torch.int64, device=dev())
    return check_train_step(net, S, p, x, d_out.to(dev()), seed)


@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("H,B", [(4096, 256), (128, 50)])
@pytest.mark.parametrize("e", [-12, 0, 8])
def test_train_step_at_activation_scale(e, H, B, p):
    """BatchNorm gamma and beta times 2^e: the forward GEMMs' X and the dW GEMMs' activation operand scale with them
    (at 2^8, B = 256 and p = 0.5 the activations exceed fp16's range unless they are range-normalised)."""
    _train_case(17, H, 1, p, B, bn_exp=e)


@pytest.mark.parametrize("B,J", [(B, 17) for B in (2, 31, 33, 63, 65, 96, 127, 129, 200)] + [(65, 21), (65, 22)])
def test_train_step_batch_and_width_edges(B, J):
    """H = 128 on the tensor cores: dW's K = B padded to a multiple of 32 (k_real < K, K not a multiple of 64), ragged
    128-row M tiles in the forward and dX GEMMs, the smallest legal batch; 3J = 63 still runs the output layer on the
    tensor cores, 3J = 66 on the fp32 GEMM."""
    _train_case(J, 128, 1, 0.5, B)


def test_zero_upstream_gradient_gives_exactly_zero_gradients():
    net = _net(17, 128, 1, 0.5)
    x = torch.randn(64, 34, generator=torch.Generator().manual_seed(3)).to(dev())
    x.requires_grad_(True)
    out = net.forward_train_native(x, seed=torch.tensor(SEED, dtype=torch.int64, device=dev()))
    out.backward(torch.zeros_like(out))
    assert torch.isfinite(out).all()
    assert torch.equal(x.grad, torch.zeros_like(x))
    for k, v in net.named_parameters():
        if v.grad is not None:
            assert torch.equal(v.grad, torch.zeros_like(v)), k


@pytest.mark.parametrize("v", [1e30, 1e-30])
def test_single_extreme_upstream_gradient(v):
    d_out = torch.zeros(64, 51)
    d_out[37, 20] = v
    _train_case(17, 128, 1, 0.5, 64, d_out=d_out)
