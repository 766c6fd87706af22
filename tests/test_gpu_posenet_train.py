"""PoseNet's native train-mode forward and backward on the GPU against the float64 reference with the masks the seed
defines (tests/posenet_train_ref.py), element-wise within the derived bound; determinism, the mask's distribution, the
module's torch path at p = 0, CUDA-graph capture, and FlatPose2Mesh in train()."""
import numpy as np
import pytest
import torch

import fp64_ref as R
import posenet_train_ref as T
from helpers import graph_from_fixture

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def _net(J, H, S, p, seed=7):
    """Seeded weights with randomised BatchNorm affine parameters and running statistics."""
    from pose2mesh_release_b200 import posenet

    torch.manual_seed(seed)
    net = posenet.LinearModel(J, H, S, p)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, t in net.state_dict().items():
            if "batch_norm" in name and t.dtype.is_floating_point:
                t.copy_(torch.rand(t.shape, generator=g) + 0.5 if name.endswith(("weight", "running_var"))
                        else torch.randn(t.shape, generator=g) * 0.3)
    return net.to(dev()).train()


def _run(net, x, seed, d_out, with_combine=False):
    """One native forward + backward: (out, dx, {parameter name: grad}, pose_combine)."""
    for prm in net.parameters():
        prm.grad = None
    x = x.detach().clone().requires_grad_(True)
    res = net.forward_train_native(x, seed=seed, with_combine=with_combine)
    out, comb = res if with_combine else (res, None)
    out.backward(d_out)
    return out.detach(), x.grad, {k: v.grad for k, v in net.named_parameters() if v.grad is not None}, comb


CASES = [  # H, B, J, num_stage, p, scale of the upstream gradient
    (4096, 256, 17, 2, 0.5, 1.0),       # the reference's PoseNet: tensor cores in all three directions
    (4096, 256, 17, 2, 0.5, 1e-6),      # gradients far below fp16's range
    (1024, 64, 21, 1, 0.0, 1.0),
    (1024, 50, 21, 2, 0.5, 1e-6),       # dW's K = B padded with zero rows to 64
    (96, 50, 17, 2, 0.5, 1.0),          # H % 64 != 0: the fp32 CUDA-core GEMMs
    (96, 33, 5, 1, 0.0, 1e-6),
]


def check_train_step(net, S, p, x, d_out, seed):
    """One native forward + backward of a freshly built `net` (_net) against posenet_train_ref with the masks `seed`
    defines: every result finite and within its element-wise bound, and the relative check below."""
    H, J = net.linear_size, net.num_joint
    sd = {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}
    out, dx, grads, _ = _run(net, x, seed, d_out)
    tc = H % 64 == 0
    masks = T.dropout_masks(seed.tolist(), p, x.shape[0], H, S)
    val, bnd = T.forward_backward(sd, x.cpu().numpy(), S, masks, d_out.cpu().numpy(), "fp16x3" if tc else "fp32",
                                  "fp16x3" if tc and 3 * J <= 64 else "fp32")
    got = {"out": out, "dx": dx, **{"grad." + k: v for k, v in grads.items()}}
    after = net.state_dict()
    got.update({k: after[k] for k in val if "running_" in k})
    assert set(got) == set(val) and len(grads) == 4 + 8 * S
    bad = [k for k, v in got.items() if not torch.isfinite(v).all()]
    assert not bad, bad
    ratios = {k: R.bound_ratio(got[k].cpu().numpy(), val[k], bnd[k]) for k in val}
    worst = max(ratios, key=ratios.get)
    assert ratios[worst] <= 1.0, (worst, ratios[worst])
    # the chained bound is loose for the deepest gradients, so also an error relative to each tensor's largest entry,
    # which a gradient flushed to zero at the 1e-6 scale fails as surely as at scale 1: 1e-4 for the forward results.
    # Gradients get 2e-2 over 98 % of the entries, not the 1e-3 that holds between two fp32 implementations: of the
    # B H = 10^6 pre-activations of a layer some tens lie within fp32 rounding of zero and take the other ReLU branch
    # than in float64; each changes one entry of g_z by its full size, and the dense dX GEMM spreads that over the whole
    # row of every gradient upstream (the bound above allows exactly those).
    rel = {}
    for k in val:
        if k.endswith(".w1.bias") and "linear_stages" in k:
            continue                     # a bias in front of a BatchNorm: its exact gradient is zero (the bound covers it)
        is_grad = k == "dx" or k.startswith("grad.")
        err = np.quantile(np.abs(got[k].cpu().numpy() - val[k]), 0.98 if is_grad else 1.0) / np.abs(val[k]).max()
        rel[k] = err / (2e-2 if is_grad else 1e-4)
    worst = max(rel, key=rel.get)
    assert rel[worst] < 1.0, (worst, rel[worst], {k: round(v, 3) for k, v in rel.items()})
    for name, t in after.items():
        if name.endswith("num_batches_tracked"):
            assert int(t) == (0 if name.startswith("batch_norm1.") else 1), name
    return max(ratios.values())


@pytest.mark.parametrize("H,B,J,S,p,gscale", CASES)
def test_train_forward_backward_within_float64_bound(H, B, J, S, p, gscale):
    net = _net(J, H, S, p)
    g = torch.Generator().manual_seed(B + H)
    x = torch.randn(B, 2 * J, generator=g).to(dev())
    d_out = (torch.randn(B, 3 * J, generator=g) * gscale).to(dev())
    seed = torch.tensor([0x5DEECE66D1234567, -987654321], dtype=torch.int64, device=dev())
    check_train_step(net, S, p, x, d_out, seed)


def test_same_seed_is_bitwise_reproducible_and_seeds_differ():
    net = _net(17, 1024, 2, 0.5)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    g = torch.Generator().manual_seed(2)
    x, d_out = torch.randn(64, 34, generator=g).to(dev()), torch.randn(64, 51, generator=g).to(dev())
    runs = []
    for s in (11, 11, 12):
        net.load_state_dict(state)
        runs.append(_run(net, x, torch.tensor([s, 5], dtype=torch.int64, device=dev()), d_out))
    (o1, dx1, g1, _), (o2, dx2, g2, _), (o3, dx3, _, _) = runs
    assert torch.equal(o1, o2) and torch.equal(dx1, dx2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    assert not torch.equal(o1, o3) and not torch.equal(dx1, dx3)
    # torch.manual_seed reproduces a run through the module's own forward
    outs = []
    for _ in range(2):
        net.load_state_dict(state)
        torch.manual_seed(99)
        outs.append(net(x).detach())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_kept_fraction_and_scale(p):
    """With gamma = 0 and beta = 1 every BatchNorm output is 1, so with zero first layers, identity second layers
    (H = 3J) and zero biases the network's output IS the multipliers of dropout layer 1."""
    J, B = 32, 512
    H = 3 * J
    net = _net(J, H, 1, p)
    st = net.linear_stages[0]
    with torch.no_grad():
        for bn in (st.batch_norm1, st.batch_norm2):
            bn.weight.zero_()
            bn.bias.fill_(1.0)
        net.w1.weight.zero_(); net.w1.bias.zero_()
        st.w1.weight.zero_(); st.w1.bias.zero_()
        st.w2.weight.copy_(torch.eye(H)); st.w2.bias.zero_()
        net.w2.weight.copy_(torch.eye(H)); net.w2.bias.zero_()
    seed = torch.tensor([31337, 42], dtype=torch.int64, device=dev())
    with torch.no_grad():
        out = net.forward_train_native(torch.zeros(B, 2 * J, device=dev()), seed=seed)    # = layer 1's multipliers
    want = T.dropout_multiplier(seed.tolist(), 1, B * H, p).reshape(B, H)
    np.testing.assert_array_equal(out.cpu().numpy(), want.astype(np.float32))
    kept = float((out > 0).float().mean())
    assert abs(kept - (1 - p)) < 5 * np.sqrt(p * (1 - p) / (B * H)), kept


def test_p_zero_matches_the_torch_path():
    net = _net(17, 1024, 2, 0.0)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    g = torch.Generator().manual_seed(4)
    x, d_out = torch.randn(96, 34, generator=g).to(dev()), torch.randn(96, 51, generator=g).to(dev())
    out, dx, grads, _ = _run(net, x, None, d_out)
    native_state = {k: v.clone() for k, v in net.state_dict().items()}
    net.load_state_dict(state)
    for prm in net.parameters():
        prm.grad = None
    xr = x.clone().requires_grad_(True)
    ref = net._forward_torch(xr)
    ref.backward(d_out)

    def rel(a, b):
        return float((a - b).abs().max() / b.abs().max())

    assert rel(out, ref.detach()) < 1e-4
    assert rel(dx, xr.grad) < 1e-3
    for k, v in net.named_parameters():
        if v.grad is None:
            continue
        if k.endswith(".w1.bias") and "linear_stages" in k:     # in front of a BatchNorm: zero but for rounding
            assert float(grads[k].abs().max()) < 1e-4 * float(grads["w1.bias"].abs().max()), k
        else:
            assert rel(grads[k], v.grad) < 1e-3, k
    for k, v in net.state_dict().items():
        if "running_" in k:
            assert rel(native_state[k], v) < 1e-4, k
        if k.endswith("num_batches_tracked"):
            assert torch.equal(native_state[k], v), k


def test_forward_backward_in_a_cuda_graph_with_fresh_seeds():
    net = _net(17, 1024, 1, 0.5)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    g = torch.Generator().manual_seed(8)
    x, d_out = torch.randn(64, 34, generator=g).to(dev()), torch.randn(64, 51, generator=g).to(dev())
    seeds = [torch.tensor(s, dtype=torch.int64, device=dev()) for s in ([3, 1], [4, 1])]
    eager = []
    for s in seeds:
        net.load_state_dict(state)
        eager.append(_run(net, x, s, d_out))
    net.load_state_dict(state)
    seed = seeds[0].clone()
    xg = x.clone().requires_grad_(True)
    params = [prm for prm in net.parameters() if not prm is net.batch_norm1.weight and not prm is net.batch_norm1.bias]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                       # warm-up outside capture
        torch.autograd.grad(net.forward_train_native(xg, seed=seed), [xg] + params, d_out)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = net.forward_train_native(xg, seed=seed)
        grads = torch.autograd.grad(out, [xg] + params, d_out)
    names = [k for k, v in net.named_parameters() if any(v is q for q in params)]
    for s, (o, dx, gr, _) in zip(seeds, eager):
        seed.copy_(s)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, o) and torch.equal(grads[0], dx)
        for k, got in zip(names, grads[1:]):
            assert torch.equal(got, gr[k]), k


def test_flat_pose2mesh_trains_through_the_native_lifter():
    from pose2mesh_release_b200 import pose2mesh_net

    mats, _ = graph_from_fixture("smpl_small")
    torch.manual_seed(5)
    flat = pose2mesh_net.get_model(17, mats).to(dev()).train()
    pose2d = torch.randn(6, 17, 2, generator=torch.Generator().manual_seed(1)).to(dev())
    before = flat.pose_lifter.linear_stages[0].batch_norm1.running_mean.clone()
    torch.manual_seed(21)
    pose3d, combine = flat._lift(pose2d)
    assert pose3d.grad_fn is not None and not combine.requires_grad
    assert torch.equal(combine[..., :2], pose2d)
    assert torch.equal(combine[..., 2:], torch.div(pose3d.detach().double(), 1000).float())    # a correctly rounded division
    mesh, pose3d = flat(pose2d)
    (mesh.square().mean() + pose3d.square().mean()).backward()
    lifter = flat.pose_lifter
    assert lifter.w1.weight.grad is not None and float(lifter.w1.weight.grad.abs().max()) > 0
    assert lifter.linear_stages[1].batch_norm2.weight.grad is not None
    assert not torch.equal(lifter.linear_stages[0].batch_norm1.running_mean, before)
    assert int(lifter.linear_stages[0].batch_norm1.num_batches_tracked) == 2
    with pytest.raises(RuntimeError, match="already released"):
        pose3d.sum().backward()
    flat.eval()
    with torch.no_grad():
        mesh_e, pose3d_e = flat(pose2d)
        want = lifter.forward_native(pose2d.reshape(6, -1))
    assert torch.equal(pose3d_e.reshape(6, -1), want) and mesh_e.shape == mesh.shape


def test_batch_of_one_raises_like_torch():
    net = _net(17, 128, 1, 0.5)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        net(torch.zeros(1, 34, device=dev()))
