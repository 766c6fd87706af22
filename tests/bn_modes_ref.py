"""Float64 restatement of torch's per-BatchNorm rules (torch/nn/modules/batchnorm.py, _BatchNorm.forward) and float64
references of MeshNet and PoseNet whose BatchNorms and Dropouts act by their own state.

The rules, per BatchNorm:
  - mini-batch statistics when bn.training, or when both running buffers are None;
  - the running buffers are updated only when bn.training and bn.track_running_stats, then num_batches_tracked += 1;
  - the update factor is momentum, or 1 / num_batches_tracked (after the increment) when momentum is None;
  - the normalisation uses the biased batch variance, the running update the unbiased one.
"""
import copy

import numpy as np
import torch
import torch.nn.functional as F

P2M_BN_BATCH_UPDATE, P2M_BN_BATCH, P2M_BN_RUNNING = 0, 1, 2


def expected_opts(bn):
    """(stats, cumulative, momentum, eps) the rules above give for a BatchNorm in its current state."""
    use_batch = bn.training or (bn.running_mean is None and bn.running_var is None)
    update = bn.training and bn.track_running_stats
    stats = (P2M_BN_BATCH_UPDATE if update else P2M_BN_BATCH) if use_batch else P2M_BN_RUNNING
    return stats, int(bn.momentum is None), 0.0 if bn.momentum is None else bn.momentum, bn.eps


def batch_norm(z, gamma, beta, state, stats, cumulative, momentum, eps):
    """z [n, F] float64 (autograd-able) -> BatchNorm output.  state: dict(rm, rv, nbt) (float64 / int tensors or None)
    updated in place like torch's buffers."""
    if stats == P2M_BN_RUNNING:
        mean, var = state["rm"], state["rv"]
    else:
        n = z.shape[0]
        mean = z.mean(0)
        var = ((z - mean) ** 2).mean(0)
        if stats == P2M_BN_BATCH_UPDATE:
            with torch.no_grad():
                state["nbt"] += 1
                f = 1.0 / float(state["nbt"]) if cumulative else momentum
                state["rm"].mul_(1 - f).add_(f * mean.detach())
                state["rv"].mul_(1 - f).add_(f * var.detach() * n / (n - 1))
    return (z - mean) / torch.sqrt(var + eps) * gamma + beta


def module64(module):
    """A float64 CPU copy of `module` (train / eval states of every submodule kept)."""
    m = copy.deepcopy(module).cpu().double()
    for a, b in zip(m.modules(), module.modules()):
        a.training = b.training
    return m


def meshnet_forward(m, laps, x):
    """Pose2Mesh.forward in float64 with the copy m (module64) of the module: the oracle's Chebyshev conv, then each
    layer's own nn.BatchNorm1d module (its mode, momentum, eps and buffers).  laps: oracle.meshnet_oracle's Laplacians."""
    from oracle import meshnet_oracle as mo

    plan = m.CL_F
    n_blk, n_joint = len(plan), laps[-1].shape[0]
    x = x.reshape(-1, n_joint, m.num_joint_input_chan)
    li = 0
    for i, chans in enumerate(plan):
        block_in = x
        lap = laps[-(i + 1) + (1 if i == n_blk - 1 else 0)]
        for j in range(len(chans) - 1):
            x = mo.cheb_conv(x, lap, m.cl[li].weight, m.cl[li].bias)
            if m.bn[li] is not None:
                b, v, f = x.shape
                x = F.relu(m.bn[li](x.reshape(b * v, f)).reshape(b, v, f))
            li += 1
        if i == 0:
            x = F.linear(x.reshape(-1, n_joint * chans[-1]), m.fc.weight, m.fc.bias).view(-1, laps[-2].shape[0],
                                                                                          plan[1][0])
        elif i < n_blk - 2:
            x = mo.unpool2(mo.channel_resample(block_in, x.shape[2]) + x)
        elif i == n_blk - 2:
            x = mo.channel_resample(block_in, x.shape[2]) + x
    return x


def laplacians64(graph_L):
    from oracle import meshnet_oracle as mo

    return [L.double() for L in mo.laplacians_to_torch(graph_L)]


def posenet_forward(m, x, masks):
    """LinearModel.forward in float64 with the copy m (module64): each stage's BatchNorms by their own state, each
    dropout as the multiplier masks[2 s + {0, 1}] ([B, H] float64, ones for no dropout)."""
    y = m.w1(x)
    for s, st in enumerate(m.linear_stages):
        h = st.w1(F.relu(st.batch_norm1(y)) * masks[2 * s])
        y = y + st.w2(F.relu(st.batch_norm2(h)) * masks[2 * s + 1])
    return m.w2(y)


def close(got, ref, tol):
    """max |got - ref| <= tol * max |ref| (plus a floor for all-zero references); returns the ratio for messages."""
    got = got.detach().double().cpu() if isinstance(got, torch.Tensor) else torch.as_tensor(np.asarray(got))
    ref = ref.detach().double().cpu() if isinstance(ref, torch.Tensor) else torch.as_tensor(np.asarray(ref))
    scale = max(float(ref.abs().max()), 1e-30)
    return float((got - ref).abs().max()) / (tol * scale)


def grad_ok(got, ref):
    """The project's gradient parity (tests/test_gpu_parity.py::grad_close): within 1e-3 of the tensor's largest entry,
    or, where a ReLU pre-activation within rounding of zero flips between fp32 and float64, a relative L2 error of
    1e-2 with no entry off by more than 5e-2 of the largest one."""
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    scale = max(float(ref.abs().max()), 1e-30)
    mx = float((got - ref).abs().max()) / scale
    l2 = float((got - ref).norm()) / max(float(ref.norm()), 1e-30)
    return mx <= 1e-3 or (l2 <= 1e-2 and mx <= 5e-2), (mx, l2)
