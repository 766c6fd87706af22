"""TEST INFRASTRUCTURE ONLY — CPU (torch fp32) restatement of the reference's MeshNet hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this package; the product path never does and fails loudly without its CUDA library.

Restates what hongsukchoi/Pose2Mesh_RELEASE computes in

    lib/models/backbones/cheby_graph_conv.py:5-42   graph_conv_cheby
    lib/models/meshnet.py:12-62                     Pose2Mesh.__init__ (channel plan, init, state_dict layout)
    lib/models/meshnet.py:71-78                     graph_upsample (nearest x2 along vertices)
    lib/models/meshnet.py:80-117                    Pose2Mesh.forward
    lib/graph_utils.py:98-109                       sparse_python_to_torch (f64 CSR -> f32)

All floating-point work runs in the same library the reference uses (PyTorch CPU kernels:
torch.sparse.mm, addmm, batch_norm, interpolate) but is re-derived from the algorithm, as a
stateless function of (state_dict, Laplacians, x).  Gradients come from torch autograd over this
restatement.

Parity status: PINNED against outputs of the unmodified reference run in the build container
(tests/golden/*.npz, made by tests/golden/make_golden.py); see tests/test_oracle_golden.py.
The reference itself holds no numeric test for this path (SURVEY.md §4).
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np
import torch
import torch.nn.functional as F

CHEB_K = 3  # meshnet.py:23,29 — every layer uses K = 3


def channel_plan(n_in: int, n_out: int, mano: bool):
    """meshnet.py:21-33: per block, the channel widths of its conv chain."""
    if mano:
        return [(n_in, 32, 64, 64), (64, 128, 256), (256, 256, 256), (256, 256, 256), (256, 256, 256),
                (256, 128, 128), (128, 64, n_out)]
    return [(n_in, 32, 64, 64), (64, 128, 256), (256, 256, 256), (256, 256, 256), (256, 256, 256),
            (256, 256, 256), (256, 128, 128), (128, 128, 128), (128, 128, 128), (128, 64, n_out)]


def laplacians_to_torch(graph_L: Sequence, drop_second_coarsest: bool = True) -> List[torch.Tensor]:
    """meshnet.py:35 (`del graph_L[-2]`) + graph_utils.py:98-109 (values cast f64 -> f32).
    Returns CSR fp32 tensors ordered fine -> coarse with the joint graph last."""
    mats = list(graph_L)
    if drop_second_coarsest:
        del mats[-2]
    out = []
    for m in mats:
        c = m.tocsr().astype(np.float32)
        c.sort_indices()
        out.append(torch.sparse_csr_tensor(torch.from_numpy(c.indptr.astype(np.int64)),
                                           torch.from_numpy(c.indices.astype(np.int64)),
                                           torch.from_numpy(c.data), size=c.shape))
    return out


def init_state_dict(n_in: int, n_out: int, level_sizes: Sequence[int], mano: bool) -> Dict[str, torch.Tensor]:
    """Parameter set with the reference's names, shapes and initialiser (meshnet.py:36-58), consuming
    the global torch RNG in the reference's order (fc first; each nn.Linear draws its default
    kaiming weight and bias before the weight is re-drawn from U(+-sqrt(2/(3Fin+Fout))))."""
    plan = channel_plan(n_in, n_out, mano)
    sd: Dict[str, torch.Tensor] = {}
    fc = torch.nn.Linear(level_sizes[-1] * plan[0][-1], level_sizes[-2] * plan[1][0])
    sd["fc.weight"], sd["fc.bias"] = fc.weight.detach().clone(), fc.bias.detach().clone()
    idx = 0
    n_layers = sum(len(p) - 1 for p in plan)
    for chans in plan:
        for fin, fout in zip(chans[:-1], chans[1:]):
            lin = torch.nn.Linear(CHEB_K * fin, fout)
            bound = float(np.sqrt(2.0 / (CHEB_K * fin + fout)))
            lin.weight.data.uniform_(-bound, bound)
            sd[f"cl.{idx}.weight"] = lin.weight.detach().clone()
            sd[f"cl.{idx}.bias"] = torch.zeros(fout)
            if idx != n_layers - 1:
                sd[f"bn.{idx}.weight"] = torch.ones(fout)
                sd[f"bn.{idx}.bias"] = torch.zeros(fout)
                sd[f"bn.{idx}.running_mean"] = torch.zeros(fout)
                sd[f"bn.{idx}.running_var"] = torch.ones(fout)
                sd[f"bn.{idx}.num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
            idx += 1
    return sd


def cheb_conv(x, lap, weight, bias, bn=None, training=False, bn_momentum=0.1, bn_eps=1e-5):
    """cheby_graph_conv.py:5-42.  x [B,V,Fin]; weight [Fout, Fin*3] with column = fin*3 + k.
    bn = None or dict(weight,bias,running_mean,running_var[,num_batches_tracked]) (updated in place
    when training, like nn.BatchNorm1d)."""
    b, v, fin = x.shape
    t0 = x.permute(1, 2, 0).reshape(v, fin * b)           # V x (Fin*B), B innermost (ref :16-17)
    t1 = torch.sparse.mm(lap, t0)                          # ref :25
    t2 = 2 * torch.sparse.mm(lap, t1) - t0                 # ref :28
    basis = torch.stack((t0, t1, t2), 0).view(CHEB_K, v, fin, b)
    basis = basis.permute(3, 1, 2, 0).reshape(b * v, fin * CHEB_K)   # ref :32-34, k fastest
    y = torch.addmm(bias, basis, weight.t())               # ref :37
    if bn is not None:                                     # ref :38-39
        if training and "num_batches_tracked" in bn:
            bn["num_batches_tracked"] += 1
        y = F.batch_norm(y, bn["running_mean"], bn["running_var"], bn["weight"], bn["bias"],
                         training, bn_momentum, bn_eps)
    return y.view(b, v, -1)


def unpool2(x):
    """meshnet.py:71-78: out[:, 2i] = out[:, 2i+1] = x[:, i]."""
    return x.repeat_interleave(2, dim=1)


def channel_resample(x, fout):
    """meshnet.py:109,114: F.interpolate(mode='linear', align_corners=False) along the LAST axis of
    [B,V,F] — a 1-D resampling of the feature axis (F4 in SURVEY.md)."""
    return F.interpolate(x, size=fout, mode="linear")


def forward(sd: Dict[str, torch.Tensor], laps: Sequence[torch.Tensor], x: torch.Tensor, *, mano: bool = False,
            training: bool = False, n_in: int = 5, n_out: int = 3, collect=None, plan=None) -> torch.Tensor:
    """meshnet.py:80-117.  `laps` from laplacians_to_torch (fine -> coarse, joint graph last).
    `sd` is a reference-layout state dict (tensors may require grad).  If `collect` is a list, every
    conv layer's post-activation output is appended (layer-by-layer parity).  `plan` replaces the
    reference's channel plan (len(laps) == len(plan) - 1); the dtype of `sd` and `x` is the one computed in."""
    if plan is None:
        plan = channel_plan(n_in, n_out, mano)
    n_blk = len(plan)
    n_joint = laps[-1].shape[0]
    x = x.reshape(-1, n_joint, n_in)
    li = 0
    for i, chans in enumerate(plan):
        block_in = x
        lap = laps[-(i + 1) + (1 if i == n_blk - 1 else 0)]          # ref :92-94 (last block re-uses the finest level)
        for j in range(len(chans) - 1):
            last = (i == n_blk - 1) and (j == len(chans) - 2)
            bn = None
            if not last:
                bn = {k: sd[f"bn.{li}.{k}"] for k in ("weight", "bias", "running_mean", "running_var")}
                if f"bn.{li}.num_batches_tracked" in sd:
                    bn["num_batches_tracked"] = sd[f"bn.{li}.num_batches_tracked"]
            x = cheb_conv(x, lap, sd[f"cl.{li}.weight"], sd[f"cl.{li}.bias"], bn, training)
            if not last:
                x = F.relu(x)                                       # ref :99-100
            if collect is not None:
                collect.append(x)
            li += 1
        if i == 0:                                                  # ref :104-106
            x = F.linear(x.reshape(-1, n_joint * chans[-1]), sd["fc.weight"], sd["fc.bias"])
            x = x.view(-1, laps[-2].shape[0], plan[1][0])
        elif i < n_blk - 2:                                         # ref :108-111
            x = unpool2(channel_resample(block_in, x.shape[2]) + x)
        elif i == n_blk - 2:                                        # ref :113-115
            x = channel_resample(block_in, x.shape[2]) + x
    return x


def randomize_bn_(sd: Dict[str, torch.Tensor], seed: int = 7):
    """SURVEY.md §8(d): make eval-mode BN non-trivial so folding bugs show."""
    g = torch.Generator().manual_seed(seed)
    for k in sorted(sd):
        if not k.startswith("bn."):
            continue
        t = sd[k]
        if k.endswith(".weight") or k.endswith(".running_var"):
            t.copy_(torch.rand(t.shape, generator=g) + 0.5)
        elif k.endswith(".bias") or k.endswith(".running_mean"):
            t.copy_(torch.randn(t.shape, generator=g) * 0.1)
    return sd
