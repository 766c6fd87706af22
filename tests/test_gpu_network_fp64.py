"""MeshNet's network schedules layer by layer against float64 (tests/fp64_ref.py), at both precisions.

The eval forward, the training forward and p2m_meshnet_backward run paths no single-layer entry point reaches: padding
-vertex elision, the dedup classes, the fused 64 -> 3 head, the virtual x2 unpool, residuals in the epilogue and in the
BatchNorm pass, backward-data as a conv on dz, dW from the basis of dz, the dT GEMMs, the thin head's backward, the fc
on the tensor cores; and their tensor-core operands follow the network's precision model (activations split as they
are, weights at the fixed 2^6: split='network' of the conv bounds).  p2m_debug_set_capture copies every layer's tensors
as the device produced them, so each layer is checked from its own captured inputs: no error bound is carried through
the network.  Every check is max |err| / bound <= 1, element-wise.

The worst error-to-bound ratio per precision is written to the JSON file named by P2M_NET_FP64_REPORT (if set)."""
import json
import os
import time

import numpy as np
import pytest
import torch

import fp64_ref as R
import graphs as G
from helpers import CASES, graph_from_fixture

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16x3"]
_WORST = {}

# levels {128, 64, joint 17}: block 0 on the joint level, block 1's 64 -> 256 has Fout > 3 Fin (dX by the dT GEMMs:
# the conv on dz needs Fout <= 3 Fin, and a 64-wide output) and ends in a resampled residual + unpool, block 2 in an
# identity residual, block 3 is the fused 256 -> 64 -> 3 head
CUSTOM_PLAN = [(5, 32, 64), (64, 256), (256, 128, 256), (256, 64, 3)]


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    out = os.environ.get("P2M_NET_FP64_REPORT")
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


def cuda(a):
    return torch.as_tensor(np.asarray(a)).float().to(dev()).contiguous()


def npy(t):
    return t.detach().double().cpu().numpy()


# ------------------------------------------------------------------------------------------------------------- nets
def net_levels(name):
    if name in G.ELISION:   # a padded level and its hierarchy (tests/test_gpu_elision_tiles_fp64.py)
        return G.elision_hierarchy(G.elision(name)), G.ELISION_PLAN
    if name == "custom":
        mats = graph_from_fixture("smpl_small")[0]
        return [next(m for m in mats if m.shape[0] == V) for V in (128, 64, 17)], CUSTOM_PLAN
    from pose2mesh_release_b200.meshnet import channel_plan

    if name == "smpl_like":   # its fixture stores digests only: rebuild the hierarchy (test_gpu_at_size._hierarchy)
        from pose2mesh_release_b200 import graph as pg

        n, seed, levels, _ = CASES[name]
        face = pg.synthetic_sphere_faces(n, seed)
        mats = list(pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=levels)[1])
    else:
        mats = list(graph_from_fixture(name)[0])
    del mats[-2]   # meshnet.py:35
    return mats, channel_plan(5, 3, name == "mano_like")


class Net:
    """A MeshNet of `plan` through BakedHierarchy (test_gpu_batchnorm_fp64.small_net's parameters) plus the block
    structure of p2m_api.cu's schedules, mirrored for the references."""

    def __init__(self, name, precision, seed, open_relus, bias_shift=0.0):
        import test_gpu_batchnorm_fp64 as T

        self.levels, self.plan = net_levels(name)
        self.hier, self.sd, self.n_layers, _ = T.small_net(self.levels, self.plan, precision, seed, open_relus,
                                                           bias_shift)
        # the Laplacians as the device holds them (fp32 values)
        self.L32 = [m.tocsr().astype(np.float32).astype(np.float64) for m in self.levels]
        nb, nlev = len(self.plan), len(self.levels)
        self.blocks, self.layers = [], []
        for b, chans in enumerate(self.plan):
            blk = dict(first=len(self.layers), n=len(chans) - 1, level=0 if b == nb - 1 else nlev - 1 - b,
                       res=1 <= b <= nb - 2, out_unpool=1 <= b < nb - 2, in_unpool=2 <= b <= nb - 2,
                       cin=chans[0], cout=chans[-1])
            self.blocks.append(blk)
            for j in range(len(chans) - 1):
                self.layers.append(dict(block=b, j=j, fin=chans[j], fout=chans[j + 1], level=blk["level"],
                                        bn=len(self.layers) != self.n_layers_total() - 1, end=j == len(chans) - 2))
        self.p = {k: v.double().numpy() for k, v in self.sd.items() if v.is_floating_point()}

    def n_layers_total(self):
        return sum(len(c) - 1 for c in self.plan)

    def V(self, li):
        return self.levels[self.layers[li]["level"]].shape[0]

    def route(self, li, B, need_dx=True):
        return self.hier.layer_route(0, li, B, need_dx)

    @property
    def precision(self):
        """The precision the net's hierarchy runs at, by its name in _lib.PRECISIONS."""
        from pose2mesh_release_b200 import _lib

        return next(k for k, v in _lib.PRECISIONS.items() if v == self.hier.precision)

    def conv_precision(self, on_tc):
        """The precision a conv pass runs at: the net's on the tensor cores, fp32 on the CUDA cores."""
        return self.precision if on_tc else "fp32"

    def fc_precision(self):
        """The precision the fc runs at: an fp16x3 dense GEMM at every tensor-core precision."""
        return "fp32" if self.precision == "fp32" else "fp16x3"

    def capture_buffers(self, B, names):
        cap = {}
        for name in names:
            if name in ("fc_out", "fc_dx"):
                n = self.levels[-2].shape[0] * self.plan[1][0] if name == "fc_out" else \
                    self.levels[-1].shape[0] * self.plan[0][-1]
                cap[name] = torch.full((B, n), float("nan"), device=dev())
            else:
                f = "fin" if name == "dx" else "fout"
                cap[name] = [torch.full((B, self.V(li) // (2 if name == "dx" and self.in_unpool(li) else 1),
                                         L[f]), float("nan"), device=dev()) for li, L in enumerate(self.layers)]
        return cap

    def in_unpool(self, li):
        L = self.layers[li]
        return L["j"] == 0 and self.blocks[L["block"]]["in_unpool"]


def layer_input(net, li, x, fc_out, act, ref=R):
    """The conv input of layer li (unpooled where the block reads its input through the virtual x2 unpool) and the
    block input (for the residual), from the captured activations act[l].  ref: the reference module (fp64_ref, or
    fp64_ref_torch for device tensors)."""
    R = ref
    L = net.layers[li]
    blk = net.blocks[L["block"]]
    b = L["block"]
    if b == 0:
        block_in = x
    elif b == 1:
        block_in = fc_out.reshape(x.shape[0], net.levels[-2].shape[0], -1)
    else:
        prev = net.blocks[b - 1]
        block_in = act[prev["first"] + prev["n"] - 1]
    if blk["in_unpool"]:
        block_in = R.unpool(block_in)
    inp = block_in if L["j"] == 0 else act[li - 1]
    return inp, block_in


def conv_ref(net, li, inp, precision):
    W, b = net.p[f"cl.{li}.weight"], net.p[f"cl.{li}.bias"]
    L = net.L32[net.layers[li]["level"]]
    return R.cheb_conv_fwd(inp, L, W, b), R.cheb_conv_fwd_bound(inp, L, W, b, precision, split="network")


def fc_ref(a0, W, b, precision):
    """The fc (launch_umma_gemm at fp16x3: activations range-normalised, weights at the fixed 2^6) and its bound."""
    ref = R.dense(a0, W, b)
    bound = R.gamma(a0.shape[1], precision) * (np.abs(a0) @ np.abs(W).T) + R.U32 * (np.abs(b) + np.abs(ref))
    if precision == "fp16x3":
        bound = bound + (2.0 ** -34 * float(np.abs(a0).max()) * np.abs(W).sum(axis=1)[None, :]
                         + R.NET_LO / R.NET_W_SCALE * np.abs(a0).sum(axis=1, keepdims=True))
    return ref, bound


def residual(net, li, block_in, ref=R):
    """The residual added at the end of layer li's block (resampled or identity) and its fp32 evaluation bound."""
    L, blk = net.layers[li], net.blocks[net.layers[li]["block"]]
    if not (L["end"] and blk["res"]):
        return 0.0, 0.0
    return ref.channel_resample(block_in, blk["cout"]), ref.channel_resample_bound(block_in, blk["cout"])


# ----------------------------------------------------------------------------------------------------------- running
def forward_train_backward(net, x, tgt, need_dx=True, loss_fn=None):
    """One train-mode forward + L1 loss (or loss_fn(y, tgt)) + backward with every tensor captured.  Returns (cap,
    grads, buffers, y)."""
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    B = x.shape[0]
    n = net.n_layers
    n_bn = n - 1
    sd = net.sd
    p = {k: cuda(v).requires_grad_(True) for k, v in sd.items() if "running" not in k and "num_batches" not in k}
    buf = {k: cuda(v) if v.is_floating_point() else v.to(dev()) for k, v in sd.items()
           if "running" in k or "num_batches" in k}
    names = (["fc.weight", "fc.bias"] + [f"cl.{i}.weight" for i in range(n)] + [f"cl.{i}.bias" for i in range(n)]
             + [f"bn.{i}.weight" for i in range(n_bn)] + [f"bn.{i}.bias" for i in range(n_bn)])
    buffers = ([buf[f"bn.{i}.running_mean"] for i in range(n_bn)] + [None],
               [buf[f"bn.{i}.running_var"] for i in range(n_bn)] + [None],
               [buf[f"bn.{i}.num_batches_tracked"] for i in range(n_bn)] + [None])
    cap = net.capture_buffers(B, ("z", "a", "fc_out", "g_a", "g_z", "dx", "fc_dx"))
    for k in ("z", "a"):    # the last layer has no BatchNorm: nothing captured
        cap[k][-1] = None
    if not need_dx:
        cap["dx"][0] = None
    net.hier.set_capture(0, cap)
    try:
        xg = cuda(x).requires_grad_(need_dx)
        y = _MeshNetFunction.apply(xg, net.hier, True, buffers, n, *[p[k] for k in names])
        loss = (y - cuda(tgt)).abs().mean() if loss_fn is None else loss_fn(y, cuda(tgt))
        loss.backward()
        torch.cuda.synchronize()
    finally:
        net.hier.set_capture(0, None)
    assert net.hier.kernel_status(0) == 0
    grads = {k: npy(p[k].grad) for k in names}
    if need_dx:
        assert torch.equal(xg.grad, cap["dx"][0])
    out = {k: ([None if t is None else npy(t) for t in v] if isinstance(v, list) else npy(v)) for k, v in cap.items()}
    return out, grads, {k: npy(v) for k, v in buf.items() if v.is_floating_point()}, npy(y)


def check_train(net, tag, x, y, cap, grads, bufs, need_dx):
    """Every layer of the training forward and of the backward from its captured inputs."""
    prec = net.precision
    B = x.shape[0]
    n = net.n_layers
    a = {li: cap["a"][li].reshape(B, net.V(li), -1) for li in range(n - 1)}
    fc_out = cap["fc_out"]
    # ---- forward
    for li, L in enumerate(net.layers):
        r = net.route(li, B, need_dx)
        inp, block_in = layer_input(net, li, x, fc_out, a)
        z64, E = conv_ref(net, li, inp, net.conv_precision(r["tc"]))
        t = f"{tag} layer {li} ({L['fin']}->{L['fout']} V={net.V(li)})"
        if not L["bn"]:
            check(t + " y", prec, y.reshape(z64.shape), z64, E)
            continue
        z = cap["z"][li].reshape(z64.shape)
        check(t + " z", prec, z, z64, E)
        g, be = net.p[f"bn.{li}.weight"], net.p[f"bn.{li}.bias"]
        rm, rv = net.p[f"bn.{li}.running_mean"], net.p[f"bn.{li}.running_var"]
        y64, _, _, rm64, rv64 = R.bn_train_fwd(z, g, be, rm, rv, relu=True)
        bd = R.bn_train_fwd_bound(z, np.zeros_like(z), g, be, rm, rv)
        res, eres = residual(net, li, block_in)
        a64 = y64 + res
        check(t + " a", prec, a[li], a64, bd["y"] + eres + R.U32 * np.abs(a64))
        check(t + " running_mean", prec, bufs[f"bn.{li}.running_mean"], rm64, bd["rm"])
        check(t + " running_var", prec, bufs[f"bn.{li}.running_var"], rv64, bd["rv"])
        if li == net.blocks[0]["first"] + net.blocks[0]["n"] - 1:   # the fc
            check(f"{tag} fc_out", prec, fc_out,
                  *fc_ref(a[li].reshape(B, -1), net.p["fc.weight"], net.p["fc.bias"], net.fc_precision()))
    # ---- backward
    for li in range(n - 1, -1, -1):
        L = net.layers[li]
        blk = net.blocks[L["block"]]
        r = net.route(li, B, need_dx)
        t = f"{tag} bwd layer {li} ({L['fin']}->{L['fout']} V={net.V(li)})"
        inp, block_in = layer_input(net, li, x, fc_out, a)
        Lm = net.L32[L["level"]]
        g_a = cap["g_a"][li].reshape(B, net.V(li), -1)
        g_z = cap["g_z"][li].reshape(g_a.shape)
        if L["bn"]:
            z = cap["z"][li].reshape(g_a.shape)
            g, be = net.p[f"bn.{li}.weight"], net.p[f"bn.{li}.bias"]
            gz64, dg64, db64, pre = R.bn_train_bwd(z, g_a, g, be, relu=True)
            bz, bg, bb = R.bn_train_bwd_bound(z, g_a, g, be, relu=True)
            assert float(np.abs(pre).min()) > 1e-2, t + ": a ReLU near its switch in a backward case"
            check(t + " g_z", prec, g_z, gz64, bz)
            check(t + " dgamma", prec, grads[f"bn.{li}.weight"], dg64, bg)
            check(t + " dbeta", prec, grads[f"bn.{li}.bias"], db64, bb)
            assert np.count_nonzero(grads[f"cl.{li}.bias"]) == 0, t
        else:
            assert np.array_equal(g_z, g_a), t
        W = net.p[f"cl.{li}.weight"]
        dx64, dW64, db64 = R.cheb_conv_bwd(inp, Lm, W, g_z)
        on_dw = r["tc_dw"] or r["dw_dz_basis"]
        on_dx = r["tc_dx"] or r["tc_dt"]
        bdx, _, bdb = R.cheb_conv_bwd_bound(inp, Lm, W, g_z, net.conv_precision(on_dx), split="network")
        _, bdw, _ = R.cheb_conv_bwd_bound(inp, Lm, W, g_z, net.conv_precision(on_dw), split="network",
                                          dw_chain=dw_chain(net, li, B))
        check(t + " dW", prec, grads[f"cl.{li}.weight"], dW64, bdw)
        if not L["bn"]:
            check(t + " db", prec, grads[f"cl.{li}.bias"], db64, R.col_sum_bound(g_z))
        if li == 0 and not need_dx:
            continue
        ref, bound = dx64, bdx
        if L["j"] == 0 and blk["res"]:
            g_res = cap["g_a"][blk["first"] + blk["n"] - 1].reshape(B, net.V(li), -1)
            rt = R.channel_resample_t(g_res, L["fin"])
            ref = ref + rt
            bound = bound + R.channel_resample_t_bound(g_res, L["fin"]) + R.U32 * (np.abs(dx64) + np.abs(rt))
        if net.in_unpool(li):
            ref, bound = R.unpool_t(ref), R.unpool_t(bound) + R.U32 * np.abs(R.unpool_t(ref))
        dx = cap["dx"][li].reshape(ref.shape)
        check(t + " dx", prec, dx, ref, bound)
        if li == blk["first"] and L["block"] == 1:    # the fc backward, from the gradient it read
            gf = dx.reshape(B, -1)
            a0 = a[net.blocks[0]["first"] + net.blocks[0]["n"] - 1].reshape(B, -1)
            Wf = net.p["fc.weight"]
            g_dw = R.gamma(B, "fp32") + B.bit_length() * R.U32
            check(f"{tag} fc dW", prec, grads["fc.weight"], gf.T @ a0, g_dw * (np.abs(gf).T @ np.abs(a0)))
            check(f"{tag} fc db", prec, grads["fc.bias"], gf.sum(axis=0), R.col_sum_bound(gf))
            ref_fx = gf @ Wf
            check(f"{tag} fc dx", prec, cap["fc_dx"], ref_fx,
                  R.gamma(Wf.shape[0], "fp32") * (np.abs(gf) @ np.abs(Wf)))
            assert np.array_equal(cap["fc_dx"].reshape(B, -1), cap["g_a"][blk["first"] - 1].reshape(B, -1)), tag


def dw_chain(net, li, B):
    """With the persistent grids capped at net.sm_cap SMs (tests/test_gpu_persistent_tiles_fp64.py): the fp32 adds a dW
    element of layer li goes through, the rows of one CTA's 128-row tiles and then one atomic add per CTA; 0 (the
    default bound) without a cap."""
    cap = getattr(net, "sm_cap", 0)
    if not cap:
        return 0
    n_tiles = B * -(-net.V(li) // 128)
    grid = min(n_tiles, cap)
    return -(-n_tiles // grid) * 128 + grid


def train_inputs(net, B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, net.levels[-1].shape[0], 5, generator=g).numpy().astype(np.float32)
    tgt = torch.randn(B, net.levels[0].shape[0], 3, generator=g).numpy().astype(np.float32)
    return x, tgt


TRAIN_CASES = [  # (net, elide_padding, B, need_dx): every net at elide 0 / 1 / 2, B 1 and 3, with and without dx
    ("custom", 0, 1, True), ("custom", 1, 3, False), ("custom", 2, 3, True), ("custom", 1, 1, False),
    ("custom", 2, 1, True), ("custom", 0, 3, False),
    ("mano_like", 0, 3, False), ("mano_like", 1, 1, True), ("mano_like", 2, 3, True),
    ("smpl_small", 0, 1, True), ("smpl_small", 1, 3, True), ("smpl_small", 2, 1, False),
]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,elide,B,need_dx", TRAIN_CASES, ids=lambda v: str(v))
def test_train_step_layer_by_layer(name, elide, B, need_dx, precision):
    """Training forward (z, a, running statistics, fc_out) and backward (g_z, dgamma, dbeta, dW, db, dx, the fc's
    gradients) of every layer against float64 from the layer's captured inputs; open ReLUs (BN bias 6)."""
    net = Net(name, precision, seed=100 * elide + B, open_relus=True)
    net.hier.set_debug(0, elide_padding=elide)
    x, tgt = train_inputs(net, B, seed=B + elide)
    cap, grads, bufs, y = forward_train_backward(net, x, tgt, need_dx)
    check_train(net, f"{name} elide={elide} B={B} dx={need_dx}", x, y, cap, grads, bufs, need_dx)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_train_step_with_shifted_channels(precision):
    """Every pre-BN channel at mean / sigma ~ 1000 (1000 added to every conv bias in front of a BatchNorm): the BN
    backward's affine coefficients and the statistics under cancellation."""
    net = Net("custom", precision, seed=7, open_relus=True, bias_shift=1000.0)
    x, tgt = train_inputs(net, 3, seed=9)
    cap, grads, bufs, y = forward_train_backward(net, x, tgt, True)
    check_train(net, "custom shifted", x, y, cap, grads, bufs, True)


# -------------------------------------------------------------------------------------------------------------- eval
def forward_eval(net, x, elide, dedup, fuse, capture=True):
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    B = x.shape[0]
    n = net.n_layers
    sd = net.sd
    net.hier.set_debug(0, elide_padding=elide, dedup_padding=dedup, fuse_head=fuse)
    n_bn = n - 1
    params = ([cuda(sd["fc.weight"]), cuda(sd["fc.bias"])] + [cuda(sd[f"cl.{i}.weight"]) for i in range(n)]
              + [cuda(sd[f"cl.{i}.bias"]) for i in range(n)] + [cuda(sd[f"bn.{i}.weight"]) for i in range(n_bn)]
              + [cuda(sd[f"bn.{i}.bias"]) for i in range(n_bn)])
    buffers = ([cuda(sd[f"bn.{i}.running_mean"]) for i in range(n_bn)] + [None],
               [cuda(sd[f"bn.{i}.running_var"]) for i in range(n_bn)] + [None], [None] * n)
    cap = net.capture_buffers(B, ("y", "fc_out")) if capture else None
    if capture:
        net.hier.set_capture(0, cap)
    try:
        with torch.no_grad():
            y = _MeshNetFunction.apply(cuda(x), net.hier, False, buffers, n, *params)
        torch.cuda.synchronize()
    finally:
        net.hier.set_capture(0, None)
    assert net.hier.kernel_status(0) == 0
    if not capture:
        return npy(y), None
    return npy(y), {k: ([npy(t) for t in v] if isinstance(v, list) else npy(v)) for k, v in cap.items()}


def eval_layer(net, li, inp, block_in, precision):
    """Float64 eval output of layer li (folded BatchNorm + ReLU + residual, or the head's conv) and its bound with the
    conv at `precision`."""
    L = net.layers[li]
    z64, E = conv_ref(net, li, inp, precision)
    if not L["bn"]:
        return z64, E
    g, be = net.p[f"bn.{li}.weight"], net.p[f"bn.{li}.bias"]
    rm, rv, b = net.p[f"bn.{li}.running_mean"], net.p[f"bn.{li}.running_var"], net.p[f"cl.{li}.bias"]
    y64 = R.bn_eval_fwd(z64, g, be, rm, rv, relu=True)
    bound = R.bn_eval_fwd_bound(z64, E, g, be, rm, rv, b)
    res, eres = residual(net, li, block_in)
    return y64 + res, bound + eres + R.U32 * np.abs(y64 + res)


EVAL_CASES = [(name, elide, B) for name in ("custom", "mano_like", "smpl_small") for elide, B in ((0, 3), (1, 1), (2, 3))]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,elide,B", EVAL_CASES, ids=lambda v: str(v))
def test_eval_forward_layer_by_layer(name, elide, B, precision):
    """Eval forward, dedup and fused head off: every layer's output (and the fc's) against folded BatchNorm + conv of its
    captured input, live ReLUs (an element within its bound of zero may take either branch: ReLU is 1-Lipschitz, so
    the bound covers it).  Then the fused head against the two-layer float64 composition from the fused layer's
    captured input, and dedup on against dedup off bit for bit: a representative row is computed by the same
    combined-weight GEMM as with every isolated row computed, and no connected row reads an isolated one."""
    net = Net(name, precision, seed=31 + B + elide, open_relus=False)
    x, _ = train_inputs(net, B, seed=5 + elide)
    tag = f"{name} eval elide={elide} B={B}"
    y, yf, _, _ = check_eval(net, tag, x, elide)
    # dedup: bit for bit against dedup off, with the fused head on and off
    for fuse in (False, True):
        yd, _ = forward_eval(net, x, elide, dedup=True, fuse=fuse, capture=False)
        yo = y if not fuse else yf
        assert np.array_equal(yd, yo), (tag, "dedup", fuse, float(np.abs(yd - yo).max()))


def check_eval(net, tag, x, elide):
    """The eval forward with dedup off, fused head off and then on: every layer's output (and the fc's) from its
    captured input, then the fused head from the fused layer's captured input.  Returns (y, y with the fused head,
    the layers' captured outputs, the fc's), the captures of the run with the fused head off."""
    precision = net.precision
    B = x.shape[0]
    y, cap = forward_eval(net, x, elide, dedup=False, fuse=False)
    n = net.n_layers
    act = {li: cap["y"][li].reshape(B, net.V(li), -1) for li in range(n)}
    fc_out = cap["fc_out"]
    assert np.array_equal(act[n - 1], y.reshape(act[n - 1].shape)), tag
    for li in range(n):
        inp, block_in = layer_input(net, li, x, fc_out, act)
        ref, bound = eval_layer(net, li, inp, block_in, net.conv_precision(net.route(li, B)["tc"]))
        check(f"{tag} layer {li}", precision, act[li], ref, bound)
        if li == net.blocks[0]["first"] + net.blocks[0]["n"] - 1:
            check(f"{tag} fc_out", precision, fc_out,
                  *fc_ref(act[li].reshape(B, -1), net.p["fc.weight"], net.p["fc.bias"], net.fc_precision()))
    # fused head
    yf, capf = forward_eval(net, x, elide, dedup=False, fuse=True)
    fused = [li for li in range(n) if net.route(li, B)["fuse_head"]]
    if precision != "fp32" and B * net.V(n - 2) >= 64:
        assert fused == [n - 2], (tag, fused)
    if fused:
        li = fused[0]
        act_f = {k: capf["y"][k].reshape(B, net.V(k), -1) for k in range(n) if k != li}
        inp, block_in = layer_input(net, li, x, capf["fc_out"], act_f)
        y1, e1 = eval_layer(net, li, inp, block_in, precision)
        Lh = net.L32[net.layers[n - 1]["level"]]
        Wh, bh = net.p[f"cl.{n - 1}.weight"], net.p[f"cl.{n - 1}.bias"]
        ref = R.cheb_conv_fwd(y1, Lh, Wh, bh)
        bound = R.cheb_conv_fwd_bound(y1, Lh, Wh, bh, "fp32") + R.thin_head_fused_bound(y1, e1, Lh, Wh)
        check(f"{tag} fused head", precision, yf.reshape(ref.shape), ref, bound)
    return y, yf, act, fc_out


# ------------------------------------------------------------------------------------------- launches and coverage
def test_capture_leaves_the_launches_unchanged():
    """The capture copies are stream-ordered memcpys, not kernels; with no capture set the schedules issue the same
    launches before a capture was ever set and after it is cleared."""
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    net = Net("custom", "fp16x3", seed=3, open_relus=True)
    x, tgt = train_inputs(net, 3, seed=1)

    def counts():
        lib.p2m_launch_count_reset()
        forward_eval(net, x, 1, True, True, capture=False)
        ev = lib.p2m_launch_count()
        lib.p2m_launch_count_reset()
        forward_train_backward_no_capture(net, x, tgt)
        return ev, lib.p2m_launch_count()

    before = counts()
    forward_train_backward(net, x, tgt)
    after = counts()
    assert before == after and min(before) > 10, (before, after)


def forward_train_backward_no_capture(net, x, tgt):
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    n = net.n_layers
    sd = net.sd
    names = (["fc.weight", "fc.bias"] + [f"cl.{i}.weight" for i in range(n)] + [f"cl.{i}.bias" for i in range(n)]
             + [f"bn.{i}.weight" for i in range(n - 1)] + [f"bn.{i}.bias" for i in range(n - 1)])
    p = [cuda(sd[k]).requires_grad_(True) for k in names]
    buffers = ([cuda(sd[f"bn.{i}.running_mean"]) for i in range(n - 1)] + [None],
               [cuda(sd[f"bn.{i}.running_var"]) for i in range(n - 1)] + [None], [None] * n)
    y = _MeshNetFunction.apply(cuda(x).requires_grad_(True), net.hier, True, buffers, n, *p)
    (y - cuda(tgt)).abs().mean().backward()
    torch.cuda.synchronize()


def test_route_coverage_of_the_grid():
    """Over the configurations the tests above run at fp16x3, every route flag of p2m_debug_layer_route is observed both
    on and off, per role (forward, backward)."""
    seen = {}
    nets = {}
    for name, elide, B, need_dx in TRAIN_CASES + [(n_, e, B, True) for n_, e, B in EVAL_CASES]:
        net = nets.get(name) or nets.setdefault(name, Net(name, "fp16x3", seed=0, open_relus=True))
        for fuse in (False, True):
            net.hier.set_debug(0, elide_padding=elide, fuse_head=fuse)
            for li in range(net.n_layers):
                for k, v in net.route(li, B, need_dx).items():
                    seen.setdefault(k, set()).add(v)
    missing = {k: v for k, v in seen.items() if v != {False, True}}
    assert not missing and len(seen) == 9, missing
