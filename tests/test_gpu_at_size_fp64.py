"""MeshNet layer by layer against float64 at the sizes it is benchmarked at: SMPL B = 256 and MANO B = 1024.

test_gpu_network_fp64.py checks every layer of the schedules element-wise on small nets; here the same checks run on
the SMPL-size hierarchy (6890 vertices padded to 12288 rows, 21 layers) and the MANO-size one at the benchmark's
batches, where only the full size has: the dW chain of a CTA over ~187 tiles, the gradient operand's one power-of-two
scale over 3.1 M rows, 5398 padding rows per mesh in the BatchNorm statistics, the full-size reductions and the tile
patterns, halos and wide configurations of the big levels.  The float64 references are fp64_ref_torch (fp64_ref.py on
the device, chunked over meshes).

A step's tensors do not fit at once (one 128-wide fp32 activation of the 12288-row level is 1.6 GB), so the same step
runs once per layer with only that layer's tensors captured and what its checks read (its input, the block input of a
residual, the fc's tensors, the block's last g_a); every layer is checked from tensors of its own run, every check is
max |err| / bound <= 1 element-wise.  The loss weights mesh b by 2^-(b mod 17), so the gradient's single scale is set
by a few meshes while the rest sit up to 2^16 below it; mesh B - 1 repeats mesh 3 (input, target and weight), and their
rows are bitwise equal in every captured tensor: a tile's arithmetic does not depend on where the mesh sits.

dW is held to the larger of the default bound and n u of the chain of the launch that ran (conv log: tiles per CTA x
128 rows + grid; SIMT k_gemm_tn_atomic: TN_CHUNK + ceil(M / TN_CHUNK); the thin head: ceil(rows / grid) + grid);
the ratio against the default bound alone is reported.

Every run also asserts the path it took: each layer's route (p2m_debug_layer_route), and from the conv log each
layer's forward launches (columns per CTA, slices, ring slots, stages, single-pass fp16 exactly at fp16 and
fp16_mixed, the persistent grid, many tiles per CTA on the two finest levels), its dW launches and the fc's GEMM.
P2M_AT_SIZE_FP64_REPORT names a JSON report."""
import json
import os
import time

import numpy as np
import pytest
import torch

import fp64_ref as R
import fp64_ref_torch as T
import test_gpu_network_fp64 as N

pytestmark = pytest.mark.gpu

MEM_BUDGET = 40 * 2 ** 30      # peak device memory of the module (the GPUs are shared)
TN_CHUNK = 4096                # kernels_simt.cu: rows per block of k_gemm_tn_atomic
DW_TILE_ROWS = 128
ROWS_PER_CHUNK = 1 << 17       # rows of one chunk of the float64 references

_REPORT = {"worst": {}, "dw_vs_default": {}, "near_zero_relus": {}, "routes": {}, "tiles_per_cta": {}}


@pytest.fixture(scope="module", autouse=True)
def _report():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    _REPORT["peak_memory_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    _REPORT["wall_s"] = time.time() - t0
    out = os.environ.get("P2M_AT_SIZE_FP64_REPORT")
    if out:
        with open(out, "w") as f:
            json.dump(_REPORT, f, indent=1)


def dev():
    return torch.device("cuda:0")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def qclass(what):
    return what.rsplit(" ", 1)[-1]


def check(case, what, got, ref, bound):
    r = T.bound_ratio(got, ref, bound)
    w = _REPORT["worst"].setdefault(case, {})
    q = qclass(what)
    if r > w.get(q, [0.0])[0]:
        w[q] = [r, what]
    assert r <= 1.0, f"{case} {what}: max |err| / bound = {r:.3g}"


def chunk_of(net, li):
    return max(1, ROWS_PER_CHUNK // net.V(li))


# ----------------------------------------------------------------------------------------------------------- running
def inputs(net, B, seed):
    """x, targets and per-mesh loss weights 2^-(b mod 17); mesh B - 1 a copy of mesh 3."""
    x, tgt = N.train_inputs(net, B, seed)
    w = 2.0 ** -(np.arange(B) % 17)
    x[B - 1], tgt[B - 1], w[B - 1] = x[3], tgt[3], w[3]
    return x, tgt, w.astype(np.float32)


def params(net):
    n = net.n_layers
    names = (["fc.weight", "fc.bias"] + [f"cl.{i}.weight" for i in range(n)] + [f"cl.{i}.bias" for i in range(n)]
             + [f"bn.{i}.weight" for i in range(n - 1)] + [f"bn.{i}.bias" for i in range(n - 1)])
    return names


def alloc(net, B, want):
    """Capture buffers for `want` (name -> set of layers; fc_out / fc_dx -> True), None elsewhere."""
    cap = {}
    for name, sel in want.items():
        if name in ("fc_out", "fc_dx"):
            n = net.levels[-2].shape[0] * net.plan[1][0] if name == "fc_out" else net.levels[-1].shape[0] * net.plan[0][-1]
            cap[name] = torch.full((B, n), float("nan"), device=dev())
            continue
        f = "fin" if name == "dx" else "fout"
        cap[name] = [torch.full((B, net.V(li) // (2 if name == "dx" and net.in_unpool(li) else 1), L[f]), float("nan"),
                                device=dev()) if li in sel else None for li, L in enumerate(net.layers)]
    return cap


def train_step(net, x, tgt, w, want, need_dx=True):
    """One train-mode forward + weighted L1 + backward from the state dict with `want` captured.
    Returns (cap, grads, buffers, y, conv log) on the device."""
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    n, sd = net.n_layers, net.sd
    p = {k: N.cuda(v).requires_grad_(True) for k, v in sd.items() if "running" not in k and "num_batches" not in k}
    buf = {k: N.cuda(v) if v.is_floating_point() else v.to(dev()) for k, v in sd.items()
           if "running" in k or "num_batches" in k}
    buffers = ([buf[f"bn.{i}.running_mean"] for i in range(n - 1)] + [None],
               [buf[f"bn.{i}.running_var"] for i in range(n - 1)] + [None],
               [buf[f"bn.{i}.num_batches_tracked"] for i in range(n - 1)] + [None])
    cap = alloc(net, x.shape[0], want)
    net.hier.set_capture(0, cap)
    _lib.conv_log(reset=True)
    try:
        xg = N.cuda(x).requires_grad_(need_dx)
        y = _MeshNetFunction.apply(xg, net.hier, True, buffers, n, *[p[k] for k in params(net)])
        wt = N.cuda(w)[:, None, None]
        (wt * (y - N.cuda(tgt)).abs()).mean().backward()
        torch.cuda.synchronize()
    finally:
        net.hier.set_capture(0, None)
    log = _lib.conv_log(reset=True)
    assert net.hier.kernel_status(0) == 0
    grads = {k: p[k].grad for k in params(net)}
    if need_dx and "dx" in want and 0 in want["dx"]:
        assert torch.equal(xg.grad, cap["dx"][0])
    return cap, grads, buf, y.detach(), log


def block_of(net, li):
    return net.blocks[net.layers[li]["block"]]


def last_of(blk):
    return blk["first"] + blk["n"] - 1


def train_window(net, li, need_dx):
    """What the checks of layer li read: its own tensors, its input, the block input, the fc's tensors."""
    L, blk, b = net.layers[li], block_of(net, li), net.layers[li]["block"]
    want = {"g_a": {li}, "g_z": {li}, "a": set(), "z": set()}
    if L["bn"]:
        want["z"].add(li)
        want["a"].add(li)
    if not (li == 0 and not need_dx):
        want["dx"] = {li}
    if L["j"] > 0:
        want["a"].add(li - 1)
    if b >= 2:
        want["a"].add(last_of(net.blocks[b - 1]))
    if b == 1 or li == last_of(net.blocks[0]):
        want["fc_out"] = True
    if L["j"] == 0 and blk["res"]:
        want["g_a"].add(last_of(blk))
    if li == blk["first"] and b == 1:
        want["fc_dx"] = True
        want["g_a"].add(li - 1)
        want["a"].add(li - 1)
    return want


def act_view(net, cap, B):
    return {k: t.reshape(B, net.V(k), -1) for k, t in enumerate(cap["a"]) if t is not None}


FC = 32                        # cheb_umma.cu: features per chunk; launch_umma_dw launches once per chunk and 64 columns


def conv_path(net, level, fin, fout):
    import ctypes as C

    from pose2mesh_release_b200 import _lib

    out = (C.c_int32 * 9)()
    _lib.check(_lib.load().p2m_debug_conv_path(net.hier.handle(0), level, fin, fout, out), "p2m_debug_conv_path")
    return tuple(out)


def dw_chains(net, B, log, need_dx):
    """layer -> (the fp32 chain of its dW, its dw launches).  On the tensor cores launch_umma_dw issues, per layer in
    the backward's order, ceil(plain / 64) x gathered / FC launches of one grid over the level's tiles (gathered: the
    side whose basis is built, dz on the dz-basis route, else x); each CTA adds the rows of its tiles in registers and
    then once atomically: tiles per CTA x 128 + grid.  SIMT: k_gemm_tn_atomic (TN_CHUNK rows per block, then one
    atomic add per block) or the thin head's k_thin_bwd_main, whose grid = min(ceil(rows / 128), 4 SMs) CTAs walk the
    128-row tiles with 16 row slots: a thread adds 8 rows of each of its tiles, then the 16 slots meet in shared-memory
    atomics and the CTAs in global ones, ceil(tiles / grid) x 8 + 16 + grid adds."""
    dws = [e for e in log if e["kind"] == "dw"]
    out, i = {}, 0
    for li in range(net.n_layers - 1, -1, -1):
        r = net.route(li, B, need_dx)
        L = net.layers[li]
        rows = B * net.V(li)
        if r["tc_dw"] or r["dw_dz_basis"]:
            gathered, plain = (L["fout"], L["fin"]) if r["dw_dz_basis"] else (L["fin"], L["fout"])
            k = -(-plain // 64) * (gathered // FC)
            mine = dws[i:i + k]
            i += k
            assert len(mine) == k and len({(e["grid_x"], e["n_tiles"]) for e in mine}) == 1, (li, mine)
            e = mine[0]
            assert e["n_tiles"] % B == 0 and e["grid_x"] == min(e["n_tiles"], sms()), (li, e)
            out[li] = (e["tiles_per_cta"] * DW_TILE_ROWS + e["grid_x"], mine)
        elif r["thin"] and li == net.n_layers - 1:
            tiles = -(-rows // 128)
            grid = min(tiles, 4 * sms())
            out[li] = (-(-tiles // grid) * (128 // 16) + 16 + grid, [])
        else:
            out[li] = (TN_CHUNK + -(-rows // TN_CHUNK), [])
    assert i == len(dws), ("dw launches the routes do not account for", len(dws) - i)
    return out


FWD_KEYS = ("tc", "elide", "fuse_head")


def conv_cfg_named(fin, fout):
    """(columns per CTA, column slices) of the forward conv a fin -> fout layer is named after: the 64 x 256
    configuration for 256 -> 256, 128 x 64 for 64-wide outputs, 64 x 128 otherwise (two slices of 128 for a 256-wide
    output)."""
    if fin == fout == 256:
        return 256, 1
    if fout == 64:
        return 64, 1
    return 128, fout // 128


# On the SMPL hierarchy's elided levels (12288 and 6144 rows), by (fin, fout) at both tensor-core precisions:
# (ring slots, X / T1 stages) of the connected rows' conv over real_tiles (the full-tile p2m_debug_conv_tiling does
# not describe that tile set), and (columns, slices, ring slots, stages) of the isolated rows' plain GEMM, over all of
# them or over the class representatives alike
ELIDED_CFG = {(128, 128): (6, 2), (128, 64): (3, 2)}
ISO_CFG = {(128, 128): (128, 1, 6, 2), (128, 64): (64, 1, 3, 2)}


def conv_tiling(net, level, fin, fout):
    import ctypes as C

    from pose2mesh_release_b200 import _lib

    out = (C.c_int32 * 3)()
    _lib.check(_lib.load().p2m_debug_conv_tiling(net.hier.handle(0), level, fin, fout, out), "p2m_debug_conv_tiling")
    return tuple(out)


def forward_launches(net, case, B, log, train):
    """The tensor-core launches of the forward, per layer in schedule order (a conv of the layer's tiles, then on an
    elided level the isolated rows' plain GEMM; the fc's GEMM after block 0), each asserted to be the instantiation
    the layer is named after: columns per CTA and slices by conv_cfg_named, ring slots and stages by
    p2m_debug_conv_tiling (ELIDED_CFG on elided levels), single-pass fp16 exactly at the single-pass precisions, the
    persistent grid min(tiles, SMs / slices) and, on the two finest levels, many tiles per CTA.  Returns the launches
    after the forward's (the backward's), whose convs and dWs carry the same single-pass bit."""
    f16 = int(net.precision in ("fp16", "fp16_mixed"))
    tc_prec = net.precision != "fp32"
    rep = _REPORT["tiles_per_cta"].setdefault(case + (" forward" if train else " eval"), {})
    i = 0
    for li in range(net.n_layers):
        L = net.layers[li]
        r = net.route(li, B)
        if r["tc"]:
            k = 1 + int(r["elide"])
            mine = log[i:i + k]
            i += k
            assert [(e["kind"], e["mode"], e["f16"]) for e in mine] == [("conv", 1, f16), ("conv", 0, f16)][:k], \
                (case, li, mine)
            e = mine[0]
            nc, slices = conv_cfg_named(L["fin"], L["fout"])
            key = (L["fin"], L["fout"])
            if r["elide"]:
                ns_xs = ELIDED_CFG[key]
            else:
                til = conv_tiling(net, L["level"], L["fin"], L["fout"])
                assert til[0] == nc, (case, li, til)
                ns_xs = til[1:]
            got = (e["nc"], e["grid_y"], e["ns"], e["xs"])
            rep[str(li)] = dict(cfg=got, tiles_per_cta=e["tiles_per_cta"], grid_x=e["grid_x"], n_tiles=e["n_tiles"],
                                iso=[(x["nc"], x["grid_y"], x["ns"], x["xs"], x["tiles_per_cta"]) for x in mine[1:]])
            assert got == (nc, slices) + tuple(ns_xs), (case, li, got, ns_xs)
            for x in mine:
                assert x["n_tiles"] % B == 0 and x["grid_x"] == min(x["n_tiles"], max(1, sms() // x["grid_y"])), \
                    (case, li, x)
            if r["elide"]:
                iso = (mine[1]["nc"], mine[1]["grid_y"], mine[1]["ns"], mine[1]["xs"])
                assert iso == ISO_CFG[key], (case, li, iso)
            if net.V(li) >= 6144:   # the production regime: every CTA runs many tiles of the two finest levels
                assert e["tiles_per_cta"] >= 16, (case, li, e)
        if li == last_of(net.blocks[0]) and tc_prec:
            e = log[i]
            i += 1
            assert e["kind"] == "gemm" and e["f16"] == 0, (case, "fc", e)
            rep["fc"] = dict(cfg=(e["nc"], e["grid_y"], e["ns"], e["xs"]), grid_x=e["grid_x"], n_tiles=e["n_tiles"])
    if not train:
        assert i == len(log), (case, "launches the eval schedule does not account for", log[i:])
    assert all(e["f16"] == f16 for e in log[i:] if e["kind"] in ("conv", "dw")), (case, log[i:])
    return log[i:]


def expected_route(net, name, precision, li):
    """The paths each layer takes at these sizes: the joint level's 5 -> 32 and the fp32 precision on the CUDA
    cores, the 64 -> 128 after the fc without backward-data on the tensor cores (its dx is the fc's input), every
    other tensor-core layer with dX as a conv on dz and dW on the basis of dz; the padding rows of the SMPL
    hierarchy's two finest levels elided; the layer in front of the 64 -> 3 head fused with it in eval; the head on the thin kernels."""
    n = net.n_layers
    if li == n - 1:
        return {"thin"}
    if precision == "fp32" or li == 0:
        return set()
    if li == 1:
        return {"tc", "tc_dw"}
    s = {"tc", "tc_dw", "dw_dz_basis", "tc_dx"}
    if name == "smpl_like" and net.layers[li]["level"] <= 1:   # 5398 of 12288 and 2503 of 6144 rows isolated
        s |= {"elide", "dx_elide"}
    if li == n - 2:
        s.add("fuse_head")
    return s


def mirrored(case, what, t, B):
    """Rows of mesh 3 and mesh B - 1 (same input, target and loss weight) bitwise equal."""
    assert torch.equal(t[3], t[B - 1]), f"{case} {what}: mesh 3 and mesh {B - 1} differ"


def relu_mask(net, li, z, a, g_a, g_z, pre, E_y, case, blk):
    """The ReLU's branches as the device took them.  Where the float64 pre-activation is farther than its forward
    bound from zero they are pre > 0; within it, a > 0 where a is the activation itself, and where the block adds a
    residual to it, the branch whose g_z the device's g_z is nearer to.  Returns (mask, count of near-zero)."""
    mask = pre > 0
    near = pre.abs() <= E_y
    cnt = int(near.sum())
    if cnt == 0:
        return mask, 0
    L = net.layers[li]
    if not (L["end"] and blk["res"]):
        mask = torch.where(near, a > 0, mask)
    else:
        gm = net.p[f"bn.{li}.weight"]
        ch = chunk_of(net, li)
        for _ in range(2):   # the device's g_z against both branches, with the means of the current mask
            gz, _, _, _ = T.bn_train_bwd(z, g_a, gm, net.p[f"bn.{li}.bias"], mask=mask, chunk=ch)
            alt = gz + torch.where(mask, -1.0, 1.0) * (torch.as_tensor(gm, device=z.device)
                                                       / torch.sqrt(z.double().var(dim=(0, 1), unbiased=False) + R.BN_EPS)
                                                       * g_a.double())
            flip = near & ((g_z.double() - alt).abs() < (g_z.double() - gz).abs())
            if not bool(flip.any()):
                break
            mask = torch.where(flip, ~mask, mask)
    return mask, cnt


def check_train_layer(net, case, li, x, y, cap, grads, bufs, chain, need_dx):
    """test_gpu_network_fp64.check_train for layer li, in torch on the device, from the tensors of its own run."""
    B = x.shape[0]
    L, blk = net.layers[li], block_of(net, li)
    r = net.route(li, B, need_dx)
    ch = chunk_of(net, li)
    a = act_view(net, cap, B)
    xt = torch.as_tensor(x, device=dev())
    fc_out = cap.get("fc_out")
    inp, block_in = N.layer_input(net, li, xt, fc_out, a, ref=T)
    Lm = net.lap[L["level"]]
    W, bias = net.p[f"cl.{li}.weight"], net.p[f"cl.{li}.bias"]
    t = f"layer {li} ({L['fin']}->{L['fout']} V={net.V(li)})"
    z64 = T.cheb_conv_fwd(inp, Lm, W, bias, ch)
    E = T.cheb_conv_fwd_bound(inp, Lm, W, bias, net.conv_precision(r["tc"]), "network", ch)
    g_a = cap["g_a"][li].reshape(B, net.V(li), -1)
    g_z = cap["g_z"][li].reshape(g_a.shape)
    mirrored(case, t + " g_z", g_z, B)
    if not L["bn"]:
        check(case, t + " y", y.reshape(z64.shape), z64, E)
        del z64, E
        assert torch.equal(g_z, g_a), t
    else:
        z = cap["z"][li].reshape(z64.shape)
        mirrored(case, t + " z", z, B)
        mirrored(case, t + " a", a[li], B)
        check(case, t + " z", z, z64, E)
        del z64, E
        g, be = net.p[f"bn.{li}.weight"], net.p[f"bn.{li}.bias"]
        rm, rv = net.p[f"bn.{li}.running_mean"], net.p[f"bn.{li}.running_var"]
        y64, _, _, rm64, rv64 = T.bn_train_fwd(z, g, be, rm, rv, relu=True, chunk=ch)
        bd = T.bn_train_fwd_bound(z, None, g, be, rm, rv, chunk=ch)
        res, eres = N.residual(net, li, block_in, ref=T)
        bound = bd["y"] + eres
        y64 += res
        bound += R.U32 * y64.abs()
        check(case, t + " a", a[li], y64, bound)
        del y64, bound, res, eres
        check(case, t + " running_mean", bufs[f"bn.{li}.running_mean"], rm64, bd["rm"])
        check(case, t + " running_var", bufs[f"bn.{li}.running_var"], rv64, bd["rv"])
        if li == last_of(net.blocks[0]):
            check(case, "fc_out", fc_out,
                  *T.fc(a[li].reshape(B, -1), net.p["fc.weight"], net.p["fc.bias"], net.fc_precision()))
        # backward of the BatchNorm: the ReLU's branches as the device took them
        gz64, dg64, db64, pre = T.bn_train_bwd(z, g_a, g, be, relu=True, chunk=ch)
        del gz64
        mask, near = relu_mask(net, li, z, a[li], g_a, g_z, pre, bd["y"], case, blk)
        _REPORT["near_zero_relus"].setdefault(case, {})[str(li)] = near
        del pre, bd
        gz64, dg64, db64, _ = T.bn_train_bwd(z, g_a, g, be, mask=mask, chunk=ch)
        bz, bg, bb = T.bn_train_bwd_bound(z, g_a, g, be, mask=mask, chunk=ch)
        check(case, t + " g_z", g_z, gz64, bz)
        check(case, t + " dgamma", grads[f"bn.{li}.weight"], dg64, bg)
        check(case, t + " dbeta", grads[f"bn.{li}.bias"], db64, bb)
        del gz64, bz, mask
        assert int(torch.count_nonzero(grads[f"cl.{li}.bias"])) == 0, t
    on_dw = r["tc_dw"] or r["dw_dz_basis"]
    on_dx = r["tc_dx"] or r["tc_dt"]
    want_dx = not (li == 0 and not need_dx)
    dx64, dW64, db64 = T.cheb_conv_bwd(inp, Lm, W, g_z, ch)
    bdx, bdw, _, bdw0 = T.cheb_conv_bwd_bound(inp, Lm, W, g_z, net.conv_precision(on_dx), "network", chain, ch,
                                              precision_dw=net.conv_precision(on_dw), with_default=True)
    del inp
    dW = grads[f"cl.{li}.weight"]
    _REPORT["dw_vs_default"].setdefault(case, {})[str(li)] = T.bound_ratio(dW, dW64, bdw0)
    check(case, t + " dW", dW, dW64, bdw)
    if not L["bn"]:
        check(case, t + " db", grads[f"cl.{li}.bias"], db64, T.col_sum_bound(g_z, ch))
    del dW64, bdw0, bdw
    if not want_dx:
        return
    if L["j"] == 0 and blk["res"]:
        g_res = cap["g_a"][last_of(blk)].reshape(B, net.V(li), -1)
        rt = T.channel_resample_t(g_res, L["fin"], ch)
        bdx += T.channel_resample_t_bound(g_res, L["fin"], ch) + R.U32 * (dx64.abs() + rt.abs())
        dx64 += rt
        del rt
    if net.in_unpool(li):
        dx64, bdx = T.unpool_t(dx64), T.unpool_t(bdx)
        bdx += R.U32 * dx64.abs()
    dx = cap["dx"][li].reshape(dx64.shape)
    mirrored(case, t + " dx", dx, B)
    check(case, t + " dx", dx, dx64, bdx)
    del dx64, bdx
    if li == blk["first"] and L["block"] == 1:    # the fc backward, from the gradient it read
        gf = dx.reshape(B, -1).double()
        a0 = a[last_of(net.blocks[0])].reshape(B, -1).double()
        Wf = torch.as_tensor(net.p["fc.weight"], device=dev())
        g_dw = R.gamma(B, "fp32") + B.bit_length() * R.U32
        check(case, "fc dW", grads["fc.weight"], gf.T @ a0, g_dw * (gf.abs().T @ a0.abs()))
        check(case, "fc db", grads["fc.bias"][None], gf.sum(dim=0)[None], T.col_sum_bound(gf)[None])
        check(case, "fc dx", cap["fc_dx"], gf @ Wf, R.gamma(Wf.shape[0], "fp32") * (gf.abs() @ Wf.abs()))
        assert torch.equal(cap["fc_dx"].reshape(B, -1), cap["g_a"][li - 1].reshape(B, -1)), case


def at_size_net(name, precision, seed, open_relus):
    net = N.Net(name, precision, seed=seed, open_relus=open_relus)
    net.lap = [T.Lap(m, dev()) for m in net.L32]
    return net


def run_train_case(name, B, precision, need_dx=True):
    case = f"{name} B={B} {precision} train"
    net = at_size_net(name, precision, seed=B, open_relus=True)
    x, tgt, w = inputs(net, B, seed=B + 1)
    routes = {li: {k for k, v in net.route(li, B, need_dx).items() if v} for li in range(net.n_layers)}
    _REPORT["routes"][case] = {str(li): sorted(r) for li, r in routes.items()}
    for li, r in routes.items():
        assert r == expected_route(net, name, precision, li), (case, li, sorted(r))
    for li in range(net.n_layers - 1, -1, -1):
        cap, grads, bufs, y, log = train_step(net, x, tgt, w, train_window(net, li, need_dx), need_dx)
        bwd_log = forward_launches(net, case, B, log, train=True)
        chain, mine = dw_chains(net, B, bwd_log, need_dx)[li]
        if mine:
            # k_cheb_dw_umma: 64 plain-side channels per launch, DW_NS = 3 ring slots, the level's X stages
            xs = conv_path(net, net.layers[li]["level"], net.layers[li]["fin"], net.layers[li]["fout"])[3]
            assert xs == 2 and {(x["nc"], x["ns"], x["xs"]) for x in mine} == {(64, 3, xs)}, (case, li, mine)
            e = mine[0]
            _REPORT["tiles_per_cta"].setdefault(case, {})[str(li)] = dict(
                tiles_per_cta=e["tiles_per_cta"], grid_x=e["grid_x"], n_tiles=e["n_tiles"], chain=chain,
                instantiations=sorted({(x["nc"], x["ns"], x["xs"]) for x in mine}))
            if net.layers[li]["level"] == 0:   # the production regime: every CTA runs many tiles of the finest level
                assert e["tiles_per_cta"] >= 64, (case, li, e)
        check_train_layer(net, case, li, x, y, cap, grads, bufs, chain, need_dx)
        del cap, grads, bufs, y
        torch.cuda.empty_cache()
    assert torch.cuda.max_memory_allocated() <= MEM_BUDGET, torch.cuda.max_memory_allocated() / 2 ** 30
    return net


def test_smpl_b256_train_fp16x3():
    run_train_case("smpl_like", 256, "fp16x3")


@pytest.mark.parametrize("precision", ["fp16x3", "fp32"])
def test_mano_b1024_train(precision):
    run_train_case("mano_like", 1024, precision)


# -------------------------------------------------------------------------------------------------------------- eval
def eval_run(net, x, dedup, fuse, want, check_log=None):
    """One eval forward (elision 1) with `want` captured; check_log (the case's name): its tensor-core launches are
    asserted layer by layer (forward_launches)."""
    from pose2mesh_release_b200 import _lib
    from pose2mesh_release_b200.meshnet import _MeshNetFunction

    B, n, sd = x.shape[0], net.n_layers, net.sd
    net.hier.set_debug(0, elide_padding=1, dedup_padding=dedup, fuse_head=fuse)
    prm = [N.cuda(sd[k]) for k in params(net)]
    buffers = ([N.cuda(sd[f"bn.{i}.running_mean"]) for i in range(n - 1)] + [None],
               [N.cuda(sd[f"bn.{i}.running_var"]) for i in range(n - 1)] + [None], [None] * n)
    cap = alloc(net, B, want) if want else None
    if cap:
        net.hier.set_capture(0, cap)
    _lib.conv_log(reset=True)
    try:
        with torch.no_grad():
            y = _MeshNetFunction.apply(N.cuda(x), net.hier, False, buffers, n, *prm)
        torch.cuda.synchronize()
    finally:
        net.hier.set_capture(0, None)
        net.hier.set_debug(0, elide_padding=1, dedup_padding=True, fuse_head=True)
    log = _lib.conv_log(reset=True)
    assert net.hier.kernel_status(0) == 0
    if check_log:
        forward_launches(net, check_log, B, log, train=False)
    return y, cap


def eval_window(net, li):
    b = net.layers[li]["block"]
    want = {"y": {li}}
    if net.layers[li]["j"] > 0:
        want["y"].add(li - 1)
    if b >= 2:
        want["y"].add(last_of(net.blocks[b - 1]))
    if b <= 1:
        want["fc_out"] = True
    return want


def eval_layer(net, li, inp, block_in, on_tc, ch):
    L = net.layers[li]
    W, bias = net.p[f"cl.{li}.weight"], net.p[f"cl.{li}.bias"]
    Lm = net.lap[L["level"]]
    z64 = T.cheb_conv_fwd(inp, Lm, W, bias, ch)
    E = T.cheb_conv_fwd_bound(inp, Lm, W, bias, net.conv_precision(on_tc), "network", ch)
    if not L["bn"]:
        return z64, E
    g, be = net.p[f"bn.{li}.weight"], net.p[f"bn.{li}.bias"]
    rm, rv = net.p[f"bn.{li}.running_mean"], net.p[f"bn.{li}.running_var"]
    bound = T.bn_eval_fwd_bound(z64, E, g, be, rm, rv, bias, chunk=ch)
    del E
    y64 = T.bn_eval_fwd(z64, g, be, rm, rv, relu=True, chunk=ch)
    del z64
    res, eres = N.residual(net, li, block_in, ref=T)
    y64 += res
    bound += eres + R.U32 * y64.abs()
    return y64, bound


def run_eval_case(net, name, case, B, fused_check):
    x, _, _ = inputs(net, B, seed=B + 2)
    xt = torch.as_tensor(x, device=dev())
    n = net.n_layers
    for li in range(n):
        got = {k for k in FWD_KEYS if net.route(li, B)[k]}
        assert got == {k for k in expected_route(net, name, net.precision, li) if k in FWD_KEYS}, (case, li, got)
    y_off, _ = eval_run(net, x, dedup=False, fuse=False, want=None, check_log=case)
    for li in range(n):
        y, cap = eval_run(net, x, dedup=False, fuse=False, want=eval_window(net, li), check_log=case)
        assert torch.equal(y, y_off), f"{case}: two eval runs differ"
        act = {k: t.reshape(B, net.V(k), -1) for k, t in enumerate(cap["y"]) if t is not None}
        inp, block_in = N.layer_input(net, li, xt, cap.get("fc_out"), act, ref=T)
        ch = chunk_of(net, li)
        ref, bound = eval_layer(net, li, inp, block_in, net.route(li, B)["tc"], ch)
        del inp, block_in
        mirrored(case, f"layer {li} y", act[li], B)
        check(case, f"layer {li} y", act[li], ref, bound)
        del ref, bound
        if li == last_of(net.blocks[0]):
            check(case, "fc_out", cap["fc_out"],
                  *T.fc(act[li].reshape(B, -1), net.p["fc.weight"], net.p["fc.bias"], net.fc_precision()))
        del cap, act
        torch.cuda.empty_cache()
    y_on, _ = eval_run(net, x, dedup=False, fuse=True, want=None, check_log=case + " fused")
    if fused_check:
        fused = [li for li in range(n) if net.route(li, B)["fuse_head"]]
        assert fused == [n - 2], (case, fused)
        li = n - 2
        want = {"y": {li - 1, last_of(net.blocks[net.layers[li]["block"] - 1])}}
        yf, capf = eval_run(net, x, dedup=False, fuse=True, want=want)
        assert torch.equal(yf, y_on)
        act = {k: t.reshape(B, net.V(k), -1) for k, t in enumerate(capf["y"]) if t is not None}
        inp, block_in = N.layer_input(net, li, xt, None, act, ref=T)
        ch = chunk_of(net, li)
        y1, e1 = eval_layer(net, li, inp, block_in, True, ch)
        del inp, block_in
        Lh = net.lap[net.layers[n - 1]["level"]]
        Wh, bh = net.p[f"cl.{n - 1}.weight"], net.p[f"cl.{n - 1}.bias"]
        ref = T.cheb_conv_fwd(y1, Lh, Wh, bh, ch)
        bound = T.cheb_conv_fwd_bound(y1, Lh, Wh, bh, "fp32", "normalised", ch)
        bound += T.thin_head_fused_bound(y1, e1, Lh, Wh, ch)
        del y1, e1
        check(case, "fused head y", yf.reshape(ref.shape), ref, bound)
    for fuse, yo in ((False, y_off), (True, y_on)):
        yd, _ = eval_run(net, x, dedup=True, fuse=fuse, want=None, check_log=f"{case} dedup fuse={fuse}")
        assert torch.equal(yd, yo), (case, "dedup", fuse)
    assert torch.cuda.max_memory_allocated() <= MEM_BUDGET


def test_smpl_b256_eval_fp16x3():
    net = at_size_net("smpl_like", "fp16x3", seed=3, open_relus=False)
    run_eval_case(net, "smpl_like", "smpl_like B=256 fp16x3 eval", 256, True)


def test_smpl_b256_eval_fp16():
    net = at_size_net("smpl_like", "fp16", seed=4, open_relus=False)
    run_eval_case(net, "smpl_like", "smpl_like B=256 fp16 eval", 256, False)
