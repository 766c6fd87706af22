"""The torch float64 references (tests/fp64_ref_torch.py) against their specification, tests/fp64_ref.py, on the CPU;
and the bound's teeth at the shape of the SMPL-size network's finest level.

1. Every ported reference and bound equals the numpy one to 1e-12 relative, on the layers of the three small nets
   (custom, mano_like, smpl_small) and on one mesh of the SMPL-size hierarchy's 12288-row level, with the meshes
   taken 1, 2 and all at a time (the batch-wide sums accumulated across chunks).  Bounds are non-negative sums and
   are compared element by element; signed references relative to their largest entry.
2. fp64_ref.emulate_cheb_conv on one mesh of the 12288-row level, 128 -> 128 at the network split: fp16x3 stays
   within the bound, one K-block's lo products dropped or single-pass fp16 do not.
3. One-signed fp32 accumulation over a dW chain of production length (one CTA adding the rows of ~187 tiles of 128):
   within the bound of dw_chain; the default sqrt(n) bound holds for round-to-nearest adds and not for a worst-case
   model whose every add truncates toward zero."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import fp64_ref as R
import fp64_ref_torch as T
from helpers import CASES, graph_from_fixture

TOL = 1e-12


def close(got, ref, what, signed=True):
    got = got.numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = float(np.abs(ref).max(initial=0.0)) if signed else np.abs(ref)
    err = np.abs(got - ref)
    assert np.all(err <= TOL * scale), (what, float((err / np.maximum(scale, 1e-300)).max()))


# ------------------------------------------------------------------------------------------------------------- layers
def small_layers(name):
    """(Laplacian, fin, fout) of every layer of one of the small nets."""
    if name == "custom":
        mats = graph_from_fixture("smpl_small")[0]
        levels = [next(m for m in mats if m.shape[0] == V) for V in (128, 64, 17)]
        plan = [(5, 32, 64), (64, 256), (256, 128, 256), (256, 64, 3)]
    else:
        from pose2mesh_release_b200.meshnet import channel_plan

        levels = list(graph_from_fixture(name)[0])
        del levels[-2]
        plan = channel_plan(5, 3, name == "mano_like")
    out, nb, nl = [], len(plan), len(levels)
    for b, chans in enumerate(plan):
        lvl = levels[0 if b == nb - 1 else nl - 1 - b]
        for fin, fout in zip(chans[:-1], chans[1:]):
            out.append((lvl, fin, fout))
    return out


def layer_data(V, B, fin, fout, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32).astype(np.float64)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout))).astype(np.float32).astype(np.float64)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32).astype(np.float64)
    dz = rng.standard_normal((B, V, fout)).astype(np.float32).astype(np.float64)
    # a per-mesh scale over orders of magnitude, like the weighted loss of the at-size GPU test
    dz *= 2.0 ** -np.arange(B)[:, None, None] * 8
    return x, W, b, dz


def check_conv(L, x, W, b, dz, chunk, tag):
    t = torch.from_numpy
    Lt = T.Lap(L)
    close(T.basis(t(x), Lt, chunk), R.basis(x, L), tag + " basis")
    close(T.cheb_conv_fwd(t(x), Lt, W, b, chunk), R.cheb_conv_fwd(x, L, W, b), tag + " fwd")
    for prec in R.SPLIT_TERM:
        for split in ("normalised", "network"):
            tg = f"{tag} {prec} {split}"
            close(T.cheb_conv_fwd_bound(t(x), Lt, W, b, prec, split, chunk),
                  R.cheb_conv_fwd_bound(x, L, W, b, prec, split), tg + " fwd bound", False)
            for chain in ((0, 1000) if prec != "fp32" and split == "network" else (0,)):
                got = T.cheb_conv_bwd_bound(t(x), Lt, W, t(dz), prec, split, chain, chunk)
                ref = R.cheb_conv_bwd_bound(x, L, W, dz, prec, split, chain)
                for k, g, r in zip(("dx", "dW", "db"), got, ref):
                    close(g, r, f"{tg} chain={chain} bwd bound {k}", False)
    # dX and dW at different precisions (a layer whose dW runs on the tensor cores and dX on the CUDA cores), with the
    # default dW bound alongside the chain's
    bdx, bdw, bdb, bdw0 = T.cheb_conv_bwd_bound(t(x), Lt, W, t(dz), "fp32", "network", 1000, chunk,
                                                precision_dw="fp16x3", with_default=True)
    close(bdx, R.cheb_conv_bwd_bound(x, L, W, dz, "fp32", "network")[0], tag + " mixed bwd bound dx", False)
    close(bdw, R.cheb_conv_bwd_bound(x, L, W, dz, "fp16x3", "network", 1000)[1], tag + " mixed bwd bound dW", False)
    close(bdw0, R.cheb_conv_bwd_bound(x, L, W, dz, "fp16x3", "network")[1], tag + " default bwd bound dW", False)
    close(bdb, R.cheb_conv_bwd_bound(x, L, W, dz, "fp16x3", "network")[2], tag + " mixed bwd bound db", False)
    for k, g, r in zip(("dx", "dW", "db"), T.cheb_conv_bwd(t(x), Lt, W, t(dz), chunk), R.cheb_conv_bwd(x, L, W, dz)):
        close(g, r, f"{tag} bwd {k}")
    y = R.cheb_conv_fwd(x, L, W, b)
    E = R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3", "network")
    Wh = np.abs(W[:3, :1]) * np.ones((3, 3 * W.shape[0]))        # a 3-wide head on this layer's output
    close(T.thin_head_fused_bound(t(y), t(E), Lt, Wh, chunk), R.thin_head_fused_bound(y, E, L, Wh),
          tag + " thin head bound", False)


def check_bn(z, g_a, gam, bet, rm, rv, chunk, tag):
    t = torch.from_numpy
    for k, g, r in zip(("y", "mean", "var", "rm", "rv"), T.bn_train_fwd(t(z), gam, bet, rm, rv, True, chunk=chunk),
                       R.bn_train_fwd(z, gam, bet, rm, rv, relu=True)):
        close(g, r, f"{tag} bn fwd {k}")
    E = np.abs(z) * 1e-6
    for e in (None, E):
        got = T.bn_train_fwd_bound(t(z), None if e is None else t(e), gam, bet, rm, rv, chunk=chunk)
        ref = R.bn_train_fwd_bound(z, np.zeros_like(z) if e is None else e, gam, bet, rm, rv)
        for k in ref:
            close(got[k], ref[k], f"{tag} bn fwd bound {k} E={e is not None}", False)
    mask = R.relu_mask(z.astype(np.float32), np.float32(1.0), np.float32(-0.2))
    for kw in (dict(relu=True), dict(relu=False), dict(mask=mask)):
        tkw = dict(kw, mask=t(kw["mask"])) if "mask" in kw else kw
        for k, g, r in zip(("g_z", "dgamma", "dbeta", "pre"), T.bn_train_bwd(t(z), t(g_a), gam, bet, chunk=chunk, **tkw),
                           R.bn_train_bwd(z, g_a, gam, bet, **kw)):
            close(g, r, f"{tag} bn bwd {k} {list(kw)}")
        for k, g, r in zip(("g_z", "dgamma", "dbeta"), T.bn_train_bwd_bound(t(z), t(g_a), gam, bet, chunk=chunk, **tkw),
                           R.bn_train_bwd_bound(z, g_a, gam, bet, **kw)):
            close(g, r, f"{tag} bn bwd bound {k} {list(kw)}", False)
    close(T.bn_eval_fwd(t(z), gam, bet, rm, rv, True, chunk=chunk), R.bn_eval_fwd(z, gam, bet, rm, rv, relu=True),
          tag + " bn eval")
    close(T.bn_eval_fwd_bound(t(z), t(E), gam, bet, rm, rv, bet * 0.5, chunk=chunk),
          R.bn_eval_fwd_bound(z, E, gam, bet, rm, rv, bet * 0.5), tag + " bn eval bound", False)
    close(T.col_sum_bound(t(g_a), chunk), R.col_sum_bound(g_a), tag + " col_sum_bound", False)


def check_glue(x, chunk, tag):
    t = torch.from_numpy
    fin = x.shape[-1]
    close(T.unpool(t(x)), R.unpool(x), tag + " unpool")
    close(T.unpool_t(t(x)), R.unpool_t(x), tag + " unpool_t")
    for other in (fin, 2 * fin, fin // 2, 3):
        close(T.channel_resample(t(x), other, chunk), R.channel_resample(x, other), f"{tag} resample {other}")
        close(T.channel_resample_t(t(x), other, chunk), R.channel_resample_t(x, other), f"{tag} resample_t {other}")
        close(T.channel_resample_bound(t(x), other, chunk), R.channel_resample_bound(x, other),
              f"{tag} resample bound {other}", False)
        close(T.channel_resample_t_bound(t(x), other, chunk), R.channel_resample_t_bound(x, other),
              f"{tag} resample_t bound {other}", False)


CHUNKS = [1, 2, None]


@pytest.mark.parametrize("chunk", CHUNKS, ids=lambda c: f"chunk={c or 'all'}")
@pytest.mark.parametrize("name", ["custom", "mano_like", "smpl_small"])
def test_small_net_layers_match_numpy(name, chunk):
    """Every layer of the net (3 meshes, per-mesh gradient scales 8 ... 2): the conv, its backward and every bound,
    the BatchNorm forward / backward and bounds with the ReLU's own mask, the glue of the blocks."""
    B = 3
    for li, (L, fin, fout) in enumerate(small_layers(name)):
        V = L.shape[0]
        x, W, b, dz = layer_data(V, B, fin, fout, seed=li)
        L32 = L.tocsr().astype(np.float32).astype(np.float64)
        tag = f"{name} layer {li} ({fin}->{fout} V={V}) chunk={chunk}"
        check_conv(L32, x, W, b, dz, chunk, tag)
        z = R.cheb_conv_fwd(x, L32, W, b)
        rng = np.random.default_rng(li)
        gam, bet = rng.random(fout) + 0.5, rng.standard_normal(fout) * 0.1
        rm, rv = rng.standard_normal(fout) * 0.1, rng.random(fout) + 0.5
        check_bn(z, dz, gam, bet, rm, rv, chunk, tag)
        if V % 2 == 0:
            check_glue(x, chunk, tag)


def test_fc_matches_the_network_test():
    import test_gpu_network_fp64 as N

    rng = np.random.default_rng(0)
    a0 = rng.standard_normal((5, 17 * 64)) * 2.0 ** -np.arange(5)[:, None]
    W, b = rng.standard_normal((96 * 64, 17 * 64)) * 0.03, rng.standard_normal(96 * 64) * 0.1
    for prec in ("fp32", "fp16x3"):
        ref, bound = N.fc_ref(a0, W, b, prec)
        got, gb = T.fc(torch.from_numpy(a0), W, b, prec)
        close(got, ref, "fc")
        close(gb, bound, "fc bound", False)


_SMPL = {}


def smpl_level0():
    """The SMPL-size hierarchy's finest Laplacian (12288 rows, 6890 connected), rebuilt by the graph oracle."""
    if not _SMPL:
        from oracle import graph_oracle as go

        n, seed, levels, _ = CASES["smpl_like"]
        face = go.synthetic_sphere_faces(n, seed)
        _, lap, _, _ = go.build_coarse_graphs(face, 17, go.H36M_SKELETON, go.H36M_FLIP_PAIRS, levels=levels)
        _SMPL["L0"] = sp.csr_matrix(lap[0]).astype(np.float32).astype(np.float64)
    return _SMPL["L0"]


def test_smpl_level0_mesh_matches_numpy():
    """One mesh of the 12288-row level, 128 -> 128 (the finest level's width in the SMPL plan), and two meshes of
    128 -> 64 at chunk 1."""
    L = smpl_level0()
    assert L.shape == (12288, 12288)
    for B, fin, fout, chunk in ((1, 128, 128, None), (2, 128, 64, 1)):
        x, W, b, dz = layer_data(L.shape[0], B, fin, fout, seed=fin + fout)
        tag = f"smpl level 0 B={B} {fin}->{fout}"
        check_conv(L, x, W, b, dz, chunk, tag)
        z = R.cheb_conv_fwd(x, L, W, b)
        rng = np.random.default_rng(1)
        gam, bet = rng.random(fout) + 0.5, np.full(fout, 6.0)
        check_bn(z, dz, gam, bet, np.zeros(fout), np.ones(fout), chunk, tag)


# ------------------------------------------------------------------------------------------------------- the teeth
def test_bound_tells_a_subtly_wrong_kernel_at_the_12288_row_level():
    """128 -> 128 on one mesh of the 12288-row level, network split (activations as they are, weights at 2^6), held to
    the torch bound: the fp16x3 arithmetic passes; one K-block's lo(T) * hi(W) products missing, or one fp16 product
    per pair, fail."""
    L = smpl_level0()
    x, W, b, _ = layer_data(L.shape[0], 1, 128, 128, seed=5)
    t = torch.from_numpy
    y64 = T.cheb_conv_fwd(t(x), L, W, b)
    bound = T.cheb_conv_fwd_bound(t(x), L, W, b, "fp16x3", "network")
    ok = T.bound_ratio(t(R.emulate_cheb_conv(x, L, W, b, "fp16x3", split="network")), y64, bound)
    assert ok <= 0.5, ok
    for kw in (dict(mode="fp16x3", drop_block=0), dict(mode="fp16")):
        r = T.bound_ratio(t(R.emulate_cheb_conv(x, L, W, b, split="network", **kw)), y64, bound)
        assert r > 1.0, (kw, r)


def _trunc32(v: np.ndarray) -> np.ndarray:
    """Round float64 values toward zero to fp32: a worst-case model of an accumulator whose every add loses its
    rounding error in one direction (not a measured property of the hardware)."""
    f = v.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def test_production_dw_chain_within_its_chain_bound():
    """A dW element accumulated by one CTA over the rows of its tiles is a sequential fp32 chain of one-signed terms
    (|dz| |T| over rows of one channel keeps a sign where dz does): at SMPL B = 256 on the 12288-row level, 24 576
    tiles of 128 rows over ~132 CTAs, ~187 tiles or ~24 000 adds per CTA.  Emulated for 256 elements at once, with
    round-to-nearest adds and under the worst-case model of adds truncated toward zero, the error stays within
    dw_chain's n u; the default bound of a grid of many CTAs (sqrt(3 R) u over the R = 3.1 M rows of the batch) holds
    for the rounded chain and not for the truncated one, which is why the at-size GPU test holds dW to the chain of
    the launch that ran."""
    rng = np.random.default_rng(0)
    rows, grid = 256 * 12288, 132
    tiles = 256 * 96
    n = -(-tiles // grid) * 128                                   # the rows one CTA adds
    terms = rng.random((n, 256)) + 0.25                           # one sign, one magnitude: the worst case for sqrt(n)
    exact = terms.sum(axis=0)
    rn = np.zeros(256, np.float32)
    rz = np.zeros(256, np.float32)
    for i in range(n):
        rn = (rn + terms[i].astype(np.float32)).astype(np.float32)
        rz = _trunc32(rz.astype(np.float64) + terms[i].astype(np.float32).astype(np.float64))
    chain = n + grid
    g_chain = chain * R.U32
    g_default = T.dw_gamma_default(rows, "fp32", 0) - R.LAMBDA * np.sqrt(3) * R.U32   # without the basis' deg term
    rel_rn = np.abs(rn - exact) / exact
    rel_rz = np.abs(rz - exact) / exact
    # the terms' own fp32 rounding is part of the kernel's input, not of the chain: at most u each
    assert rel_rn.max() <= g_chain + R.U32 and rel_rz.max() <= g_chain + R.U32, (rel_rn.max(), rel_rz.max(), g_chain)
    assert rel_rn.max() <= g_default, (rel_rn.max(), g_default)
    assert rel_rz.max() > g_default, (rel_rz.max(), g_default)
