"""CPU checks of the float64 references (tests/fp64_ref.py) and the graph families (tests/graphs.py) the GPU kernel
tests rely on: the element-wise bound accepts the fp16x3 arithmetic and rejects anything weaker, and every family
has the structure its name claims."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import fp64_ref as R
import graphs as G


def _layer(fin, fout, seed=0):
    L = G.get("band8")
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((1, L.shape[0], fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2 / (3 * fin + fout))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    return L, x, W, b


TEETH_SHAPES = [(32, 64), (96, 64), (160, 128), (256, 64)]


@pytest.mark.parametrize("fin,fout", TEETH_SHAPES)
def test_bound_accepts_fp16x3_and_rejects_weaker_arithmetic(fin, fout):
    L, x, W, b = _layer(fin, fout)
    y64 = R.cheb_conv_fwd(x, L, W, b)
    bound = R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3")
    ok = R.bound_ratio(R.emulate_cheb_conv(x, L, W, b, "fp16x3"), y64, bound)
    assert ok <= 0.25, ok                         # fp16x3 passes with margin for the hardware's accumulator
    for mode in ("fp16", "tf32"):                 # one fp16 product, or TF32 operands: ~2^-11 per product
        r = R.bound_ratio(R.emulate_cheb_conv(x, L, W, b, mode), y64, bound)
        assert r > 1.0, (mode, r)
    # the lo(T) * hi(W) products of ONE K-block (32 of the 3 Fin columns) missing; at Fin = 256 that is 1/24 of the
    # reduction and below the accumulation allowance sqrt(3K) u of 768-long sums
    if fin > 160:
        return
    r = R.bound_ratio(R.emulate_cheb_conv(x, L, W, b, "fp16x3", drop_block=0), y64, bound)
    assert r > 1.0, ("drop lo*Whi of block 0", r)


def test_bound_rejects_an_unscaled_split_of_small_inputs():
    """The floor scales with the input: an fp16 split of x * 2^-16 without a power-of-two range normalisation loses
    the lo parts to fp16's subnormals, and the bound must see it."""
    L, x, W, b = _layer(32, 64)
    x = x * np.float32(2.0 ** -16)
    y64 = R.cheb_conv_fwd(x, L, W, None)
    bound = R.cheb_conv_fwd_bound(x, L, W, None, "fp16x3")
    assert R.bound_ratio(R.emulate_cheb_conv(x, L, W, None, "fp16x3"), y64, bound) <= 0.25
    T = R._flat(R.basis(x, L)).astype(np.float32).astype(np.float64)
    Wp = W.astype(np.float64)
    th, tl = R._f16_split(T)
    wh, wl = R._f16_split(Wp * 64)
    y_unscaled = ((th @ wh.T) + (tl @ wh.T) + (th @ wl.T)) / 64
    assert R.bound_ratio(y_unscaled.reshape(y64.shape), y64, bound) > 1.0


def test_dense_gemm_bound_needs_range_normalised_activations():
    """PoseNet's H x H GEMM (K = 1024) on ReLU activations of scale 2^e, held to posenet_forward's per-GEMM bound: the
    fp16 split of the activations scaled into [2^9, 2^10) by a power of two meets it at every scale; split as they
    are, their lo parts fall into fp16's subnormals at small scales and the hi parts overflow at large ones."""
    rng = np.random.default_rng(3)
    K, n = 1024, 64
    W = ((rng.random((n, K)) * 2 - 1) / np.sqrt(K)).astype(np.float32).astype(np.float64)
    wh, wl = R._f16_split(W * 64)
    act = np.maximum(rng.standard_normal((16, K)), 0.0)
    ratios = {}
    for e in range(-20, 17, 4):
        a = (act * 2.0 ** e).astype(np.float32).astype(np.float64)
        y64 = a @ W.T
        bound = R.gamma(K, "fp16x3") * (np.abs(a) @ np.abs(W).T) + R.floor_matmul(a, W.T)
        for name, s in (("normalised", R._pow2_scale(float(np.abs(a).max()))), ("as is", 1.0)):
            with np.errstate(over="ignore", invalid="ignore"):
                ah, al = R._f16_split(a * s)
                y = (ah @ wh.T + al @ wh.T + ah @ wl.T) / (s * 64)
            ratios[name, e] = R.bound_ratio(y, y64, bound)
    assert max(r for (name, _), r in ratios.items() if name == "normalised") <= 0.1, ratios
    assert all(ratios["as is", e] > 1.0 for e in (-20, -16, -12, 16)), ratios


def test_fp64_backward_matches_autograd_for_a_nonsymmetric_matrix():
    L = G.get("nonsymmetric")
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, L.shape[0], 5))
    W = rng.standard_normal((7, 15))
    dz = rng.standard_normal((2, L.shape[0], 7))
    dx, dW, db = R.cheb_conv_bwd(x, L, W, dz)
    Lt = torch.tensor(L.toarray())
    xt = torch.tensor(x, requires_grad=True)
    Wt = torch.tensor(W, requires_grad=True)
    bt = torch.zeros(7, dtype=torch.float64, requires_grad=True)
    t1 = Lt @ xt
    T = torch.stack([xt, t1, 2 * (Lt @ t1) - xt], dim=3).reshape(2, L.shape[0], 15)   # column fin*3 + k
    (T @ Wt.T + bt).backward(torch.tensor(dz))
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dW, Wt.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-12, atol=1e-12)
    y = R.cheb_conv_fwd(x, L, W, None)
    np.testing.assert_allclose(y, (T @ Wt.T).detach().numpy(), rtol=1e-12, atol=1e-12)


def test_posenet_reference_matches_the_oracle():
    from oracle import demo_oracle

    g = torch.Generator().manual_seed(0)
    J, H = 17, 64
    sd = {"w1.weight": torch.randn(H, 2 * J, generator=g) * 0.2, "w1.bias": torch.randn(H, generator=g),
          "w2.weight": torch.randn(3 * J, H, generator=g) * 0.2, "w2.bias": torch.randn(3 * J, generator=g)}
    for s in range(2):
        p = f"linear_stages.{s}."
        for n in ("w1", "w2"):
            sd[p + n + ".weight"] = torch.randn(H, H, generator=g) * 0.1
            sd[p + n + ".bias"] = torch.randn(H, generator=g)
        for n in ("batch_norm1", "batch_norm2"):
            sd[p + n + ".weight"] = torch.rand(H, generator=g) + 0.5
            sd[p + n + ".bias"] = torch.randn(H, generator=g)
            sd[p + n + ".running_mean"] = torch.randn(H, generator=g)
            sd[p + n + ".running_var"] = torch.rand(H, generator=g) + 0.5
    x = torch.randn(5, 2 * J, generator=g)
    y, bound = R.posenet_forward({k: v.numpy() for k, v in sd.items()}, x.numpy(), 2)
    yo = demo_oracle.posenet_forward({k: v.double() for k, v in sd.items()}, x.double(), 2).numpy()
    np.testing.assert_allclose(y, yo, rtol=1e-12, atol=1e-12)
    assert np.all(bound > 0)


# ------------------------------------------------------------------------------------------------------ BatchNorm
def _levels():
    from helpers import graph_from_fixture

    return {"joint17": graph_from_fixture("smpl_small")[0][-1], "joint21": graph_from_fixture("mano_like")[0][-1],
            "v1088": graph_from_fixture("mano_like")[0][0]}


def bn_layer(L, B, fin, fout, ratios, seed):
    """A conv layer in front of a BatchNorm: channels of spread scale (sigma over ~2^5) whose conv bias carries
    mean / sigma = ratios[f % len(ratios)] (a constant added in front of a train-mode BN cancels in exact arithmetic).
    Returns (x, W, b, z64 [B, V, fout] float64 with the fp32 b, E = the fp32 conv's bound) and BN parameters."""
    V = L.shape[0]
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2 / (3 * fin + fout))
         * 2.0 ** rng.uniform(-4, 1, (fout, 1))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    sig = R.cheb_conv_fwd(x, L, W, b).reshape(-1, fout).std(axis=0)
    b = (b + np.resize(np.asarray(ratios, np.float64), fout) * sig).astype(np.float32)
    bn = dict(gamma=((rng.random(fout) + 0.5) * rng.choice([-1, 1], fout)).astype(np.float32),
              beta=(rng.standard_normal(fout) * 0.5).astype(np.float32),
              rm=(rng.standard_normal(fout)).astype(np.float32), rv=(rng.random(fout) + 0.5).astype(np.float32))
    return x, W, b, R.cheb_conv_fwd(x, L, W, b), R.cheb_conv_fwd_bound(x, L, W, b, "fp32"), bn


def bn_ratios(got, z64, E, bn, relu):
    """Error / bound of (y, mean, invstd, running_mean, running_var) from an emulation against float64."""
    y64, mean, var, rm64, rv64 = R.bn_train_fwd(z64, bn["gamma"], bn["beta"], bn["rm"], bn["rv"], relu)
    bd = R.bn_train_fwd_bound(z64, E, bn["gamma"], bn["beta"], bn["rm"], bn["rv"])
    ref = (y64, mean, 1 / np.sqrt(var + R.BN_EPS), rm64, rv64)
    return {k: R.bound_ratio(g, r, bd[k]) for k, g, r in zip(("y", "mean", "invstd", "rm", "rv"), got, ref)}


BN_SHAPES = [("joint17", 1, 5, 32), ("joint17", 3, 64, 64), ("joint21", 2, 32, 64), ("joint21", 3, 64, 36),
             ("v1088", 2, 64, 64), ("v1088", 1, 32, 300)]


@pytest.mark.parametrize("lvl,B,fin,fout", BN_SHAPES, ids=lambda v: str(v))
def test_bn_bound_accepts_the_shifted_statistics(lvl, B, fin, fout):
    L = _levels()[lvl]
    x, W, b, z64, E, bn = bn_layer(L, B, fin, fout, [0, 10, 100, 1000], seed=fin + fout + B)
    for relu in (False, True):
        got = R.emulate_bn_train(z64.astype(np.float32), bn["gamma"], bn["beta"], bn["rm"], bn["rv"], relu)
        r = bn_ratios(got, z64, E, bn, relu)
        assert max(r["mean"], r["invstd"]) <= 0.25, r
        # y per channel group: at mean / sigma = 1000 its error is the fixed roundings of z's storage, fp32(mean),
        # mean * scale and shift (~3 u |mean| scale against the bound's ~8 u), not a sum with statistical margin
        y64, *_ = R.bn_train_fwd(z64, bn["gamma"], bn["beta"], bn["rm"], bn["rv"], relu)
        by = R.bn_train_fwd_bound(z64, E, bn["gamma"], bn["beta"], bn["rm"], bn["rv"])["y"]
        ry = (np.abs(got[0] - y64) / by).reshape(-1, fout).max(axis=0)
        assert ry[0::4].max() <= 0.25 and ry[1::4].max() <= 0.25 and ry[2::4].max() <= 0.25, ry
        assert ry[3::4].max() <= 0.5, ry
        # the running updates are a few fixed fp32 roundings (0.9f, 0.1f, two products, a sum: <= ~2.5 u against the
        # bound's 4 u), not a long sum: no statistical margin to ask for
        assert max(r["rm"], r["rv"]) <= 0.7, r


@pytest.mark.parametrize("ratio", [30, 100, 1000])
def test_bn_bound_rejects_the_one_pass_variance(ratio):
    """var = E[z^2] - mean^2 from fp32 partials cancels once |mean| >> sigma: at mean / sigma >= 30 the y it gives is
    outside the bound on 2 x 1088 rows, while the shifted sums of the same z pass at every ratio."""
    L = _levels()["v1088"]
    x, W, b, z64, E, bn = bn_layer(L, 2, 64, 64, [ratio], seed=ratio)
    z32 = z64.astype(np.float32)
    args = (bn["gamma"], bn["beta"], bn["rm"], bn["rv"], False)
    ok = bn_ratios(R.emulate_bn_train(z32, *args), z64, E, bn, False)
    assert max(ok["mean"], ok["invstd"]) <= 0.25 and ok["y"] <= 0.5, ok
    r = bn_ratios(R.emulate_bn_train(z32, *args, mutation="one_pass"), z64, E, bn, False)
    assert r["y"] > 1.0, r


# mutation -> the outputs of which at least one must leave the bound
BN_TEETH = {"unbiased_in_norm": ("y", "invstd"), "biased_in_running": ("rv",), "eps_1e-3": ("y", "invstd"),
            "eps_outside_sqrt": ("y", "invstd"), "momentum_0.01": ("rm", "rv"), "relu_before_affine": ("y",)}


@pytest.mark.parametrize("mutation", sorted(BN_TEETH))
@pytest.mark.parametrize("lvl,B", [("joint17", 1), ("joint21", 1), ("joint17", 3), ("joint21", 3)])
def test_bn_bound_rejects_planted_defects(mutation, lvl, B):
    """On the joint-graph levels (n = 17 ... 63 rows) a 1/n change (biased <-> unbiased variance) moves y by ~1/(2n),
    far outside the bound; eps-outside-sqrt shows on the small-sigma channels the spread of scales provides."""
    L = _levels()[lvl]
    x, W, b, z64, E, bn = bn_layer(L, B, 64, 64, [0, 10], seed=B)
    relu = mutation == "relu_before_affine"
    got = R.emulate_bn_train(z64.astype(np.float32), bn["gamma"], bn["beta"], bn["rm"], bn["rv"], relu, mutation)
    r = bn_ratios(got, z64, E, bn, relu)
    assert max(r[k] for k in BN_TEETH[mutation]) > 1.0, r


def test_bn_eval_bound_accepts_the_folded_affine():
    """k_bn_fold_eval + the conv epilogue in fp32 (scale = gamma / sqrtf(rv + eps), shift = beta + (b - rm) scale,
    y = fma(z - b, scale, shift)) within a quarter of the eval bound, with tiny and large running variances."""
    L = _levels()["joint21"]
    x, W, b, z64, E, bn = bn_layer(L, 3, 64, 64, [0, 10, 100, 1000], seed=4)
    f32 = np.float32
    rv = (np.resize([1e-8, 1e-3, 1.0, 1e4], 64) * (np.random.default_rng(5).random(64) + 0.5)).astype(f32)
    rm = (z64.reshape(-1, 64).mean(axis=0) + np.random.default_rng(6).standard_normal(64)).astype(f32)
    sc = (bn["gamma"] / np.sqrt((rv + f32(1e-5)).astype(f32)).astype(f32)).astype(f32)
    sh = (bn["beta"] + ((b - rm).astype(f32) * sc).astype(f32)).astype(f32)
    acc = (z64 - b.astype(np.float64)).astype(f32)
    y = (acc.astype(np.float64) * sc + sh).astype(f32)
    y64 = R.bn_eval_fwd(z64, bn["gamma"], bn["beta"], rm, rv)
    bound = R.bn_eval_fwd_bound(z64, E, bn["gamma"], bn["beta"], rm, rv, b)
    assert R.bound_ratio(y, y64, bound) <= 0.25
    y_eps = (acc.astype(np.float64) * (bn["gamma"] / np.sqrt(rv + 1e-3)).astype(f32)
             + (bn["beta"] + (b - rm) * (bn["gamma"] / np.sqrt(rv + 1e-3)))).astype(f32)
    assert R.bound_ratio(y_eps, y64, bound) > 1.0


def test_bn_backward_off_by_one_row_count_is_visible_at_17_rows():
    """The network's BN backward g_z = gamma invstd (g - m1 - zhat m2), m1 = sum g / n, m2 = sum g zhat / n: with n - 1
    in place of n, at the 17 rows of the joint level (B = 1), the gradient moves by far more than the 1e-3 of its
    largest entry that the strict open-ReLU gradient parity allows."""
    rng = np.random.default_rng(0)
    z = torch.tensor(rng.standard_normal((17, 34)) * 2 + 3, requires_grad=True)
    g = torch.tensor(rng.standard_normal((17, 34)))
    gamma = torch.tensor(rng.random(34) + 0.5)
    torch.nn.functional.batch_norm(z, None, None, gamma, None, True, 0.1, R.BN_EPS).backward(g)
    zd = z.detach()
    mean, var = zd.mean(0), zd.var(0, unbiased=False)
    invstd = 1 / torch.sqrt(var + R.BN_EPS)
    zh = (zd - mean) * invstd
    ok = gamma * invstd * (g - g.mean(0) - zh * (g * zh).mean(0))
    np.testing.assert_allclose(ok.numpy(), z.grad.numpy(), rtol=1e-10, atol=1e-12)
    for m1, m2 in (((g.sum(0) / 16), (g * zh).mean(0)), (g.mean(0), (g * zh).sum(0) / 16)):
        bad = gamma * invstd * (g - m1 - zh * m2)
        assert float((bad - z.grad).abs().max() / z.grad.abs().max()) > 5e-3


# ------------------------------------------------------------------------------------------------- graph families
@pytest.mark.parametrize("name", sorted(G.FAMILIES))
def test_graph_family_structure(name):
    L = G.get(name)
    assert sp.isspmatrix_csr(L) and L.dtype == np.float64
    V = L.shape[0]
    asym = abs(L - L.T).max() if L.nnz else 0.0
    if name == "nonsymmetric":
        assert asym > 0.1
    else:
        assert asym == 0.0
        assert abs(L.astype(np.float32) - L.astype(np.float32).T).max() == 0   # exactly symmetric after the fp32 cast
    ev = np.linalg.eigvals(L.toarray())
    assert np.abs(ev).max() <= 1 + 1e-9                                        # spectrum inside [-1, 1]
    deg = np.diff(L.indptr)
    if name.startswith("V"):
        assert V == int(name[1:]) and deg.max() <= 5
    if name.startswith("band"):
        bw = int(name[4:])
        assert V == 1024 and deg.max() == 2 * bw + 1
    if name in ("h1_256", "h1_257"):
        c = sp.csr_matrix(L)
        staged = set(range(128)) | set(c[:128].indices.tolist())
        assert len(staged) == (256 if name == "h1_256" else 257)
    if name == "farband20":
        c = sp.csr_matrix(L)
        staged = set(range(128)) | set(c[:128].indices.tolist())
        assert V == 512 and deg.max() == 2 * 20 + 2 and len(staged) == 128 + 20 + 80
    if name.startswith("clique"):
        e = int(name[6:])
        assert V == 512 and deg.max() == 128 + e and np.all(L[:64, :64].toarray() != 0)
    if name == "twoclique49":
        c = sp.csr_matrix(L)
        staged = set(range(64)) | set(c[:64].indices.tolist())
        assert V == 128 and len(staged) == 64 + 49 and c[:64].nnz == 64 * 64 + 49 * 49
    if name == "far":
        assert V == 1088 and L[0, V - 1] != 0 and L[63, V - 64] != 0
    if name == "hub":
        assert deg.max() > 60 and R.headroom_log2(L) >= 5
    if name == "empty_rows":
        dead = np.arange(3, V, 5)
        assert np.all(deg[dead] == 0) and np.all(deg[np.setdiff1d(np.arange(V), dead)] > 0)
    if name.startswith("iso"):
        iso = np.flatnonzero(deg == 1)
        assert len(iso) == 512 and np.all(L.indices[L.indptr[iso]] == iso)
        diag = np.unique(L.diagonal()[iso])
        assert len(diag) == (1 if name == "iso_uniform" else 2)
    if name == "dense":
        c = sp.csr_matrix(L)
        rows = set(range(128)) | set(c[:128].indices.tolist())
        assert len(rows) > 512                                                  # tile 0's staged rows alone


def test_torch_coo_with_duplicates_coalesces_to_the_same_matrix():
    L = G.get("far")
    t = G.torch_coo_with_duplicates(L)
    assert t._nnz() == 2 * L.nnz
    c = t.coalesce()
    back = sp.csr_matrix((c.values().numpy(), (c.indices()[0].numpy(), c.indices()[1].numpy())), shape=L.shape)
    assert abs(back - L).max() == 0


def test_pose2mesh_on_a_nonsymmetric_hierarchy_raises():
    """The network's backward (dX as a forward conv, the swapped dW, the thin head) relies on L~ = L~^T."""
    from helpers import graph_from_fixture
    from pose2mesh_release_b200.meshnet import Pose2Mesh

    mats = list(graph_from_fixture("mano_like")[0])
    bad = mats[2].tolil()
    bad[0, 1] = bad[0, 1] + 0.25
    mats[2] = bad.tocsr()
    with pytest.raises(ValueError, match="symmetric"):
        Pose2Mesh(5, 3, mats, joint_set="mano")
    Pose2Mesh(5, 3, graph_from_fixture("mano_like")[0], joint_set="mano")


# ------------------------------------------------------------------------------------------ the network's precision model
NET_SHAPES = [(32, 64), (64, 128), (128, 64)]


@pytest.mark.parametrize("fin,fout", NET_SHAPES)
def test_network_split_bound_accepts_fp16x3_and_rejects_a_dropped_block(fin, fout):
    """The network forward splits its activations as they are and its weights at the fixed 2^6 (split='network'):
    that arithmetic meets the network bound on post-BatchNorm activations, and losing the lo(T) * hi(W) products of one
    K-block does not."""
    L, x, W, b = _layer(fin, fout)
    x = np.maximum(x + np.float32(0.5), 0).astype(np.float32)     # ReLU activations of O(1)
    y64 = R.cheb_conv_fwd(x, L, W, b)
    bound = R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3", split="network")
    ok = R.bound_ratio(R.emulate_cheb_conv(x, L, W, b, "fp16x3", split="network"), y64, bound)
    assert ok <= 0.25, ok
    r = R.bound_ratio(R.emulate_cheb_conv(x, L, W, b, "fp16x3", drop_block=0, split="network"), y64, bound)
    assert r > 1.0, ("drop lo*Whi of block 0", r)


def test_network_split_floor_is_needed_for_small_activations():
    """Activations of 2^-16 split as they are lose their lo parts to fp16's subnormals: the normalised floor (which
    assumes a power-of-two range normalisation) rejects that arithmetic, the network floor (2^-25 per lo part) covers
    it."""
    L, x, W, b = _layer(32, 64)
    x = x * np.float32(2.0 ** -16)
    y64 = R.cheb_conv_fwd(x, L, W, None)
    y = R.emulate_cheb_conv(x, L, W, None, "fp16x3", split="network")
    assert R.bound_ratio(y, y64, R.cheb_conv_fwd_bound(x, L, W, None, "fp16x3", split="network")) <= 1.0
    assert R.bound_ratio(y, y64, R.cheb_conv_fwd_bound(x, L, W, None, "fp16x3")) > 1.0


def _bn_bwd_case(n, F, ratio, seed):
    """z [n, F] with channels at mean / sigma = ratio, gradients correlated with zhat (m2 != 0), the forward's fp32
    statistics."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, F)) * (rng.random(F) + 0.5)
    z = (z + ratio * z.std(axis=0)).astype(np.float32)
    g = (rng.standard_normal((n, F)) + 0.5 * z / np.abs(z).max(axis=0)).astype(np.float32)
    gam = ((rng.random(F) + 0.5) * rng.choice([-1, 1], F)).astype(np.float32)
    bet = np.where(rng.random(F) < 0.5, 10.0, -10.0).astype(np.float32)    # ReLU open or closed, never near zero
    _, mean, invstd, _, _ = R.emulate_bn_train(z, gam, bet, np.zeros(F), np.ones(F))
    return z, g, gam, bet, mean, invstd


BN_BWD_CASES = [(17, 36, 0), (17, 64, 1000), (1088, 64, 10), (1088, 64, 1000), (600, 256, 100)]


@pytest.mark.parametrize("n,F,ratio", BN_BWD_CASES)
def test_bn_backward_bound_accepts_the_affine_kernel(n, F, ratio):
    """k_bn_bwd_coef + k_bn_bwd_apply4 in fp32 (including its ~3 u |mean| / sigma |gamma invstd m2| coefficient
    error on channels far from zero) meets bn_train_bwd_bound, with and without the ReLU mask."""
    z, g, gam, bet, mean, invstd = _bn_bwd_case(n, F, ratio, seed=n + F + ratio)
    for relu in (False, True):
        gz64, dgam64, dbet64, _ = R.bn_train_bwd(z, g, gam, bet, relu)
        bz, bgam, bbet = R.bn_train_bwd_bound(z, g, gam, bet, relu)
        gz, dgam, dbet = R.emulate_bn_bwd(z, g, gam, bet, mean.astype(np.float32), invstd.astype(np.float32), relu)
        if relu:   # elements within reach of the activation test may take either branch: none in these cases
            pre = R.bn_train_bwd(z, g, gam, bet, relu)[3]
            assert np.abs(pre).min() > 1e-3, "a pre-activation near zero: pick another seed"
        for what, got, ref, bd in (("g_z", gz, gz64, bz), ("dgamma", dgam, dgam64, bgam), ("dbeta", dbet, dbet64, bbet)):
            r = R.bound_ratio(got, ref, bd)
            assert r <= 0.5, (what, relu, r)


@pytest.mark.parametrize("mutation", R.BN_BWD_MUTATIONS)
def test_bn_backward_bound_rejects_a_mutated_kernel(mutation):
    """m2 dropped, the mean not subtracted (c without its a invstd m2 mean term) or 1 / (rows - 1) in place of 1 / rows:
    each makes g_z leave its bound."""
    for n, F, ratio in BN_BWD_CASES:
        z, g, gam, bet, mean, invstd = _bn_bwd_case(n, F, ratio, seed=n + F + ratio)
        gz64 = R.bn_train_bwd(z, g, gam, bet)[0]
        bz = R.bn_train_bwd_bound(z, g, gam, bet)[0]
        gz = R.emulate_bn_bwd(z, g, gam, bet, mean.astype(np.float32), invstd.astype(np.float32), mutation=mutation)[0]
        r = R.bound_ratio(gz, gz64, bz)
        assert r > 1.0, (mutation, n, F, ratio, r)


def test_resample_and_unpool_transposes():
    """<resample(x), g> == <x, resample_t(g)> and <unpool(x), g> == <x, unpool_t(g)>; the resample equals the oracle's
    F.interpolate; the library's fp32 tables are exact at the plans' power-of-two channel ratios."""
    from oracle import meshnet_oracle as mo

    rng = np.random.default_rng(5)
    for fin, fout in ((64, 256), (256, 128), (32, 128), (128, 32), (48, 80)):
        x = rng.standard_normal((2, 6, fin))
        g = rng.standard_normal((2, 6, fout))
        y = R.channel_resample(x, fout)
        np.testing.assert_allclose(y, mo.channel_resample(torch.tensor(x), fout).numpy(), rtol=1e-12, atol=1e-12)
        assert abs((y * g).sum() - (x * R.channel_resample_t(g, fin)).sum()) < 1e-9
        pow2 = max(fin, fout) % min(fin, fout) == 0 and ((max(fin, fout) // min(fin, fout)) & (max(fin, fout) // min(fin, fout) - 1)) == 0
        assert pow2 == np.array_equal(R.resample_matrix(fin, fout), R.resample_matrix(fin, fout, np.float32)) or not pow2
    x = rng.standard_normal((2, 5, 3))
    g = rng.standard_normal((2, 10, 3))
    assert abs((R.unpool(x) * g).sum() - (x * R.unpool_t(g)).sum()) < 1e-12
