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
