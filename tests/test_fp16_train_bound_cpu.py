"""The accuracy contract of the single-pass fp16 backward (P2M_PREC_FP16_MIXED_TC), checked without a GPU.

The backward's tensor-core passes are emulated in numpy the way the single-pass kernels compute them: the gradient dz
scaled into fp16's range by its power of two, the weights at 2^6 and the basis operands are each rounded to the nearest
fp16 once, and the products and sums are taken in float64.  Four passes:
  * dX as a conv on dz:       [dz | L~dz | 2 L~(L~dz) - dz] (scaled, rounded) against the transposed weights;
  * dX by the three dT GEMMs: dT_k = fl(dz) fl(W_k), then dT0 - dT2 + L~^T (dT1 + 2 L~^T dT2) exactly;
  * dW on the basis of x:     sum_rows fl(dz) (x) fl(T_k(x))  (swap 0);
  * dW on the basis of dz:    sum_rows fl(T_k(dz)) (x) fl(x)  (swap 1).
On the repository's graph fixtures each must lie within fp64_ref's bound at "fp16_mixed", and most elements must lie
outside the fp16x3 bound, which shows that the emulation is the single pass and not the split.  That bound is also
the independent formula of the single pass, the fp32 bound plus SPLIT16 times each pass's absolute contraction."""
import numpy as np
import pytest
import scipy.sparse as sp

import fp64_ref as R
from helpers import graph_from_fixture

W_SCALE = 64.0


def f16(v):
    return np.asarray(v, np.float64).astype(np.float16).astype(np.float64)


def scales(x, dz, L, split):
    """(s_x, s_dz): the powers of two the operands enter the rounding at.  network: x as it is, dz and its
    basis by one scale from max|dz| (launch_absmax_scale); normalised: x with the basis headroom as well."""
    s_dz = R._pow2_scale(float(np.abs(dz).max()))
    s_x = R._pow2_scale(float(np.abs(x).max()), R.headroom_log2(L)) if split == "normalised" else 1.0
    return s_x, s_dz


def emulate_bwd16(x, L, W, dz, split="network"):
    """(dx by the conv on dz, dx by the dT GEMMs, dW on the basis of x, dW on the basis of dz) of the single pass."""
    x = np.asarray(x, np.float64)
    dz = np.asarray(dz, np.float64)
    W = np.asarray(W, np.float64)
    B, V, F = x.shape
    fout = W.shape[0]
    s_x, s_dz = scales(x, dz, L, split)
    Wk = W.reshape(fout, F, 3)
    Wh = f16(Wk * W_SCALE) / W_SCALE                          # [o, f, k]
    dzh = f16(dz * s_dz) / s_dz
    # dX as the conv on dz: basis of the scaled dz, rounded, against W'[f][o*3 + k] = W[o][f*3 + k]
    Tdz = R.basis(dz * s_dz, L)                               # [B, V, 3, fout]
    Tdzh = f16(Tdz) / s_dz
    dx_conv = np.einsum("bvko,ofk->bvf", Tdzh, Wh)
    # dX by the three dT GEMMs and the exact basis backward
    dT = [np.einsum("bvo,of->bvf", dzh, Wh[:, :, k]) for k in range(3)]
    Lc = L.tocsr()
    LT = Lc.T.tocsr()

    def lt(a):
        return (LT @ a.transpose(1, 0, 2).reshape(V, -1)).reshape(V, B, F).transpose(1, 0, 2)

    dx_dt = dT[0] - dT[2] + lt(dT[1] + 2 * lt(dT[2]))
    # dW on the basis of x (swap 0): rounded dz and rounded T_k(x)
    Tx = R.basis(x * s_x, L)
    Txh = f16(Tx) / s_x
    dw_x = R._contract_rows(dzh.reshape(B * V, fout), Txh.reshape(B * V, 3, F))
    # dW on the basis of dz (swap 1): rounded T_k(dz) and rounded x; accumulator rows are input features
    xh = f16(x * s_x) / s_x
    dw_dz = np.einsum("rko,rf->ofk", Tdzh.reshape(B * V, 3, fout), xh.reshape(B * V, F)).reshape(fout, 3 * F)
    return dx_conv, dx_dt, dw_x, dw_dz


def layer(V, B, fin, fout, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout))).astype(np.float32)
    dz = (rng.standard_normal((B, V, fout)) * 1e-3).astype(np.float32)
    return x, W, dz


# (fixture, level): V = 1024 and 512 (consecutive 128-row tiles), V = 1088 and 272 (a ragged last tile)
LEVELS = [("smpl_small", 1), ("mano_like", 0), ("smpl_small", 2), ("mano_like", 2)]
# dW sums over every row: its fp16x3 bound grows like sqrt(rows) times the contraction while the single pass's relative
# error falls like 1 / sqrt(rows), so at B V = 1024 about 46 % of dW lies beyond the fp16x3 bound (dX: 70-90 %).  The
# distinction is asserted for dW up to 512 rows (61-77 %).
DW_DISTINCT_ROWS = 512
WIDTHS = [(32, 64), (64, 64), (64, 128), (128, 64), (128, 256), (256, 128), (256, 256)]


def _graph(fx, lvl):
    return graph_from_fixture(fx)[0][lvl].tocsr().astype(np.float32).astype(np.float64)


def abs_contraction(x, L, W) -> np.ndarray:
    """|T| |W|^T [B, V, Fout] with |T| the absolute-value propagated basis [|x|, |L||x|, 2|L|(|L||x|) + |x|]."""
    Labs = abs(sp.csr_matrix(L, dtype=np.float64))
    ax = np.abs(np.asarray(x, dtype=np.float64))
    Tabs = R.basis(ax, Labs)
    Tabs[:, :, 2] += 2 * ax
    return (R._flat(Tabs) @ np.abs(np.asarray(W, dtype=np.float64)).T).reshape(ax.shape[0], ax.shape[1], -1)


def bwd_contractions(x, L, W, dz):
    """(|dx| contraction [B, V, Fin], |dW| contraction [Fout, 3 Fin]) of cheb_conv_bwd."""
    Labs = abs(sp.csr_matrix(L, dtype=np.float64))
    LT = sp.csr_matrix(Labs.T)
    aW = np.abs(np.asarray(W, dtype=np.float64))
    adz = np.abs(np.asarray(dz, dtype=np.float64))
    ax = np.abs(np.asarray(x, dtype=np.float64))
    B, V, F = ax.shape
    fout = aW.shape[0]
    Wk = aW.reshape(fout, F, 3)
    dzf = adz.reshape(B * V, fout)
    A = [(dzf @ Wk[:, :, k]).reshape(B, V, F) for k in range(3)]

    def lt(a):
        return (LT @ a.transpose(1, 0, 2).reshape(V, -1)).reshape(V, B, F).transpose(1, 0, 2)

    c_dx = A[0] + A[2] + lt(A[1] + 2 * lt(A[2]))
    Tabs = R.basis(ax, Labs)
    Tabs[:, :, 2] += 2 * ax
    c_dw = R._contract_rows(dzf, Tabs.reshape(B * V, 3, F))
    return c_dx, c_dw


def test_unified_bound_is_the_single_pass_bound():
    """fp64_ref's conv bounds at both single-pass precisions equal the fp32 bound plus SPLIT16 times each pass's
    absolute contraction (to rounding), with and without dw_chain; db has no tensor-core pass."""
    L = _graph("smpl_small", 2)
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, L.shape[0], 64))
    W = rng.standard_normal((128, 192)) * 0.1
    b = rng.standard_normal(128) * 0.1
    dz = rng.standard_normal((2, L.shape[0], 128)) * 1e-3
    c_y = abs_contraction(x, L, W)
    c_dx, c_dw = bwd_contractions(x, L, W, dz)
    for split in ("network", "normalised"):
        y32 = R.cheb_conv_fwd_bound(x, L, W, b, "fp32", split=split)
        for chain in (0, 5000):
            b_dx, b_dw, b_db = R.cheb_conv_bwd_bound(x, L, W, dz, "fp32", split=split, dw_chain=chain)
            for precision in ("fp16", "fp16_mixed"):
                np.testing.assert_allclose(R.cheb_conv_fwd_bound(x, L, W, b, precision, split=split),
                                           y32 + R.SPLIT16 * c_y, rtol=1e-12)
                got = R.cheb_conv_bwd_bound(x, L, W, dz, precision, split=split, dw_chain=chain)
                for g, w in zip(got, (b_dx + R.SPLIT16 * c_dx, b_dw + R.SPLIT16 * c_dw, b_db)):
                    np.testing.assert_allclose(g, w, rtol=1e-12)


def test_fp16_backward_bound_contains_the_fp16x3_bound():
    """Same accumulation terms and floors, a larger product term: the single-pass bound is the wider one everywhere."""
    L = _graph("mano_like", 0)
    x, W, dz = layer(L.shape[0], 2, 64, 128, seed=1)
    for split in ("network", "normalised"):
        b16 = R.cheb_conv_bwd_bound(x, L, W, dz, "fp16_mixed", split=split)
        b3 = R.cheb_conv_bwd_bound(x, L, W, dz, "fp16x3", split=split)
        for a, b in zip(b16[:2], b3[:2]):
            assert (a >= b).all() and float((a / b).min()) > 1.5
        assert np.array_equal(b16[2], b3[2])


@pytest.mark.parametrize("split", ["network", "normalised"])
@pytest.mark.parametrize("fx,lvl", LEVELS, ids=lambda v: str(v))
@pytest.mark.parametrize("fin,fout", WIDTHS, ids=lambda v: str(v))
def test_emulated_single_pass_backward_within_the_fp16_bound(fin, fout, fx, lvl, split):
    L = _graph(fx, lvl)
    x, W, dz = layer(L.shape[0], 1, fin, fout, seed=fin * 1000 + fout + lvl)
    dx64, dw64, _ = R.cheb_conv_bwd(x, L, W, dz)
    b_dx, b_dw, _ = R.cheb_conv_bwd_bound(x, L, W, dz, "fp16_mixed", split=split)
    b3_dx, b3_dw, _ = R.cheb_conv_bwd_bound(x, L, W, dz, "fp16x3", split=split)
    dx_conv, dx_dt, dw_x, dw_dz = emulate_bwd16(x, L, W, dz, split)
    for name, got, ref, b16, b3 in (("dx conv on dz", dx_conv, dx64, b_dx, b3_dx), ("dx dT GEMMs", dx_dt, dx64, b_dx, b3_dx),
                                    ("dW basis of x", dw_x, dw64, b_dw, b3_dw),
                                    ("dW basis of dz", dw_dz, dw64, b_dw, b3_dw)):
        err = np.abs(got - ref)
        assert float((err / b16).max()) <= 1.0, (name, float((err / b16).max()))
        # the single pass is distinguishable from fp16x3: most elements are off by more than fp16x3 allows
        if name.startswith("dx") or L.shape[0] <= DW_DISTINCT_ROWS:
            assert float((err > b3).mean()) > 0.5, (name, float((err > b3).mean()))


def test_backward_bound_is_not_vacuous():
    """Typical errors sit within a small factor of the bound, which stays far below the gradients' scale."""
    L = _graph("smpl_small", 1)
    x, W, dz = layer(L.shape[0], 1, 128, 128, seed=3)
    dx64, dw64, _ = R.cheb_conv_bwd(x, L, W, dz)
    b_dx, b_dw, _ = R.cheb_conv_bwd_bound(x, L, W, dz, "fp16_mixed", split="network")
    dx_conv, dx_dt, dw_x, dw_dz = emulate_bwd16(x, L, W, dz, "network")
    for got, ref, b in ((dx_conv, dx64, b_dx), (dx_dt, dx64, b_dx), (dw_x, dw64, b_dw), (dw_dz, dw64, b_dw)):
        assert float((np.abs(got - ref) / b).max()) > 0.02
        assert float(b.max()) < 2e-2 * float(np.abs(ref).max())
