"""The accuracy contract of the single-pass fp16 precision (P2M_PREC_FP16_TC), checked without a GPU.

The Chebyshev conv is emulated in numpy the way the fp16 kernels compute it: the basis T = [x, L~x, 2L~(L~x) - x] and
the weights (x 2^6, the fixed packing scale) are rounded to the nearest fp16 once, and the products and sums are taken
in float64.  On the repository's graph fixtures, at the widths the kernels support, the emulated error must lie within
fp64_ref's bound at "fp16" (SPLIT16 = 2^-10 + 2^-22 times the contraction |T| |W|, plus the accumulation term and
subnormal floor), and for a sizeable fraction of the elements it must exceed the fp16x3 bound: the two
precisions are told apart by the tests on the device."""
import numpy as np
import pytest

import fp64_ref as R
from helpers import graph_from_fixture

W_SCALE = 64.0


def emulate_fp16(x, L, W, b, split):
    """y of the single pass: fp16 operands, float64 products and sums.  split='network': activations unscaled;
    'normalised': the basis scaled by the power of two the single-layer entry point picks (max|x| into
    [2^(9-h), 2^(10-h)))."""
    T = R._flat(R.basis(np.asarray(x, np.float64), L))
    if split == "normalised":
        s = R._pow2_scale(float(np.abs(x).max()), R.headroom_log2(L))
        Th = (T * s).astype(np.float16).astype(np.float64) / s
    else:
        Th = T.astype(np.float16).astype(np.float64)
    Wh = (np.asarray(W, np.float64) * W_SCALE).astype(np.float16).astype(np.float64) / W_SCALE
    y = Th @ Wh.T + np.asarray(b, np.float64)
    return y.reshape(x.shape[0], x.shape[1], -1)


def layer(V, B, fin, fout, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, V, fin)).astype(np.float32)
    W = ((rng.random((fout, 3 * fin)) * 2 - 1) * np.sqrt(2.0 / (3 * fin + fout))).astype(np.float32)
    b = (rng.standard_normal(fout) * 0.1).astype(np.float32)
    return x, W, b


# (fixture, level): V = 1024 (consecutive 128-row tiles) and V = 1088 (a ragged last tile)
LEVELS = [("smpl_small", 1), ("mano_like", 0)]
WIDTHS = [(fin, fout) for fin in (32, 64, 128, 256) for fout in (64, 128, 256)]


def test_split16_is_the_single_pass_product_bound():
    """|fl(a) fl(b) - ab| <= (2u + u^2) |ab| with u = 2^-11 for operands in fp16's normal range, and SPLIT16 is exactly
    that constant."""
    u = 2.0 ** -11
    assert R.SPLIT16 == 2 * u + u * u
    assert R.SPLIT_TERM["fp16"] == R.SPLIT_TERM["fp16_mixed"] == R.SPLIT16
    rng = np.random.default_rng(0)
    a = rng.choice([-1.0, 1.0], 100000) * 2.0 ** rng.uniform(-12, 12, 100000)
    b = rng.choice([-1.0, 1.0], 100000) * 2.0 ** rng.uniform(-12, 12, 100000)
    err = np.abs(a.astype(np.float16).astype(np.float64) * b.astype(np.float16).astype(np.float64) - a * b)
    assert (err <= R.SPLIT16 * np.abs(a * b)).all()
    assert float((err / np.abs(a * b)).max()) > 0.5 * 2 * u   # the bound is not loose by more than 2x


def test_unknown_precision_is_refused():
    """A precision without a split term raises: it must not be bounded as fp32."""
    with pytest.raises(KeyError):
        R.gamma(96, "fp16x2")


def test_fp16_bound_contains_the_fp16x3_bound():
    """Same accumulation term and floor, a larger split term: the fp16 bound is the wider one everywhere."""
    L = graph_from_fixture("mano_like")[0][0].tocsr().astype(np.float32).astype(np.float64)
    x, W, b = layer(L.shape[0], 2, 64, 128, seed=1)
    for split in ("network", "normalised"):
        b16 = R.cheb_conv_fwd_bound(x, L, W, b, "fp16", split=split)
        b3 = R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3", split=split)
        assert (b16 >= b3).all() and float((b16 / b3).min()) > 100


@pytest.mark.parametrize("split", ["network", "normalised"])
@pytest.mark.parametrize("fx,lvl", LEVELS, ids=lambda v: str(v))
@pytest.mark.parametrize("fin,fout", WIDTHS, ids=lambda v: str(v))
def test_emulated_single_pass_within_the_fp16_bound(fin, fout, fx, lvl, split):
    L = graph_from_fixture(fx)[0][lvl].tocsr().astype(np.float32).astype(np.float64)
    x, W, b = layer(L.shape[0], 1, fin, fout, seed=fin * 1000 + fout + lvl)
    y64 = R.cheb_conv_fwd(x, L, W, b)
    y16 = emulate_fp16(x, L, W, b, split)
    err = np.abs(y16 - y64)
    b16 = R.cheb_conv_fwd_bound(x, L, W, b, "fp16", split=split)
    b3 = R.cheb_conv_fwd_bound(x, L, W, b, "fp16x3", split=split)
    assert float((err / b16).max()) <= 1.0
    # the single pass is distinguishable from fp16x3: most elements are off by more than fp16x3 allows
    assert float((err > b3).mean()) > 0.5, float((err > b3).mean())


def test_bound_is_not_vacuous():
    """Typical errors sit within a small factor of the bound, which stays far below the output scale."""
    L = graph_from_fixture("smpl_small")[0][1].tocsr().astype(np.float32).astype(np.float64)
    x, W, b = layer(L.shape[0], 1, 128, 128, seed=3)
    y64 = R.cheb_conv_fwd(x, L, W, b)
    err = np.abs(emulate_fp16(x, L, W, b, "network") - y64)
    b16 = R.cheb_conv_fwd_bound(x, L, W, b, "fp16", split="network")
    assert float((err / b16).max()) > 0.02
    assert float(b16.max()) < 2e-2 * float(np.abs(y64).max())
