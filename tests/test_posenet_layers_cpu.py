"""CPU checks of the per-layer PoseNet references (tests/fp64_ref.py, tests/posenet_layers_ref.py) the GPU test
tests/test_gpu_posenet_layers_fp64.py relies on: the ReLU mask rule is exact, fp32 emulations of each layer's kernel
meet its bound, and each planted kernel defect leaves it."""
from fractions import Fraction

import numpy as np
import pytest

import fp64_ref as R
import posenet_layers_ref as PL
from posenet_train_ref import dropout_multiplier

f32 = np.float32


def test_relu_mask_is_exact():
    """relu_mask's float64 evaluation of z scale + shift has the sign of the exact sum (hence of fmaf's rounding of it)
    on random fp32 triples and on triples whose sum cancels to a few ulps of z scale, or exactly."""
    rng = np.random.default_rng(0)
    n = 10_000
    z = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(f32)
    sc = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(f32)
    sh = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(f32)
    half = n // 2                      # near-cancelling: shift = -fp32(z scale) moved by -2 .. 2 ulps
    prod = (z[:half].astype(np.float64) * sc[:half]).astype(f32)
    steps = rng.integers(-2, 3, half)
    sh[:half] = np.array([-np.nextafter(p, np.sign(k) * np.inf) if k else -p for p, k in zip(prod, steps)], f32)
    got = R.relu_mask(z, sc, sh)
    exact = np.array([Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)) > 0 for a, b, c in zip(z, sc, sh)])
    assert np.array_equal(got, exact)
    fma32 = np.array([float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))) for a, b, c in
                      zip(z, sc, sh)]).astype(f32)   # correctly rounded to float64, then fp32: the sign survives
    assert np.array_equal(got, fma32 > 0)
    assert (~got[:half]).any() and got[:half].any()


def _dense(m, k, n, seed, scale_a=1.0):
    rng = np.random.default_rng(seed)
    A = (np.maximum(rng.standard_normal((m, k)), 0) * scale_a).astype(f32)
    W = ((rng.random((k, n)) * 2 - 1) / np.sqrt(k)).astype(f32)
    return A, W


@pytest.mark.parametrize("m,k,n", [(64, 128, 128), (50, 96, 64), (128, 64, 192)])
def test_dense_gemm_emulation_meets_its_bound(m, k, n):
    """fp16x3 with a fixed-scale weight operand (forward, dX) and with a range-normalised activation operand (dW), at
    activation scales 2^-20 .. 2^12; fp32 single-precision GEMMs."""
    for e in (-20, 0, 12):
        A, W = _dense(m, k, n, k + n + e, 2.0 ** e)
        ref = A.astype(np.float64) @ W.astype(np.float64)
        for side in ("fixed", "normalised"):
            r = R.bound_ratio(R.emulate_dense_gemm(A, W, side), ref, R.dense_gemm_bound(A, W, "fp16x3", side))
            assert r <= 0.25, (e, side, r)
        r32 = R.bound_ratio((A @ W).astype(np.float64), ref, R.dense_gemm_bound(A, W, "fp32"))
        assert r32 <= 0.5, (e, r32)


@pytest.mark.parametrize("side,k", [("fixed", 128), ("normalised", 64)])
def test_dense_gemm_bound_rejects_a_dropped_lo_block(side, k):
    """dX (g against the weights at 2^6, K = H) and dW (g^T against a, K = B): one K-block of lo(A) * hi(B) missing."""
    rng = np.random.default_rng(k)
    A = rng.standard_normal((96, k)).astype(f32)
    Bm = (np.maximum(rng.standard_normal((k, 64)), 0) if side == "normalised"
          else rng.standard_normal((k, 64)) / np.sqrt(k)).astype(f32)
    ref = A.astype(np.float64) @ Bm
    bd = R.dense_gemm_bound(A, Bm, "fp16x3", side)
    assert R.bound_ratio(R.emulate_dense_gemm(A, Bm, side), ref, bd) <= 0.25
    assert R.bound_ratio(R.emulate_dense_gemm(A, Bm, side, drop_block=1), ref, bd) > 1.0


@pytest.mark.parametrize("drop", ["a", "b"])
def test_dense_gemm_bound_rejects_a_dropped_lo_operand_at_k4096(drop):
    """A dX at the production width, K = H = 4096: g of either sign against the weights at 2^6.  Leaving out every
    lo(g) * hi(W) product, or every hi(g) * lo(W) one (fp16x2 on one side), is a relative error of ~2^-12 per product
    with partial sums that cancel: the per-element bound, whose accumulation term follows those partial sums, rejects
    both, while fp16x3 passes."""
    rng = np.random.default_rng(6)
    g = rng.standard_normal((16, 4096)).astype(f32)
    W = ((rng.random((4096, 64)) * 2 - 1) / 64).astype(f32)
    ref = g.astype(np.float64) @ W
    bd = R.dense_gemm_bound(g, W, "fp16x3", "fixed")
    assert R.bound_ratio(R.emulate_dense_gemm(g, W, "fixed"), ref, bd) <= 0.25
    r = R.bound_ratio(R.emulate_dense_gemm(g, W, "fixed", drop_lo=drop), ref, bd)
    assert r > 1.0, (drop, r)


def test_dense_gemm_bound_rejects_a_stale_gradient_scale():
    """dW of g_z2 normalised with the scale of the previous GEMM's gradient g_y, 2^24 times larger: g_z2's lo parts
    fall into fp16's subnormals."""
    rng = np.random.default_rng(4)
    g_y = rng.standard_normal((64, 128)).astype(f32)
    g_z2 = (rng.standard_normal((64, 128)) * 2.0 ** -24).astype(f32)
    a1 = np.maximum(rng.standard_normal((64, 128)), 0).astype(f32)
    ref = g_z2.T.astype(np.float64) @ a1
    bd = R.dense_gemm_bound(g_z2.T, a1, "fp16x3", "normalised")
    assert R.bound_ratio(R.emulate_dense_gemm(g_z2.T, a1, "normalised"), ref, bd) <= 0.25
    stale = R._pow2_scale(float(np.abs(g_y).max()))
    assert R.bound_ratio(R.emulate_dense_gemm(g_z2.T, a1, "normalised", a_scale=stale), ref, bd) > 1.0


def test_dense_gemm_bound_rejects_garbage_in_the_padding_rows():
    """dW's K = B = 50 padded to Bp = 64: padding rows that are not zero in both operands add to every entry."""
    rng = np.random.default_rng(5)
    g = rng.standard_normal((50, 128)).astype(f32)
    a = np.maximum(rng.standard_normal((50, 128)), 0).astype(f32)
    ref = g.T.astype(np.float64) @ a
    bd = R.dense_gemm_bound(g.T, a, "fp16x3", "normalised")
    pad = lambda t: np.vstack([t, np.zeros((14, 128), f32)])
    assert R.bound_ratio(R.emulate_dense_gemm(pad(g).T, pad(a), "normalised"), ref, bd) <= 0.25
    junk = lambda t: np.vstack([t, (rng.standard_normal((14, 128)) * 1e-3).astype(f32)])
    assert R.bound_ratio(R.emulate_dense_gemm(junk(g).T, junk(a), "normalised"), ref, bd) > 1.0


def _bn_case(n, F, ratio, seed, near_zero=True):
    """z at mean / sigma = ratio, gradients correlated with zhat, the forward's fp32 statistics and scale / shift, and
    betas that put about half the pre-activations of each channel on either side of zero (some within rounding)."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, F)) * (rng.random(F) + 0.5)
    z = (z + ratio * z.std(axis=0)).astype(f32)
    g = (rng.standard_normal((n, F)) + 0.5 * z / np.abs(z).max(axis=0)).astype(f32)
    gam = ((rng.random(F) + 0.5) * rng.choice([-1, 1], F)).astype(f32)
    bet = (rng.standard_normal(F) * 0.5).astype(f32)
    _, mean, invstd, _, _ = R.emulate_bn_train(z, gam, bet, np.zeros(F), np.ones(F))
    mean, invstd = mean.astype(f32), invstd.astype(f32)
    sc = (gam * invstd).astype(f32)
    if near_zero:                      # channel f: row f's pre-activation cancels to rounding noise
        for f in range(min(F, n)):
            bet[f] = f32(f32(mean[f] * sc[f]) - f32(z[f, f] * sc[f]))
    sh = (bet - (mean * sc).astype(f32)).astype(f32)
    return z, g, gam, bet, mean, invstd, sc, sh


BN_CASES = [(33, 90, 0), (64, 128, 10), (600, 128, 1000), (256, 256, 100)]


@pytest.mark.parametrize("n,F,ratio", BN_CASES)
def test_bn_backward_with_the_device_mask_meets_its_bound(n, F, ratio):
    """emulate_bn_bwd with the device's ReLU mask, batch statistics and frozen, within the bounds that take the same
    mask, although some pre-activations sit within rounding of zero."""
    z, g, gam, bet, mean, invstd, sc, sh = _bn_case(n, F, ratio, n + F)
    mask = R.relu_mask(z, sc, sh)
    pre64 = R.bn_train_fwd(z, gam, bet, np.zeros(F), np.ones(F))[0]
    near = np.abs(pre64) <= R.bn_train_fwd_bound(z, np.zeros(z.shape), gam, bet, np.zeros(F), np.ones(F))["y"]
    assert near.any()
    gz, dgam, dbet = R.emulate_bn_bwd(z, g, gam, bet, mean, invstd, mask=mask)
    ref = R.bn_train_bwd(z, g, gam, bet, mask=mask)[:3]
    for what, got, r, b in zip(("g_z", "dgamma", "dbeta"), (gz, dgam, dbet), ref,
                               R.bn_train_bwd_bound(z, g, gam, bet, mask=mask)):
        assert R.bound_ratio(got, r, b) <= 0.5, (what, R.bound_ratio(got, r, b))
    rm, rv = (mean + f32(0.25)).astype(f32), (np.abs(rng_var(F)) + f32(0.5)).astype(f32)
    ist = (f32(1) / np.sqrt((rv + f32(R.BN_EPS)).astype(f32))).astype(f32)
    gm = np.where(mask, g, f32(0))
    got = R.emulate_bn_bwd(z, gm, gam, bet, rm, ist, frozen=True)
    ref = R.bn_frozen_bwd(z, gm, gam, rm, rv)
    for what, gv, r, b in zip(("g_z", "dgamma", "dbeta"), got, ref, R.bn_frozen_bwd_bound(z, gm, gam, rm, rv)):
        assert R.bound_ratio(gv, r, b) <= 0.5, ("frozen", what, R.bound_ratio(gv, r, b))


def rng_var(F):
    return np.random.default_rng(F).random(F).astype(f32)


@pytest.mark.parametrize("mutation", R.BN_BWD_MUTATIONS)
def test_bn_backward_with_the_device_mask_rejects_a_mutated_kernel(mutation):
    for n, F, ratio in BN_CASES:
        z, g, gam, bet, mean, invstd, sc, sh = _bn_case(n, F, ratio, n + F)
        mask = R.relu_mask(z, sc, sh)
        gz = R.emulate_bn_bwd(z, g, gam, bet, mean, invstd, mutation=mutation, mask=mask)[0]
        r = R.bound_ratio(gz, R.bn_train_bwd(z, g, gam, bet, mask=mask)[0],
                          R.bn_train_bwd_bound(z, g, gam, bet, mask=mask)[0])
        assert r > 1.0, (mutation, n, F, ratio, r)


@pytest.mark.parametrize("n,F,ratio", BN_CASES)
def test_bn_backward_rejects_the_wrong_statistics_branch(n, F, ratio):
    """The batch-mean terms kept in a frozen backward, or dropped in a batch-statistics one."""
    z, g, gam, bet, mean, invstd, sc, sh = _bn_case(n, F, ratio, n + F)
    mask = R.relu_mask(z, sc, sh)
    gm = np.where(mask, g, f32(0))
    rm, rv = mean, (f32(1) / (invstd.astype(np.float64) ** 2) - R.BN_EPS).astype(f32)
    ist = (f32(1) / np.sqrt((rv + f32(R.BN_EPS)).astype(f32))).astype(f32)
    kept = R.emulate_bn_bwd(z, gm, gam, bet, rm, ist, frozen=False)[0]
    assert R.bound_ratio(kept, R.bn_frozen_bwd(z, gm, gam, rm, rv)[0], R.bn_frozen_bwd_bound(z, gm, gam, rm, rv)[0]) > 1
    dropped = R.emulate_bn_bwd(z, g, gam, bet, mean, invstd, mask=mask, frozen=True)[0]
    assert R.bound_ratio(dropped, R.bn_train_bwd(z, g, gam, bet, mask=mask)[0],
                         R.bn_train_bwd_bound(z, g, gam, bet, mask=mask)[0]) > 1


@pytest.mark.parametrize("p", [0.5, 0.3])
def test_bn_backward_rejects_the_wrong_dropout_multipliers(p):
    """g' = g_a times the multipliers of the layer's own dropout (d2 for bn2): d1's in their place, or the keep mask
    without 1 / (1 - p), leave the bound."""
    n, F = 128, 64
    z, g, gam, bet, mean, invstd, sc, sh = _bn_case(n, F, 10, 7)
    seed = [0x5DEECE66D1234567, -987654321]
    m1, m2 = (dropout_multiplier(seed, d, n * F, p).reshape(n, F).astype(f32) for d in (0, 1))
    mask = R.relu_mask(z, sc, sh)
    right = (g * m2).astype(f32)
    ref = R.bn_train_bwd(z, right, gam, bet, mask=mask)[0]
    bd = R.bn_train_bwd_bound(z, right, gam, bet, mask=mask)[0]
    assert R.bound_ratio(R.emulate_bn_bwd(z, right, gam, bet, mean, invstd, mask=mask)[0], ref, bd) <= 0.5
    for wrong in ((g * m1).astype(f32), np.where(m2 != 0, g, f32(0))):
        assert R.bound_ratio(R.emulate_bn_bwd(z, wrong, gam, bet, mean, invstd, mask=mask)[0], ref, bd) > 1.0


def test_cumulative_momentum_uses_the_incremented_count():
    """momentum None after 5 batches: the update factor is 1 / 6 (the count after its increment); 1 / 7 leaves the
    running-statistics bound."""
    n, F = 64, 128
    z, g, gam, bet, mean, invstd, sc, sh = _bn_case(n, F, 3, 2, near_zero=False)
    rm, rv = np.zeros(F, f32), np.ones(F, f32)
    _, _, _, rm64, rv64 = R.bn_train_fwd(z, gam, bet, rm, rv, momentum=1 / 6)
    bd = R.bn_train_fwd_bound(z, np.zeros(z.shape), gam, bet, rm, rv, momentum=1 / 6)
    for mom, ok in ((1 / 6, True), (1 / 7, False)):
        _, _, _, rm_e, rv_e = R.emulate_bn_train(z, gam, bet, rm, rv, momentum=mom)
        r = max(R.bound_ratio(rm_e, rm64, bd["rm"]), R.bound_ratio(rv_e, rv64, bd["rv"]))
        assert (r <= 1.0) == ok, (mom, r)


def test_saved_layout_parses_to_the_documented_size():
    """parse_saved walks y_0 .. y_S, z2_0 .. z2_{S-1} and the 8 S statistics vectors, each at a multiple of 256
    bytes."""
    for B, H, S in ((50, 90, 1), (256, 4096, 2), (2, 128, 0)):
        a = lambda n: -(-4 * n // 256) * 256
        want = (S + 1) * a(B * H) + S * a(B * H) + 8 * S * a(H)
        buf = np.zeros(want, np.uint8)
        y, z2, stats, off = PL.parse_saved(buf, B, H, S)
        assert off == want and len(y) == S + 1 and len(z2) == S and all(len(s) == 2 for s in stats)
        assert all(t.shape == (B, H) for t in y + z2)
