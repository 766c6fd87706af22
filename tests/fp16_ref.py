"""The element-wise error bound of the single-pass fp16 precision (P2M_PREC_FP16_TC), built on tests/fp64_ref.py.

fp64_ref's Chebyshev-conv bound is  gamma_K |T| |W| + floor  with gamma_K = accumulation term (+ SPLIT at fp16x3).  The
single pass rounds each operand to the nearest fp16 once and takes one product per pair, so the split term becomes
    |fl(a) fl(b) - ab| <= (2u + u^2) |ab|,  u = 2^-11   ->   SPLIT16 = 2^-10 + 2^-22
with the same sqrt(n) fp32 accumulation term and the same subnormal floor (network split: an operand entry entered as
it is is off by at most 2^-25, a weight packed at 2^6 by 2^-25 / 2^6; normalised split: 2^(h-34) max|operand|):
    bound_fp16 = bound_fp32 + SPLIT16 |T| |W|."""
import numpy as np
import scipy.sparse as sp

import fp64_ref as R

SPLIT16 = 2.0 ** -10 + 2.0 ** -22


def abs_contraction(x, L, W) -> np.ndarray:
    """|T| |W|^T [B*V, Fout] with |T| the absolute-value propagated basis [|x|, |L||x|, 2|L|(|L||x|) + |x|]."""
    Labs = abs(sp.csr_matrix(L, dtype=np.float64))
    ax = np.abs(np.asarray(x, dtype=np.float64))
    Tabs = R.basis(ax, Labs)
    Tabs[:, :, 2] += 2 * ax
    return R._flat(Tabs) @ np.abs(np.asarray(W, dtype=np.float64)).T


def cheb_conv_fwd_bound16(x, L, W, b, split: str = "normalised") -> np.ndarray:
    B, V, _ = np.shape(x)
    return R.cheb_conv_fwd_bound(x, L, W, b, "fp32", split=split) + \
        SPLIT16 * abs_contraction(x, L, W).reshape(B, V, -1)
