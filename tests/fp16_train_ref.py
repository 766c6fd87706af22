"""The element-wise error bounds of the single-pass fp16 backward (P2M_PREC_FP16_MIXED_TC), built on tests/fp64_ref.py
the way tests/fp16_ref.py builds the forward's.

Every single-pass tensor-core pass of the backward rounds each of its two operands to the nearest fp16 once (the
gradient after its power-of-two scale into fp16's range, the weights at 2^6) and takes one product per pair:
    |fl(a) fl(b) - ab| <= SPLIT16 |ab|,  SPLIT16 = 2^-10 + 2^-22
so each bound is fp64_ref.cheb_conv_bwd_bound at fp32 (the accumulation terms, the cross-CTA adds, dw_chain and the
subnormal floors) plus SPLIT16 times the absolute contraction of the pass:
  * dX: |dT0| + |dT2| + |L|^T (|dT1| + 2 |L|^T |dT2|) with |dT_k| = |dz| |W_k|.  For the symmetric L~ this is also the
    contraction |T(dz)| |W'| of the conv on dz with the transposed weights, so one bound serves both dX paths.
  * dW: sum_rows |dz| (x) |T_k(x)|, which for the symmetric L~ equals sum_rows |T_k(dz)| (x) |x| (dW on the basis of dz).
  * db: no tensor-core pass, the fp32 bound as it is."""
import numpy as np
import scipy.sparse as sp

import fp16_ref as R16
import fp64_ref as R

SPLIT16 = R16.SPLIT16


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


def cheb_conv_bwd_bound16(x, L, W, dz, split: str = "normalised", dw_chain=0):
    """Bounds (dx, dW, db) of the single-pass backward: the fp32 bound plus SPLIT16 times each contraction."""
    b_dx, b_dw, b_db = R.cheb_conv_bwd_bound(x, L, W, dz, "fp32", split=split, dw_chain=dw_chain)
    c_dx, c_dw = bwd_contractions(x, L, W, dz)
    return b_dx + SPLIT16 * c_dx, b_dw + SPLIT16 * c_dw, b_db
