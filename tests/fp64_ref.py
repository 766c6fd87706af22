"""Float64 references of the operations the CUDA kernels compute, and the element-wise error bound they are held to.

Everything here is plain numpy / scipy in float64.  The bound replaces "max |y - y_ref| / max |y_ref|", which hides
errors in small entries, with one bound per output element derived from the precision model of the kernels:

    |y_ij - y64_ij|  <=  gamma_K * (|A| |B|)_ij  +  floor_ij

where |A| |B| is the contraction of the absolute values of the two operands (for the Chebyshev conv, A is the
absolute-value propagated basis |T| = [|x|, |L||x|, 2|L|(|L||x|) + |x|], which also covers the rounding of the fp32
T1 pass and of the on-chip T2).

gamma_K, fp16x3 (wgmma, each operand split as hi = fp16(v), lo = fp16(v - hi), products hi*hi + lo*hi + hi*lo):
  * the lo part is rounded to fp16: |v - hi - lo| <= 2^-11 |lo| <= 2^-22 |v|, once per operand   -> 2 * 2^-22
  * the dropped lo*lo product: |lo_a lo_b| <= 2^-22 |a b|                                         -> 1 * 2^-22
  * fp32 accumulation of 3K products and the fp32 sparse products of the basis (row length deg): rounding errors of
    unit roundoff u = 2^-24 that are independent with mean zero grow like sqrt(n) u (the probabilistic bound of
    Higham & Mary, SIAM J. Sci. Comput. 41(5), 2019, with lambda = LAMBDA)          -> LAMBDA (sqrt(3K) + sqrt(2 deg + 3)) u
gamma_K, fp16 and fp16_mixed (single pass: each operand rounded to the nearest fp16 once, one product per pair):
  * |fl(a) fl(b) - ab| <= (2u + u^2) |ab| with fp16's unit roundoff u = 2^-11                  -> 2^-10 + 2^-22
  * the same fp32 accumulation term as fp16x3.
gamma_K, fp32 (CUDA cores, FMA): only the accumulation term.
SPLIT_TERM holds each precision's product-split term (SPLIT16 for the single pass).

floor (only matters where |A||B| is tiny, i.e. a row of zeros or an entry of exact cancellation): fp16's subnormal
spacing 2^-24 bounds the absolute error of a lo part, or of a single-pass operand rounded to fp16.  The operands enter
the split scaled into [2^(9-h), 2^(10-h)) by a power of two (h = 0 for the weights, h = ceil(log2(2 r^2 + 1)) for the
basis, r = max absolute row sum of L~), so the absolute error per operand entry is <= 2^(h-34) max|operand| and the
floor is that times the other operand's absolute row sum.  It scales with the inputs: it is never an absolute
constant.

The network schedules (p2m_meshnet_forward / _backward) do not range-normalise every operand: the forward conv's
activations and the x side of dW enter the split as they are, the weights at the fixed scale 2^6.  There a lo part's
absolute error is <= 2^-25 (half of fp16's subnormal spacing) divided by that fixed scale (split="network" of the conv
bounds).  Next to the normalised floor 2^-34 max|x| this dominates once max|x| < 2^9, but next to fp16x3's relative
term 3 2^-22 |x| only where |x| falls below 2^-25 / (3 2^-22) = 1/24 (about 2^-4.6): activations after a BatchNorm
are O(1).
"""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp

U32 = 2.0 ** -24          # fp32 unit roundoff
SPLIT16 = 2.0 ** -10 + 2.0 ** -22    # single-pass fp16: one rounding of each operand
# the product-split term of each precision (see the module docstring); fp16x3: two lo roundings + the dropped lo*lo term
SPLIT_TERM = {"fp32": 0.0, "fp16x3": 3 * 2.0 ** -22, "fp16": SPLIT16, "fp16_mixed": SPLIT16}
LAMBDA = 1.0              # probabilistic accumulation constant (see the module docstring)


def gamma(k: int, precision: str, deg: int = 0) -> float:
    acc = LAMBDA * (math.sqrt(3 * k) + math.sqrt(2 * deg + 3)) * U32
    return acc + SPLIT_TERM[precision]


def headroom_log2(L: sp.spmatrix) -> int:
    """h with 2^h >= 2 r^2 + 1 >= max|T2| / max|x| (r = max absolute row sum of L~)."""
    r = float(abs(sp.csr_matrix(L)).sum(axis=1).max()) if L.shape[0] else 0.0
    return int(math.ceil(math.log2(2 * r * r + 1)))


def floor_matmul(A: np.ndarray, B: np.ndarray, h_a: int = 0, h_b: int = 0) -> np.ndarray:
    """Subnormal floor of C = A @ B (A [m, k], B [k, n]) when both operands went through the fp16 split."""
    fa = 2.0 ** (h_a - 34) * float(np.abs(A).max(initial=0.0))
    fb = 2.0 ** (h_b - 34) * float(np.abs(B).max(initial=0.0))
    return fa * np.abs(B).sum(axis=0, keepdims=True) + fb * np.abs(A).sum(axis=1, keepdims=True)


def max_degree(L: sp.spmatrix) -> int:
    c = sp.csr_matrix(L)
    return int(np.diff(c.indptr).max(initial=0))


# --------------------------------------------------------------------------------------------- Chebyshev conv (K = 3)
def basis(x: np.ndarray, L: sp.spmatrix) -> np.ndarray:
    """T = [x | L x | 2 L (L x) - x] along the last axis, laid out [B, V, 3, Fin]."""
    L = sp.csr_matrix(L, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    B, V, F = x.shape
    xf = x.transpose(1, 0, 2).reshape(V, B * F)
    t1 = L @ xf
    t2 = 2 * (L @ t1) - xf
    T = np.stack([xf, t1, t2], axis=1).reshape(V, 3, B, F).transpose(2, 0, 1, 3)
    return T


def _flat(T: np.ndarray) -> np.ndarray:
    """[B, V, 3, F] -> [B*V, 3F] with the reference's column order fin*3 + k."""
    B, V, K, F = T.shape
    return T.transpose(0, 1, 3, 2).reshape(B * V, F * K)


def cheb_conv_fwd(x, L, W, b=None) -> np.ndarray:
    """y = [T0|T1|T2] W^T + b, W [Fout, 3 Fin] with column fin*3 + k (reference layout).  -> [B, V, Fout]"""
    W = np.asarray(W, dtype=np.float64)
    B, V, _ = np.shape(x)
    y = _flat(basis(x, L)) @ W.T
    if b is not None:
        y = y + np.asarray(b, dtype=np.float64)
    return y.reshape(B, V, -1)


NET_LO = 2.0 ** -25       # network split: absolute error of one lo part of an operand entered as it is
NET_W_SCALE = 64.0        # ... and the fixed scale the weights are packed at


def cheb_conv_fwd_bound(x, L, W, b, precision: str, split: str = "normalised") -> np.ndarray:
    """split: 'normalised' (the single-layer entry points: both operands scaled into fp16's range by powers of two) or
    'network' (the network forward: activations unscaled, weights at the fixed 2^6)."""
    Labs = abs(sp.csr_matrix(L, dtype=np.float64))
    W = np.asarray(W, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    B, V, F = x.shape
    ax = np.abs(x)
    Tabs = basis(ax, Labs)
    Tabs[:, :, 2] += 2 * ax              # 2|L|(|L||x|) + |x|  (basis() gave 2|L|(|L||x|) - |x|)
    Ta = _flat(Tabs)
    k = 3 * F
    g = gamma(k, precision, max_degree(L))
    bound = g * (Ta @ np.abs(W).T)
    if b is not None:
        bound = bound + U32 * np.abs(np.asarray(b, dtype=np.float64))
    h = headroom_log2(L)
    if split == "network":
        fl = NET_LO * np.abs(W).sum(axis=1)[None, :] + NET_LO / NET_W_SCALE * Ta.sum(axis=1, keepdims=True)
    else:
        fl = (2.0 ** (h - 34) * float(ax.max(initial=0.0)) * np.abs(W).sum(axis=1)[None, :]
              + 2.0 ** -34 * float(np.abs(W).max(initial=0.0)) * Ta.sum(axis=1, keepdims=True))
    return (bound + fl).reshape(B, V, -1)


def _contract_rows(dz, T):
    """sum_rows dz[:, o] T[:, k, f] -> [o, f*3 + k] (as one GEMM)."""
    R, K, F = T.shape
    return (dz.T @ T.reshape(R, K * F)).reshape(-1, K, F).transpose(0, 2, 1).reshape(-1, F * K)


def cheb_conv_bwd(x, L, W, dz):
    """Gradients of y = [T0|T1|T2] W^T + b for any (not necessarily symmetric) L:
    dx = dT0 - dT2 + L^T (dT1 + 2 L^T dT2),  dW[o, f*3+k] = sum_rows dz[:, o] T_k[:, f],  db = sum_rows dz."""
    L = sp.csr_matrix(L, dtype=np.float64)
    W = np.asarray(W, dtype=np.float64)
    dz = np.asarray(dz, dtype=np.float64)
    B, V, F = np.shape(x)
    fout = W.shape[0]
    Wk = W.reshape(fout, F, 3)                           # [o, f, k]
    dzf = dz.reshape(B * V, fout)
    dT = [(dzf @ Wk[:, :, k]).reshape(B, V, F) for k in range(3)]
    LT = sp.csr_matrix(L.T)

    def lt(a):  # L^T applied per mesh
        return (LT @ a.transpose(1, 0, 2).reshape(V, -1)).reshape(V, B, F).transpose(1, 0, 2)

    dx = dT[0] - dT[2] + lt(dT[1] + 2 * lt(dT[2]))
    T = basis(x, L)                                       # [B, V, 3, F]
    dW = _contract_rows(dzf, T.reshape(B * V, 3, F))
    db = dzf.sum(axis=0)
    return dx, dW, db


def cheb_conv_bwd_bound(x, L, W, dz, precision: str, split: str = "normalised", dw_chain=0):
    """Bounds (dx, dW, db) of cheb_conv_bwd.  split: see cheb_conv_fwd_bound; in the network backward dz is scaled into
    fp16's range by a power of two (floor 2^-34 max|dz| per entry), the weights are at the fixed 2^6 and the x side of
    dW is unscaled.  dX there is either the dT GEMMs + the basis backward or a conv on dz ([dz | L dz | T2 dz] against
    the transposed weights), dW either on the basis of x or on the basis of dz: the floor is the larger of the two.
    For the symmetric L~ the two dX paths have one absolute contraction, |dT0| + |dT2| + |L|^T (|dT1| + 2 |L|^T |dT2|)
    = |T(dz)| |W'|, and so have the two dW paths, sum_rows |dz| (x) |T_k(x)| = sum_rows |T_k(dz)| (x) |x|: gamma's
    split term covers either (at fp16_mixed every pass rounds its two operands to fp16 once).
    dw_chain > 0: hold dW to n u of a sequential chain of that many fp32 adds at least (a grid capped to a few CTAs
    accumulates the rows of many tiles in one CTA, where dW's one-signed partial sums grow linearly, not as sqrt(n))."""
    Labs = abs(sp.csr_matrix(L, dtype=np.float64))
    W = np.abs(np.asarray(W, dtype=np.float64))
    adz = np.abs(np.asarray(dz, dtype=np.float64))
    ax = np.abs(np.asarray(x, dtype=np.float64))
    B, V, F = ax.shape
    fout = W.shape[0]
    deg = max_degree(L)
    h = headroom_log2(L)
    LT = sp.csr_matrix(Labs.T)

    def prop(a0, a1, a2):  # |dT0| + |dT2| + |L|^T (|dT1| + 2 |L|^T |dT2|)
        def lt(a):
            return (LT @ a.transpose(1, 0, 2).reshape(V, -1)).reshape(V, B, F).transpose(1, 0, 2)
        return a0 + a2 + lt(a1 + 2 * lt(a2))

    Wk = W.reshape(fout, F, 3)
    dzf = adz.reshape(B * V, fout)
    A = [(dzf @ Wk[:, :, k]).reshape(B, V, F) for k in range(3)]
    mdz, mw = float(adz.max(initial=0.0)), float(W.max(initial=0.0))
    e_dz = 2.0 ** -34 * mdz
    e_w = NET_LO / NET_W_SCALE if split == "network" else 2.0 ** -34 * mw
    Fl = [(e_dz * Wk[:, :, k].sum(axis=0)[None, :] + e_w * dzf.sum(axis=1, keepdims=True)).reshape(B, V, F)
          for k in range(3)]
    fl_dx = prop(*Fl)
    if split == "network":   # the conv on dz: e_dz per entry of its basis, e_w per weight
        Tdz = basis(adz, Labs)
        Tdz[:, :, 2] += 2 * adz
        conv_fl = (e_dz * Wk.sum(axis=(0, 2))[None, :] + e_w * Tdz.reshape(B * V, -1).sum(axis=1, keepdims=True))
        fl_dx = np.maximum(fl_dx, conv_fl.reshape(B, V, F))
    g_dx = gamma(fout, precision, deg)
    b_dx = g_dx * prop(*A) + fl_dx
    # dW: contraction over all B*V rows of |dz| and the absolute basis
    Tabs = basis(ax, Labs)
    Tabs[:, :, 2] += 2 * ax
    Tf = Tabs.reshape(B * V, 3, F)
    R = B * V
    g_dw = gamma(R, precision, deg) + (R.bit_length() * U32)   # + the cross-CTA fp32 atomic adds (log-depth tree)
    if dw_chain:   # the fp32 accumulation as a sequential chain of dw_chain adds: the deterministic worst case
        g_dw = max(g_dw, dw_chain * U32 + SPLIT_TERM[precision])
    b_dw = g_dw * _contract_rows(dzf, Tf)
    if split == "network":
        Tdz = basis(adz, Labs)
        Tdz[:, :, 2] += 2 * adz
        Tdz = Tdz.reshape(B * V, 3, fout)
        on_x = e_dz * np.einsum("rkf->fk", Tf).reshape(1, 3 * F) + NET_LO * dzf.sum(axis=0)[:, None]
        on_dz = (e_dz * np.repeat(ax.reshape(B * V, F).sum(axis=0), 3)[None, :]
                 + NET_LO * np.einsum("rko->ok", Tdz)[:, None, :].repeat(F, axis=1).reshape(fout, 3 * F))
        fl_dw = np.maximum(on_x, on_dz)
    else:
        fl_dw = (2.0 ** -34 * mdz * np.einsum("rkf->fk", Tf).reshape(1, 3 * F)
                 + 2.0 ** (h - 34) * float(ax.max(initial=0.0)) * dzf.sum(axis=0)[:, None])
    b_db = 2 * U32 * dzf.sum(axis=0)
    return b_dx, b_dw + fl_dw, b_db


# --------------------------------------------------------------------------------------------- dense GEMM / PoseNet
def dense(x, W, b=None, scale=None, shift=None, relu=False, res=None):
    """The dense GEMM epilogue: y = relu?(((x W^T) + b) * scale + shift) + res."""
    y = np.asarray(x, np.float64) @ np.asarray(W, np.float64).T
    if b is not None:
        y = y + b
    if scale is not None:
        y = y * scale + shift
    if relu:
        y = np.maximum(y, 0.0)
    if res is not None:
        y = y + res
    return y


def posenet_forward(sd, x, num_stage: int, eps: float = 1e-5, precision: str = "fp16x3", last_precision: str = "fp32"):
    """PoseNet eval (oracle/demo_oracle.posenet_forward's op order) in float64, with a first-order bound on the error
    of an implementation whose every GEMM satisfies the element-wise bound above.  sd: name -> numpy array.
    Returns (y [B, 3J], bound [B, 3J])."""
    f = {k: np.asarray(v, np.float64) for k, v in sd.items()}
    x = np.asarray(x, np.float64)

    def gemm(a, ea, W, k_prec):
        y = a @ W.T
        aw = np.abs(a) @ np.abs(W).T
        e = gamma(W.shape[1], k_prec) * aw + np.abs(ea) @ np.abs(W).T
        if k_prec == "fp16x3":
            e = e + floor_matmul(a, W.T)
        return y, e

    # the first layer (K = 2J) runs on the fp32 SIMT GEMM, the H x H ones at `precision`, the last at `last_precision`
    y, e = gemm(x, np.zeros_like(x), f["w1.weight"], "fp32")
    y = y + f["w1.bias"]
    e = e + U32 * np.abs(y)
    for s in range(num_stage):
        p = f"linear_stages.{s}."
        sc1 = f[p + "batch_norm1.weight"] / np.sqrt(f[p + "batch_norm1.running_var"] + eps)
        a = np.maximum((y - f[p + "batch_norm1.running_mean"]) * sc1 + f[p + "batch_norm1.bias"], 0.0)
        ea = np.abs(sc1) * e + 4 * U32 * (np.abs(a) + np.abs(y * sc1))
        sc2 = f[p + "batch_norm2.weight"] / np.sqrt(f[p + "batch_norm2.running_var"] + eps)
        z, ez = gemm(a, ea, f[p + "w1.weight"], precision)
        z = z + f[p + "w1.bias"]
        hpre = (z - f[p + "batch_norm2.running_mean"]) * sc2 + f[p + "batch_norm2.bias"]
        h = np.maximum(hpre, 0.0)
        eh = np.abs(sc2) * ez + 4 * U32 * (np.abs(hpre) + np.abs(z * sc2) + np.abs(f[p + "w1.bias"] * sc2))
        o, eo = gemm(h, eh, f[p + "w2.weight"], precision)
        y = y + o + f[p + "w2.bias"]
        e = e + eo + 2 * U32 * (np.abs(y) + np.abs(o))
    out, eout = gemm(y, e, f["w2.weight"], last_precision)
    out = out + f["w2.bias"]
    return out, eout + U32 * np.abs(out)


# --------------------------------------------------------------------------------------------- BatchNorm1d over rows
BN_EPS, BN_MOMENTUM = 1e-5, 0.1
STAT_ROWS = 512           # rows per statistics block of the kernels (fp32 partials inside a block, fp64 across)


def _rows(z) -> np.ndarray:
    z = np.asarray(z, np.float64)
    return z.reshape(-1, z.shape[-1])


def bn_train_fwd(z, gamma, beta, rm, rv, relu=False, eps=BN_EPS, momentum=BN_MOMENTUM):
    """Train-mode BatchNorm1d over the rows of z [..., F] (F.batch_norm, training=True), optionally followed by ReLU.
    Returns (y [z's shape], batch mean [F], biased batch variance [F], new running_mean, new running_var); the running
    update uses the unbiased variance n / (n - 1) like nn.BatchNorm1d."""
    zr = _rows(z)
    n = zr.shape[0]
    mean = zr.mean(axis=0)
    var = ((zr - mean) ** 2).mean(axis=0)
    y = (zr - mean) / np.sqrt(var + eps) * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64)
    if relu:
        y = np.maximum(y, 0.0)
    unbiased = var * n / (n - 1) if n > 1 else var
    rm_new = (1 - momentum) * np.asarray(rm, np.float64) + momentum * mean
    rv_new = (1 - momentum) * np.asarray(rv, np.float64) + momentum * unbiased
    return y.reshape(np.shape(z)), mean, var, rm_new, rv_new


def bn_eval_fwd(z, gamma, beta, rm, rv, relu=False, eps=BN_EPS):
    """Eval-mode BatchNorm1d (running statistics) over the rows of z [..., F], optionally followed by ReLU."""
    z = np.asarray(z, np.float64)
    y = (z - rm) / np.sqrt(np.asarray(rv, np.float64) + eps) * gamma + np.asarray(beta, np.float64)
    return np.maximum(y, 0.0) if relu else y


def col_sum_bound(g) -> np.ndarray:
    """Bound on k_col_sum (the bias gradient of a layer without BatchNorm) over the rows of g [..., F]: the layout of
    the statistics sums (stat_allowance), bounded worst-case, (m + rl) u sum |g|, not probabilistically: the L1 loss's
    gradient has entries of one magnitude and sign pattern, whose rounding errors do not average out."""
    gr = _rows(g)
    n, F = gr.shape
    rl = 256 // min(F, 256)
    m = min(n, -(-STAT_ROWS // rl))
    return (m + rl) * U32 * np.abs(gr).sum(axis=0) + U32 * np.abs(gr.sum(axis=0))


def stat_allowance(n: int, F: int) -> float:
    """Relative rounding allowance of one fp32 statistics sum (k_col_stats): a block of 256 threads splits into
    rl = 256 / min(F, 256) row lanes, each sums <= ceil(STAT_ROWS / rl) rows in fp32, the lanes are added in fp32 and
    the blocks in fp64 (exact at this precision); plus the rounding of z - K and of the square.  Same probabilistic
    sqrt(m) u model as gamma()."""
    rl = 256 // min(F, 256)
    m = min(n, -(-STAT_ROWS // rl))
    return LAMBDA * (math.sqrt(m) + math.sqrt(rl) + 2) * U32


def bn_train_fwd_bound(z, E, gamma, beta, rm, rv, eps=BN_EPS, momentum=BN_MOMENTUM):
    """Element-wise bound on the error of a train-mode BatchNorm (+ optional ReLU: 1-Lipschitz) computed from an fp32 z
    whose every element is within E of the exact z (z: the float64 reference of the layer's pre-BN output).

    First order, the error e of z moves y_i by gamma/sigma (e_i - mean(e) - zhat_i mean(zhat e)), sigma = sqrt(var +
    eps); the local roundings are those of z's fp32 storage (u|z|, the floor of any fp32 implementation), of the
    statistics summed around K = z[0] (stat_allowance), of scale = fp32(gamma invstd), shift = beta - mean scale and
    of the fma(z, scale, shift).  Returns dict(y, mean, invstd, rm, rv) of bounds."""
    zr = _rows(z)
    n, F = zr.shape
    Er = _rows(E) + U32 * np.abs(zr)
    g, b = np.abs(np.asarray(gamma, np.float64)), np.abs(np.asarray(beta, np.float64))
    mean = zr.mean(axis=0)
    var = ((zr - mean) ** 2).mean(axis=0)
    sig = np.sqrt(var + eps)
    zh = np.abs(zr - mean) / sig
    sc = g / sig
    mE, mzE = Er.mean(axis=0), (zh * Er).mean(axis=0)
    # local rounding of the statistics: S = sum (z - K), Q = sum (z - K)^2
    a = stat_allowance(n, F)
    d = zr - zr[0]
    D, Q2 = np.abs(d).mean(axis=0), (d * d).mean(axis=0)
    d_mean = a * D + U32 * np.abs(mean)
    d_var_local = a * Q2 + 2 * np.abs(d.mean(axis=0)) * a * D
    d_var = d_var_local + 2 * sig * mzE                  # + first order of e: 2 mean(|z - mean| E)
    rel_is = d_var_local / (2 * sig ** 2) + 2 * U32
    # scale: u gamma |zhat|; fp32 mean and mean * scale: 2 u |mean| scale; shift: u (|beta| + |mean| scale);
    # fma: u |y| <= u (gamma |zhat| + |beta|)
    ey = (sc * (Er + mE + zh * mzE) + sc * d_mean + g * zh * rel_is
          + U32 * (2 * g * zh + 3 * sc * np.abs(mean) + 2 * b))
    unb = n / (n - 1) if n > 1 else 1.0
    e_rm = momentum * (mE + d_mean) + 4 * U32 * ((1 - momentum) * np.abs(rm) + momentum * np.abs(mean))
    e_rv = momentum * unb * d_var + 4 * U32 * ((1 - momentum) * np.abs(rv) + momentum * unb * var)
    e_is = (1 / sig) * (rel_is + mzE / sig)
    return dict(y=ey.reshape(np.shape(z)), mean=mE + d_mean, invstd=e_is, rm=e_rm, rv=e_rv)


def bn_eval_fwd_bound(z, E, gamma, beta, rm, rv, bias, eps=BN_EPS):
    """Element-wise bound on eval-mode BatchNorm (+ optional ReLU) folded into the conv epilogue (k_bn_fold_eval;
    on the tensor cores launch_rescaled_epilogue only multiplies scale by powers of two):
        scale = gamma / sqrtf(rv + eps),  shift = beta + (bias - rm) scale,  y = fma(z - bias, scale, shift)
    z: the float64 pre-BN conv output WITH bias, E: the conv's bound.  Roundings: three in scale, three in shift, the
    epilogue's product and sum."""
    zr = _rows(z)
    sc = np.abs(np.asarray(gamma, np.float64)) / np.sqrt(np.asarray(rv, np.float64) + eps)
    bias = np.asarray(bias, np.float64)
    zb = np.abs(zr - bias)
    bm = np.abs(bias - rm)
    y = np.abs(bn_eval_fwd(zr, gamma, beta, rm, rv, eps=eps))
    ey = sc * _rows(E) + U32 * (4 * zb * sc + 3 * bm * sc + 2 * np.abs(beta) + 2 * y)
    return ey.reshape(np.shape(z))


def bn_train_bwd(z, g_a, gamma, beta, relu=False, eps=BN_EPS, mask=None):
    """Backward of train-mode BatchNorm1d (+ ReLU) over the rows of z [..., F] from the gradient g_a of its output, with
    the exact batch statistics of z.  Returns (g_z, dgamma, dbeta, pre): g' = g_a [bn(z) > 0],
    g_z = gamma invstd (g' - mean(g') - zhat mean(g' zhat)), dgamma = sum g' zhat, dbeta = sum g'.
    mask (bool, z's shape): the ReLU's open entries as the kernel decided them (relu_mask), in place of the float64
    pre > 0; given, it implies the ReLU."""
    zr, gr = _rows(z), _rows(g_a)
    mean = zr.mean(axis=0)
    invstd = 1.0 / np.sqrt(((zr - mean) ** 2).mean(axis=0) + eps)
    zh = (zr - mean) * invstd
    pre = zh * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64)
    if mask is not None:
        mask = _rows(mask)
    else:
        mask = pre > 0 if relu else np.ones_like(pre, bool)
    g = np.where(mask, gr, 0.0)
    m1, m2 = g.mean(axis=0), (g * zh).mean(axis=0)
    g_z = np.asarray(gamma, np.float64) * invstd * (g - m1 - zh * m2)
    return g_z.reshape(np.shape(z)), (g * zh).sum(axis=0), g.sum(axis=0), pre.reshape(np.shape(z))


def bn_train_bwd_bound(z, g_a, gamma, beta, relu=False, eps=BN_EPS, mask=None):
    """Element-wise bounds (g_z, dgamma, dbeta) on launch_bn_relu_bwd given the exact z and g_a it read (the captured
    fp32 tensors) and the fp32 mean / invstd the forward saved (bn_train_fwd_bound's bounds with E = 0: the error of
    the statistics sums plus the backward error of z's fp32 storage, u |z|).

    First order, with zhat = (z - mean) invstd, a = gamma invstd, m1 = mean(g'), m2 = mean(g' zhat):
      zhat:  |z - mean| e_is + invstd e_mean + 2 u |zhat|                  (the saved statistics; z - mean, the product)
      m1, m2: the sums in the blocks of k_bn_bwd_reduce (stat_allowance), the fp64 division's final rounding
      g_z:   e_a |g' - m1 - zhat m2| + |a| (e_m1 + |m2| e_zhat + |zhat| e_m2) + the evaluation's own roundings.
    Those roundings cover both forms of the kernel: the scalar k_bn_bwd_apply (a (g' - m1 - zhat m2): 5 roundings) and
    the affine k_bn_bwd_coef + k_bn_bwd_apply4, g_z = fma(a, g', fma(b, z, c)) with b = -a invstd m2 and
    c = -a m1 + a invstd m2 mean, whose b z + c cancels to a invstd m2 (mean - z): its coefficients' roundings
    (3 u in b, 4 u in c) are relative to |a invstd m2| |z| and |a invstd m2 mean|, i.e. a backward error of ~3 u (|z| +
    |mean|) in z, which is large next to |zhat| where the channel's mean / sigma is large.
    mask: as in bn_train_bwd.  With the kernel's own mask the bound needs no ReLU-branch allowance: it holds the kernel
    to the g' the kernel formed."""
    zr, gr = _rows(z), _rows(g_a)
    n, F = zr.shape
    gam = np.asarray(gamma, np.float64)
    g_z, dgam, dbet, pre = bn_train_bwd(z, g_a, gamma, beta, relu, eps, mask)
    pre = _rows(pre)
    st = bn_train_fwd_bound(zr, np.zeros_like(zr), gamma, beta, np.zeros(F), np.zeros(F), eps=eps)
    mean = zr.mean(axis=0)
    invstd = 1.0 / np.sqrt(((zr - mean) ** 2).mean(axis=0) + eps)
    zh = (zr - mean) * invstd
    if mask is not None:
        g = np.where(_rows(mask), gr, 0.0)
    else:
        g = np.where(pre > 0, gr, 0.0) if relu else gr
    ag = np.abs(g)
    a = np.abs(gam) * invstd
    e_a = np.abs(gam) * st["invstd"] + U32 * a
    e_zh = np.abs(zr - mean) * st["invstd"] + invstd * st["mean"] + 2 * U32 * np.abs(zh)
    al = stat_allowance(n, F)
    m1, m2 = g.mean(axis=0), (g * zh).mean(axis=0)
    e_m1 = al * ag.mean(axis=0) + U32 * np.abs(m1)
    e_m2 = al * (ag * np.abs(zh)).mean(axis=0) + (ag * e_zh).mean(axis=0) + U32 * np.abs(m2)
    inner = np.abs(g - m1 - zh * m2)
    e_gz = (e_a * inner + a * (e_m1 + np.abs(m2) * e_zh + np.abs(zh) * e_m2)
            + U32 * (5 * a * (ag + np.abs(m1) + np.abs(zh * m2)) + 4 * a * invstd * np.abs(m2) * (np.abs(zr) + np.abs(mean))
                     + 2 * np.abs(g_z.reshape(n, F))))
    e_dbeta = al * ag.sum(axis=0) + U32 * np.abs(dbet)
    e_dgamma = al * (ag * np.abs(zh)).sum(axis=0) + (ag * e_zh).sum(axis=0) + U32 * np.abs(dgam)
    return e_gz.reshape(np.shape(z)), e_dgamma, e_dbeta


# --------------------------------------------------------------------------------------------- network glue
def unpool(x):
    """Nearest x2 unpool along the vertex axis of [B, V, F] (row r reads row r >> 1; meshnet.py:71-78)."""
    return np.repeat(np.asarray(x, np.float64), 2, axis=1)


def unpool_t(g):
    """Transpose of unpool: the pair-sum of rows 2r and 2r + 1."""
    g = np.asarray(g, np.float64)
    B, V, F = g.shape
    return g.reshape(B, V // 2, 2, F).sum(axis=2)


def resample_matrix(fin: int, fout: int, dtype=np.float64) -> np.ndarray:
    """M [fout, fin] of F.interpolate(size=fout, mode='linear', align_corners=False) along the channel axis
    (oracle.meshnet_oracle.channel_resample): src = (j + 0.5) fin / fout - 0.5 clamped at 0, taps floor(src) and the
    next one (clamped at fin - 1), weights 1 - lam, lam.  dtype=np.float32 gives the table the library builds."""
    M = np.zeros((fout, fin), np.float64)
    scale = dtype(fin) / dtype(fout)
    for j in range(fout):
        src = max(dtype(scale * (dtype(j) + dtype(0.5)) - dtype(0.5)), dtype(0))
        a = min(int(src), fin - 1)
        b = a + (1 if a < fin - 1 else 0)
        lam = float(dtype(src - dtype(a)))
        M[j, a] += 1 - lam
        M[j, b] += lam
    return M


def channel_resample(x, fout: int):
    x = np.asarray(x, np.float64)
    return x if x.shape[-1] == fout else x @ resample_matrix(x.shape[-1], fout).T


def channel_resample_t(g, fin: int):
    g = np.asarray(g, np.float64)
    return g if g.shape[-1] == fin else g @ resample_matrix(fin, g.shape[-1])


def channel_resample_bound(x, fout: int):
    """fp32 evaluation of the resample, fma((1 - lam), x_a, lam x_b), against the float64 one: the table's fp32 lam (exact
    when fin / fout is a power of two) and two roundings of the weighted sum."""
    x = np.asarray(x, np.float64)
    fin = x.shape[-1]
    if fin == fout:
        return np.zeros_like(x)
    M, M32 = resample_matrix(fin, fout), resample_matrix(fin, fout, np.float32)
    return np.abs(x) @ (np.abs(M - M32) + 3 * U32 * np.abs(M)).T


def channel_resample_t_bound(g, fin: int):
    """The transposed resample (k_dx_finish, k_basis_bwd_dx: fma over the taps of each input channel, at most
    max_taps of them) against float64."""
    g = np.asarray(g, np.float64)
    fout = g.shape[-1]
    if fin == fout:
        return np.zeros_like(g)
    M, M32 = resample_matrix(fin, fout), resample_matrix(fin, fout, np.float32)
    taps = int((M32 != 0).sum(axis=0).max())
    return np.abs(g) @ (np.abs(M - M32) + (taps + 1) * U32 * np.abs(M))


def thin_head_fused_bound(y_in, E_in, L, W):
    """First-order propagation of an error E_in of the head's input y_in through the 64 -> 3 head (the fused eval head:
    the previous layer's epilogue forms Z = act(y) W' from its fp32 y): |T|(E_in) |W|^T, the head's own fp32 bound
    added by the caller."""
    Labs = abs(sp.csr_matrix(L, dtype=np.float64))
    E_in = np.asarray(E_in, np.float64)
    T = basis(E_in, Labs)
    T[:, :, 2] += 2 * E_in
    B, V, _ = E_in.shape
    return (_flat(T) @ np.abs(np.asarray(W, np.float64)).T).reshape(B, V, -1)


# --------------------------------------------------------------------------------------------- emulators (bound teeth)
def _f16_split(v: np.ndarray):
    hi = v.astype(np.float16).astype(np.float64)
    lo = (v - hi).astype(np.float16).astype(np.float64)
    return hi, lo


def _pow2_scale(m: float, headroom: int = 0) -> float:
    """2^e with m 2^e in [2^(9-headroom), 2^(10-headroom))  (1 for m == 0)."""
    if m <= 0 or not np.isfinite(m):
        return 1.0
    _, e = math.frexp(m)
    return 2.0 ** (10 - e - headroom)


def _tf32(v: np.ndarray) -> np.ndarray:
    """Round fp32 values to TF32 (10 explicit mantissa bits, round to nearest)."""
    b = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x1000) & ~np.uint64(0x1FFF)).astype(np.uint32)
    return b.view(np.float32).astype(np.float64)


def emulate_cheb_conv(x, L, W, b=None, mode: str = "fp16x3", drop_block: int = -1,
                      split: str = "normalised") -> np.ndarray:
    """What a tensor-core kernel of the given arithmetic returns for the conv: the basis in fp32, the operands scaled
    by powers of two into fp16's range (h of headroom for the basis), then
      'fp16x3'    hi*hi + lo*hi + hi*lo
      'fp16'      hi*hi only
      'tf32'      both operands rounded to TF32
    accumulated in fp32 over K (sequentially, products of one k summed in float64 first: a slightly better accumulator
    than the tensor core's).  drop_block >= 0 removes the lo*hi products of the 32 consecutive K-columns (of the
    kernel's [k][fin] operand order) that make up K-block `drop_block`.  split='network': the network forward's
    operands, the basis as it is and the weights at the fixed 2^6."""
    L = sp.csr_matrix(L, dtype=np.float32)
    x32 = np.asarray(x, np.float32)
    B, V, F = x32.shape
    xf = x32.transpose(1, 0, 2).reshape(V, B * F)
    t1 = (L @ xf).astype(np.float32)
    t2 = (np.float32(2) * (L @ t1).astype(np.float32) - xf).astype(np.float32)
    # kernel operand order: column k*F + f
    T = np.concatenate([a.reshape(V, B, F).transpose(1, 0, 2) for a in (xf, t1, t2)], axis=2).reshape(B * V, 3 * F)
    T = T.astype(np.float64)
    Wp = np.asarray(W, np.float64).reshape(-1, F, 3).transpose(0, 2, 1).reshape(-1, 3 * F)   # [o, k*F + f]
    if split == "network":
        sa, sw = 1.0, NET_W_SCALE
    else:
        sa = _pow2_scale(float(np.abs(x32).max(initial=0.0)), headroom_log2(L))
        sw = _pow2_scale(float(np.abs(Wp).max(initial=0.0)))
    A, Bm = T * sa, Wp * sw
    if mode == "tf32":
        terms = [(_tf32(A), _tf32(Bm))]
    else:
        ah, al = _f16_split(A)
        wh, wl = _f16_split(Bm)
        if mode == "fp16":
            terms = [(ah, wh)]
        else:
            al_used = al.copy()
            if drop_block >= 0:
                al_used[:, 32 * drop_block:32 * drop_block + 32] = 0.0
            terms = [(ah, wh), (al_used, wh), (ah, wl)]
    acc = np.zeros((B * V, Wp.shape[0]), np.float32)
    for k in range(3 * F):
        p = sum(np.outer(a[:, k], w[:, k]) for a, w in terms)
        acc = (acc + p.astype(np.float32)).astype(np.float32)
    y = acc.astype(np.float64) / (sa * sw)
    if b is not None:
        y = y + np.asarray(b, np.float64)
    return y.reshape(B, V, -1)


BN_MUTATIONS = ("one_pass", "unbiased_in_norm", "biased_in_running", "eps_1e-3", "eps_outside_sqrt", "momentum_0.01",
                "relu_before_affine")


def emulate_bn_train(z, gamma, beta, rm, rv, relu=False, mutation: str = "", momentum=BN_MOMENTUM, eps=BN_EPS):
    """What k_col_stats + k_bn_finalize + k_affine_act return for an fp32 z [..., F]: per block of STAT_ROWS rows and
    row lane rr (rl = 256 / min(F, 256) lanes), an fp32 running sum of d = z - K and fma(d, d, q) with K = z[0] (the
    shifted accumulation), the lanes added in fp32, the blocks in fp64; then mean = K + S/n, var = Q/n - (S/n)^2 in fp64,
    invstd = fp32(1 / sqrt(var + eps)), scale = gamma invstd, shift = beta - fp32(mean) scale, y = fma(z, scale, shift).
    `mutation` (one of BN_MUTATIONS) plants one defect.  Returns (y, mean, invstd, rm_new, rv_new) as float64."""
    f32 = np.float32
    zr = np.asarray(z, f32).reshape(-1, np.shape(z)[-1])
    n, F = zr.shape
    rl = 256 // min(F, 256)
    K = np.zeros(F, f32) if mutation == "one_pass" else zr[0].copy()
    S, Q = np.zeros(F), np.zeros(F)
    for r0 in range(0, n, STAT_ROWS):
        blk = zr[r0:r0 + STAT_ROWS]
        s_l, q_l = np.zeros((rl, F), f32), np.zeros((rl, F), f32)
        for i in range(0, blk.shape[0], rl):
            v = (blk[i:i + rl] - K).astype(f32)
            k = v.shape[0]
            s_l[:k] = (s_l[:k] + v).astype(f32)
            q_l[:k] = (v.astype(np.float64) * v + q_l[:k]).astype(f32)                # fma: one rounding
        s, q = s_l[0].copy(), q_l[0].copy()
        for j in range(1, rl):
            s, q = (s + s_l[j]).astype(f32), (q + q_l[j]).astype(f32)
        S, Q = S + s, Q + q
    d = S / n
    mean = K.astype(np.float64) + d
    var = np.maximum(Q / n - d * d, 0.0)
    unb = var * n / (n - 1) if n > 1 else var
    eps = 1e-3 if mutation == "eps_1e-3" else eps
    v_norm = unb if mutation == "unbiased_in_norm" else var
    if mutation == "eps_outside_sqrt":
        invstd = (1.0 / (np.sqrt(v_norm) + eps)).astype(f32)
    else:
        invstd = (1.0 / np.sqrt(v_norm + eps)).astype(f32)
    mom = f32(0.01) if mutation == "momentum_0.01" else f32(momentum)
    v_run = var if mutation == "biased_in_running" else unb
    rm_new = (f32(1) - mom) * np.asarray(rm, f32) + mom * mean.astype(f32)
    rv_new = (f32(1) - mom) * np.asarray(rv, f32) + mom * v_run.astype(f32)
    sc = (np.asarray(gamma, f32) * invstd).astype(f32)
    sh = (np.asarray(beta, f32) - (mean.astype(f32) * sc).astype(f32)).astype(f32)
    if mutation == "relu_before_affine":
        zr = np.maximum(zr, f32(0))
    y = (zr.astype(np.float64) * sc + sh).astype(f32)
    if relu and mutation != "relu_before_affine":
        y = np.maximum(y, f32(0))
    return (y.astype(np.float64).reshape(np.shape(z)), mean, invstd.astype(np.float64), rm_new.astype(np.float64),
            rv_new.astype(np.float64))


BN_BWD_MUTATIONS = ("m2_dropped", "mean_not_subtracted", "rows_minus_one")


def emulate_bn_bwd(z, g_a, gamma, beta, mean, invstd, relu=False, mutation: str = "", mask=None, frozen=False):
    """What k_bn_bwd_reduce + k_bn_bwd_coef + k_bn_bwd_apply4 return for fp32 z, g_a [..., F] and the saved fp32
    mean / invstd: per block of STAT_ROWS rows and row lane (as emulate_bn_train) fp32 sums s1 = sum g' and
    s2 = fma(g', zhat, s2) with zhat = fp32((z - mean) invstd), blocks in fp64; then in fp32 m1 = s1 / n, m2 = s2 / n,
    a = gamma invstd, b = -a invstd m2, c = -a m1 + a invstd m2 mean and g_z = fma(a, g', fma(b, z, c)).  The mask
    g' = g_a [fma(z, scale, shift) > 0] uses scale = gamma invstd, shift = beta - mean scale like the forward.
    `mutation` (one of BN_BWD_MUTATIONS) plants one defect.  mask (bool): the ReLU's open entries as given (the device's
    relu_mask) in place of the emulated test.  frozen: the running-statistics backward, g_z = fp32(a g') (b = c = 0;
    mean / invstd are then the running mean and the fp32 1 / sqrt(rv + eps)).  Returns (g_z, dgamma, dbeta) as
    float64."""
    f32 = np.float32
    zr = np.asarray(z, f32).reshape(-1, np.shape(z)[-1])
    gr = np.asarray(g_a, f32).reshape(zr.shape)
    n, F = zr.shape
    mu, ist = np.asarray(mean, f32), np.asarray(invstd, f32)
    gam = np.asarray(gamma, f32)
    sc = (gam * ist).astype(f32)
    sh = (np.asarray(beta, f32) - (mu * sc).astype(f32)).astype(f32)
    if mask is not None:
        gr = np.where(np.asarray(mask).reshape(zr.shape), gr, f32(0))
    elif relu:
        gr = np.where((zr.astype(np.float64) * sc + sh).astype(f32) > 0, gr, f32(0))
    zh = (((zr - mu).astype(f32)) * ist).astype(f32)
    rl = 256 // min(F, 256)
    S, Q = np.zeros(F), np.zeros(F)
    for r0 in range(0, n, STAT_ROWS):
        gb, hb = gr[r0:r0 + STAT_ROWS], zh[r0:r0 + STAT_ROWS]
        s_l, q_l = np.zeros((rl, F), f32), np.zeros((rl, F), f32)
        for i in range(0, gb.shape[0], rl):
            k = gb[i:i + rl].shape[0]
            s_l[:k] = (s_l[:k] + gb[i:i + rl]).astype(f32)
            q_l[:k] = (gb[i:i + rl].astype(np.float64) * hb[i:i + rl] + q_l[:k]).astype(f32)
        s, q = s_l[0].copy(), q_l[0].copy()
        for j in range(1, rl):
            s, q = (s + s_l[j]).astype(f32), (q + q_l[j]).astype(f32)
        S, Q = S + s, Q + q
    rows = n - 1 if mutation == "rows_minus_one" else n
    m1, m2 = (S / rows).astype(f32), (Q / rows).astype(f32)
    if mutation == "m2_dropped":
        m2 = np.zeros(F, f32)
    a = (gam * ist).astype(f32)
    if frozen:
        g_z = (a.astype(np.float64) * gr).astype(f32)
        return (g_z.astype(np.float64).reshape(np.shape(z)), Q.astype(f32).astype(np.float64),
                S.astype(f32).astype(np.float64))
    b = (-(a * ist).astype(f32) * m2).astype(f32)
    t = (((a * ist).astype(f32) * m2).astype(f32) * mu).astype(f32)
    c = (-(a * m1).astype(f32) + (f32(0) if mutation == "mean_not_subtracted" else t)).astype(f32)
    inner = (b.astype(np.float64) * zr + c).astype(f32)
    g_z = (a.astype(np.float64) * gr + inner).astype(f32)
    return g_z.astype(np.float64).reshape(np.shape(z)), Q.astype(f32).astype(np.float64), S.astype(f32).astype(np.float64)


def bound_ratio(y, y64, bound) -> float:
    """max_ij |y - y64| / bound (<= 1 passes); inf where the kernel returned a non-finite value."""
    y = np.asarray(y, np.float64)
    if not np.all(np.isfinite(y)):
        return float("inf")
    return float((np.abs(y - y64) / np.maximum(bound, 1e-300)).max(initial=0.0))


# --------------------------------------------------------------------------------------------- PoseNet layer by layer
def relu_mask(z, scale, shift) -> np.ndarray:
    """The kernels' activation test fmaf(z, scale, shift) > 0 for fp32 z, scale, shift, reproduced bit for bit: the
    float64 product of two fp32 values is exact (48 significant bits), and the one rounding of the float64 sum to
    nearest cannot change the sign of a non-zero exact sum (nor make it zero), so its sign is the exact sum's, which
    is also the sign of fmaf's single fp32 rounding of it.  Two conditions, both far from any real pre-activation:
    |z scale| must not underflow float64's normal range (2^-1022), or the product is not exact; and |exact sum| must
    exceed 2^-150, below which fmaf rounds to zero and the kernel closes the ReLU where relu_mask opens it (the
    library is built without flushing subnormals to zero)."""
    z = np.asarray(z, np.float32).astype(np.float64)
    return z * np.asarray(scale, np.float32).astype(np.float64) + np.asarray(shift, np.float32).astype(np.float64) > 0


TC_MMAS_PER_BLOCK = 6      # launch_umma_gemm's k16 MMAs per 32-wide K-block: hi*hi x2, lo*hi x2, hi*lo x2


def tc_running_sums(A, B) -> np.ndarray:
    """sum over the k16 wgmma steps of launch_umma_gemm of |the accumulator after the step|, per element of A @ B, in
    the kernel's order: per K-block of 32 columns hi*hi over its first and second 16 columns, then lo*hi and hi*lo over
    both (cheb_umma.cu's main loop), so the accumulator holds the float64 partial sum S after the block's first 16
    columns once and S after all 32 five times.  The lo products move those sums by <= 2^-10 of their magnitude, a
    second-order term next to the truncation they bound.  K is padded with zeros to a multiple of 32."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    S = np.zeros((A.shape[0], B.shape[1]))
    acc = np.zeros_like(S)
    for k0 in range(0, A.shape[1], 32):
        S = S + A[:, k0:k0 + 16] @ B[k0:k0 + 16]
        acc += np.abs(S)
        S = S + A[:, k0 + 16:k0 + 32] @ B[k0 + 16:k0 + 32]
        acc += (TC_MMAS_PER_BLOCK - 1) * np.abs(S)
    return acc


def dense_gemm_bound(A, B, precision: str, b_side: str = "fixed") -> np.ndarray:
    """Element-wise bound on C = A @ B (A [m, k], B [k, n]) from one of PoseNet's GEMMs given its exact fp32 operands.
    fp32 (CUDA cores, FMA): gamma_k |A| |B|.
    fp16x3 (launch_umma_gemm), worst case per element rather than a probabilistic sum:
      * the split: SPLIT_TERM["fp16x3"] |A| |B| (two lo roundings and the dropped lo*lo product, as in gamma);
      * the accumulation: every k16 wgmma adds its products (exact in fp32) to the fp32 accumulator and truncates the
        result (round toward zero: Fasi et al., PeerJ Comput. Sci. 7:e330, 2021), an error below one ulp, i.e.
        < 2 u |accumulator after the step|.  Summed over the kernel's steps that is 2 u tc_running_sums(A, B): it
        grows linearly where the partial sums keep one sign (a dW over a short K = B), and stays small where they
        cancel (the K = H forward and dX GEMMs);
      * the floor of the lo parts: A, the activation or gradient operand, is always range-normalised (max|A| scaled
        into [2^9, 2^10), so a lo part's absolute error, half of fp16's subnormal spacing 2^-24 in the scaled units, is
        <= 2^-34 max|A|); B enters at the fixed 2^6 when it is a weight matrix (b_side='fixed': 2^-25 / 2^6 per
        entry), range-normalised like A when it is an activation (b_side='normalised', dW's a: 2^-34 max|B|).  The
        floor of an entry is its operand's absolute error times the other operand's absolute sums along k."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    aA, aB = np.abs(A), np.abs(B)
    if precision != "fp16x3":
        return gamma(A.shape[1], precision) * (aA @ aB)
    e = SPLIT_TERM["fp16x3"] * (aA @ aB) + 2 * U32 * tc_running_sums(A, B)
    e_a = 2.0 ** -34 * float(aA.max(initial=0.0))
    e_b = NET_LO / NET_W_SCALE if b_side == "fixed" else 2.0 ** -34 * float(aB.max(initial=0.0))
    return e + e_a * aB.sum(axis=0, keepdims=True) + e_b * aA.sum(axis=1, keepdims=True)


def emulate_dense_gemm(A, B, b_side: str = "fixed", drop_block: int = -1, a_scale: float | None = None,
                       drop_lo: str = "") -> np.ndarray:
    """What launch_umma_gemm returns for C = A @ B with fp32 operands: A scaled by a_scale (default: the power of two
    _pow2_scale(max|A|) the library finds), B by the fixed 2^6 (b_side='fixed') or by its own power of two, each split
    into fp16 hi + lo, hi*hi + lo*hi + hi*lo summed per K-block of 32 in float64 and accumulated over the blocks in fp32
    (a slightly better accumulator than the tensor core's), both scales divided out.  drop_block >= 0 leaves out the
    lo(A) * hi(B) products of K-block `drop_block`; drop_lo='a' leaves out every lo(A) * hi(B) product, 'b' every
    hi(A) * lo(B) (an fp16x2 split of one operand)."""
    A = np.asarray(A, np.float32).astype(np.float64)
    B = np.asarray(B, np.float32).astype(np.float64)
    sa = _pow2_scale(float(np.abs(A).max(initial=0.0))) if a_scale is None else a_scale
    sb = NET_W_SCALE if b_side == "fixed" else _pow2_scale(float(np.abs(B).max(initial=0.0)))
    with np.errstate(over="ignore", invalid="ignore"):
        ah, al = _f16_split(A * sa)
        bh, bl = _f16_split(B * sb)
    if drop_lo == "a":
        al = 0.0 * al
    elif drop_lo == "b":
        bl = 0.0 * bl
    acc = np.zeros((A.shape[0], B.shape[1]), np.float32)
    for k0 in range(0, A.shape[1], 32):
        k = slice(k0, k0 + 32)
        lo = al[:, k] if k0 // 32 != drop_block else 0.0 * al[:, k]
        acc = (acc + (ah[:, k] @ bh[k] + lo @ bh[k] + ah[:, k] @ bl[k]).astype(np.float32)).astype(np.float32)
    return acc.astype(np.float64) / (sa * sb)


def bn_frozen_bwd(z, g, gamma, rm, rv, eps=BN_EPS):
    """Backward of a BatchNorm with running statistics (frozen: mean and variance are constants of the forward) from
    the masked gradient g' = g [relu open] of its output: g_z = gamma invstd g', dgamma = sum g' zhat, dbeta = sum g',
    with invstd = 1 / sqrt(rv + eps) and zhat = (z - rm) invstd.  Returns (g_z, dgamma, dbeta)."""
    zr, gr = _rows(z), _rows(g)
    invstd = 1.0 / np.sqrt(np.asarray(rv, np.float64) + eps)
    zh = (zr - np.asarray(rm, np.float64)) * invstd
    g_z = np.asarray(gamma, np.float64) * invstd * gr
    return g_z.reshape(np.shape(z)), (gr * zh).sum(axis=0), gr.sum(axis=0)


def bn_frozen_bwd_bound(z, g, gamma, rm, rv, eps=BN_EPS):
    """Bounds (g_z, dgamma, dbeta) on the frozen backward of launch_bn_relu_bwd, given the exact fp32 z and g' it read.
      invstd = 1.f / sqrtf(rv + (float)eps) (k_bn_fold_eval): eps's cast and the sum 2 u relative, halved by the
      square root, plus the root's and the division's roundings: 3 u relative;
      g_z = fp32(fp32(gamma invstd) g'): one rounding in the coefficient, one in the product: 5 u |g_z| in all;
      zhat = fp32(fp32(z - rm) invstd): the difference, the product and invstd's 3 u: 5 u |zhat|;
      dgamma, dbeta: the fp32 block sums of k_bn_bwd_reduce (stat_allowance), with dgamma's terms carrying zhat's
      error, and the final fp32 rounding of the fp64 total.
    The first-order bound is raised by one u in g_z for the products of the relative errors (O(u^2))."""
    zr, gr = _rows(z), _rows(g)
    n, F = zr.shape
    g_z, dgam, dbet = bn_frozen_bwd(z, g, gamma, rm, rv, eps)
    invstd = 1.0 / np.sqrt(np.asarray(rv, np.float64) + eps)
    azh = np.abs(zr - np.asarray(rm, np.float64)) * invstd
    ag = np.abs(gr)
    al = stat_allowance(n, F)
    e_gz = 6 * U32 * np.abs(_rows(g_z))
    e_dgam = al * (ag * azh).sum(axis=0) + 5 * U32 * (ag * azh).sum(axis=0) + U32 * np.abs(dgam)
    e_dbet = al * ag.sum(axis=0) + U32 * np.abs(dbet)
    return e_gz.reshape(np.shape(z)), e_dgam, e_dbet
