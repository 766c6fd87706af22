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
gamma_K, fp32 (CUDA cores, FMA): only the last line.

floor (only matters where |A||B| is tiny, i.e. a row of zeros or an entry of exact cancellation): fp16's subnormal
spacing 2^-24 bounds the absolute error of a lo part.  The operands enter the split scaled into [2^(9-h), 2^(10-h))
by a power of two (h = 0 for the weights, h = ceil(log2(2 r^2 + 1)) for the basis, r = max absolute row sum of L~),
so the absolute error per operand entry is <= 2^(h-34) max|operand| and the floor is that times the other operand's
absolute row sum.  It scales with the inputs: it is never an absolute constant.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp

U32 = 2.0 ** -24          # fp32 unit roundoff
SPLIT = 3 * 2.0 ** -22    # fp16x3: two lo roundings + the dropped lo*lo term
LAMBDA = 1.0              # probabilistic accumulation constant (see the module docstring)


def gamma(k: int, precision: str, deg: int = 0) -> float:
    acc = LAMBDA * (math.sqrt(3 * k) + math.sqrt(2 * deg + 3)) * U32
    return acc + (SPLIT if precision == "fp16x3" else 0.0)


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


def cheb_conv_fwd_bound(x, L, W, b, precision: str) -> np.ndarray:
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
    fl = (2.0 ** (h - 34) * float(ax.max(initial=0.0)) * np.abs(W).sum(axis=1)[None, :]
          + 2.0 ** -34 * float(np.abs(W).max(initial=0.0)) * Ta.sum(axis=1, keepdims=True))
    return (bound + fl).reshape(B, V, -1)


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
    dW = np.einsum("ro,rkf->ofk", dzf, T.reshape(B * V, 3, F)).reshape(fout, 3 * F)
    db = dzf.sum(axis=0)
    return dx, dW, db


def cheb_conv_bwd_bound(x, L, W, dz, precision: str):
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
    Fl = [(2.0 ** -34 * (mdz * Wk[:, :, k].sum(axis=0)[None, :] + mw * dzf.sum(axis=1, keepdims=True))).reshape(B, V, F)
          for k in range(3)]
    g_dx = gamma(fout, precision, deg)
    b_dx = g_dx * prop(*A) + prop(*Fl)
    # dW: contraction over all B*V rows of |dz| and the absolute basis
    Tabs = basis(ax, Labs)
    Tabs[:, :, 2] += 2 * ax
    Tf = Tabs.reshape(B * V, 3, F)
    R = B * V
    g_dw = gamma(R, precision, deg) + (R.bit_length() * U32)   # + the cross-CTA fp32 atomic adds (log-depth tree)
    b_dw = g_dw * np.einsum("ro,rkf->ofk", dzf, Tf).reshape(fout, 3 * F)
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


def emulate_cheb_conv(x, L, W, b=None, mode: str = "fp16x3", drop_block: int = -1) -> np.ndarray:
    """What a tensor-core kernel of the given arithmetic returns for the conv: the basis in fp32, the operands scaled
    by powers of two into fp16's range (h of headroom for the basis), then
      'fp16x3'    hi*hi + lo*hi + hi*lo
      'fp16'      hi*hi only
      'tf32'      both operands rounded to TF32
    accumulated in fp32 over K (sequentially, products of one k summed in float64 first: a slightly better accumulator
    than the tensor core's).  drop_block >= 0 removes the lo*hi products of the 32 consecutive K-columns (of the
    kernel's [k][fin] operand order) that make up K-block `drop_block`."""
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


def emulate_bn_train(z, gamma, beta, rm, rv, relu=False, mutation: str = ""):
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
    eps = 1e-3 if mutation == "eps_1e-3" else BN_EPS
    v_norm = unb if mutation == "unbiased_in_norm" else var
    if mutation == "eps_outside_sqrt":
        invstd = (1.0 / (np.sqrt(v_norm) + eps)).astype(f32)
    else:
        invstd = (1.0 / np.sqrt(v_norm + eps)).astype(f32)
    mom = f32(0.01) if mutation == "momentum_0.01" else f32(0.1)
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


def bound_ratio(y, y64, bound) -> float:
    """max_ij |y - y64| / bound (<= 1 passes); inf where the kernel returned a non-finite value."""
    y = np.asarray(y, np.float64)
    if not np.all(np.isfinite(y)):
        return float("inf")
    return float((np.abs(y - y64) / np.maximum(bound, 1e-300)).max(initial=0.0))
