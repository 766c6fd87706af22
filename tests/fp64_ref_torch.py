"""tests/fp64_ref.py in torch float64, on any device, for the sizes the network runs at.

fp64_ref.py stays the specification: every function here computes the same quantity by the same formula (its CPU
cross-check is tests/test_fp64_torch_ref_cpu.py), only laid out for a batch of a few million rows:

* the Laplacian is a float64 CSR tensor (Lap: L, |L| and their transposes), applied to [V, meshes * F] slices;
* the contractions are dense float64 matmuls (DGEMM on a GPU);
* per-row quantities are computed `chunk` meshes at a time (chunk=None: all at once) into one float64 output, and the
  batch-wide ones (dW, db, the BatchNorm statistics, dgamma / dbeta, the column sums of the floors) are accumulated
  in float64 across chunks, so the temporaries of a 128-wide 12288-row level at B = 256 stay at one chunk's size.

Inputs are torch tensors of any float dtype (numpy arrays are taken as they are); outputs are float64 on the input's
device.  Scalars (gamma, stat_allowance, the resample tables) come from fp64_ref itself."""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp
import torch

import fp64_ref as R

F64 = torch.float64


def t64(a, device=None) -> torch.Tensor:
    if isinstance(a, torch.Tensor):
        return a.to(device=device or a.device, dtype=F64)
    return torch.as_tensor(np.asarray(a, np.float64), device=device)


def _csr(m: sp.csr_matrix, device) -> torch.Tensor:
    m = sp.csr_matrix(m, dtype=np.float64)
    m.sort_indices()
    return torch.sparse_csr_tensor(torch.as_tensor(m.indptr.astype(np.int64)),
                                   torch.as_tensor(m.indices.astype(np.int64)),
                                   torch.as_tensor(m.data), size=m.shape, dtype=F64, device=device)


class Lap:
    """One level's Laplacian on a device: L, |L|, L^T, |L|^T as float64 CSR, its largest row length and the headroom
    h of the basis (fp64_ref.max_degree, fp64_ref.headroom_log2)."""

    def __init__(self, L, device="cpu"):
        c = sp.csr_matrix(L, dtype=np.float64)
        self.V = c.shape[0]
        self.L, self.LT = _csr(c, device), _csr(c.T.tocsr(), device)
        a = abs(c)
        self.A, self.AT = _csr(a, device), _csr(a.T.tocsr(), device)
        self.deg = R.max_degree(c)
        self.h = R.headroom_log2(c)


def lap(L, device="cpu") -> Lap:
    return L if isinstance(L, Lap) else Lap(L, device)


def _chunks(B: int, chunk):
    c = B if not chunk else int(chunk)
    return [slice(i, min(B, i + c)) for i in range(0, B, c)]


def _apply(M: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """M (CSR [V, V]) applied to every mesh of x [b, V, F]."""
    b, V, F = x.shape
    y = torch.sparse.mm(M, x.permute(1, 0, 2).reshape(V, b * F))
    return y.reshape(V, b, F).permute(1, 0, 2)


def _basis(x, M) -> torch.Tensor:
    """[b, V, 3, F]: [x | M x | 2 M (M x) - x]."""
    t1 = _apply(M, x)
    return torch.stack([x, t1, 2 * _apply(M, t1) - x], dim=2)


def _abs_basis(ax, lp: Lap) -> torch.Tensor:
    """[|x|, |L||x|, 2|L|(|L||x|) + |x|] of ax = |x|."""
    t1 = _apply(lp.A, ax)
    return torch.stack([ax, t1, 2 * _apply(lp.A, t1) + ax], dim=2)


def _flat(T) -> torch.Tensor:
    """[b, V, 3, F] -> [b V, 3 F] with the reference's column order f*3 + k."""
    b, V, K, F = T.shape
    return T.permute(0, 1, 3, 2).reshape(b * V, F * K)


def _contract_rows(dz, T) -> torch.Tensor:
    """sum_rows dz[:, o] T[:, k, f] -> [o, f*3 + k]."""
    Rr, K, F = T.shape
    return (dz.T @ T.reshape(Rr, K * F)).reshape(-1, K, F).permute(0, 2, 1).reshape(-1, F * K)


def basis(x, L, chunk=None) -> torch.Tensor:
    x = t64(x)
    lp = lap(L, x.device)
    out = torch.empty(x.shape[0], x.shape[1], 3, x.shape[2], dtype=F64, device=x.device)
    for c in _chunks(x.shape[0], chunk):
        out[c] = _basis(x[c], lp.L)
    return out


# --------------------------------------------------------------------------------------------- Chebyshev conv (K = 3)
def cheb_conv_fwd(x, L, W, b=None, chunk=None) -> torch.Tensor:
    x = t64(x)
    dv = x.device
    lp, W = lap(L, dv), t64(W, dv)
    B, V, _ = x.shape
    out = torch.empty(B, V, W.shape[0], dtype=F64, device=dv)
    for c in _chunks(B, chunk):
        y = _flat(_basis(x[c], lp.L)) @ W.T
        if b is not None:
            y = y + t64(b, dv)
        out[c] = y.reshape(-1, V, W.shape[0])
    return out


def _abs_contraction(ax, lp, aW) -> torch.Tensor:
    Ta = _flat(_abs_basis(ax, lp))
    return Ta, Ta @ aW.T


def cheb_conv_fwd_bound(x, L, W, b, precision: str, split: str = "normalised", chunk=None) -> torch.Tensor:
    x = t64(x)
    dv = x.device
    lp, aW = lap(L, dv), t64(W, dv).abs()
    B, V, F = x.shape
    g = R.gamma(3 * F, precision, lp.deg)
    mx = float(x.abs().max()) if x.numel() else 0.0
    mw = float(aW.max()) if aW.numel() else 0.0
    wsum = aW.sum(dim=1)[None, :]
    out = torch.empty(B, V, aW.shape[0], dtype=F64, device=dv)
    for c in _chunks(B, chunk):
        Ta, TW = _abs_contraction(x[c].abs(), lp, aW)
        bound = g * TW
        if b is not None:
            bound = bound + R.U32 * t64(b, dv).abs()
        if split == "network":
            fl = R.NET_LO * wsum + R.NET_LO / R.NET_W_SCALE * Ta.sum(dim=1, keepdim=True)
        else:
            fl = 2.0 ** (lp.h - 34) * mx * wsum + 2.0 ** -34 * mw * Ta.sum(dim=1, keepdim=True)
        out[c] = (bound + fl).reshape(-1, V, aW.shape[0])
    return out


def cheb_conv_bwd(x, L, W, dz, chunk=None):
    """(dx, dW, db) of fp64_ref.cheb_conv_bwd; dW and db summed over the chunks in float64."""
    x, dz = t64(x), t64(dz)
    dv = x.device
    lp, W = lap(L, dv), t64(W, dv)
    B, V, F = x.shape
    fout = W.shape[0]
    Wk = W.reshape(fout, F, 3)
    dx = torch.empty(B, V, F, dtype=F64, device=dv)
    dW = torch.zeros(fout, 3 * F, dtype=F64, device=dv)
    db = torch.zeros(fout, dtype=F64, device=dv)
    for c in _chunks(B, chunk):
        dzf = dz[c].reshape(-1, fout)
        dT = [(dzf @ Wk[:, :, k]).reshape(-1, V, F) for k in range(3)]
        dx[c] = dT[0] - dT[2] + _apply(lp.LT, dT[1] + 2 * _apply(lp.LT, dT[2]))
        dW += _contract_rows(dzf, _basis(x[c], lp.L).reshape(-1, 3, F))
        db += dzf.sum(dim=0)
    return dx, dW, db


def cheb_conv_bwd_bound(x, L, W, dz, precision: str, split: str = "normalised", dw_chain=0, chunk=None,
                        precision_dw: str | None = None, with_default: bool = False):
    """Bounds (dx, dW, db) of fp64_ref.cheb_conv_bwd_bound, including its dw_chain.  precision_dw: dW's precision when
    it runs on another path than dX (default: precision).  with_default: also return dW's bound without dw_chain (the
    two differ only in the factor of the contraction), as a fourth item."""
    precision_dw = precision_dw or precision
    x, dz = t64(x), t64(dz)
    dv = x.device
    lp, aW = lap(L, dv), t64(W, dv).abs()
    B, V, F = x.shape
    fout = aW.shape[0]
    Wk = aW.reshape(fout, F, 3)
    mdz = float(dz.abs().max()) if dz.numel() else 0.0
    mw = float(aW.max()) if aW.numel() else 0.0
    mx = float(x.abs().max()) if x.numel() else 0.0
    e_dz = 2.0 ** -34 * mdz
    e_w = R.NET_LO / R.NET_W_SCALE if split == "network" else 2.0 ** -34 * mw
    g_dx = R.gamma(fout, precision, lp.deg)
    wk_sum = [Wk[:, :, k].sum(dim=0)[None, :] for k in range(3)]
    b_dx = torch.empty(B, V, F, dtype=F64, device=dv)
    con = torch.zeros(fout, 3 * F, dtype=F64, device=dv)        # sum_rows |dz| (x) |T|
    t_sum = torch.zeros(F, 3, dtype=F64, device=dv)             # sum_rows |T|, [f, k]
    dz_sum = torch.zeros(fout, dtype=F64, device=dv)            # sum_rows |dz|
    x_sum = torch.zeros(F, dtype=F64, device=dv)                # sum_rows |x|
    tdz_sum = torch.zeros(3, fout, dtype=F64, device=dv)        # sum_rows |T(dz)|, [k, o]

    def prop(a0, a1, a2):
        return a0 + a2 + _apply(lp.AT, a1 + 2 * _apply(lp.AT, a2))

    for c in _chunks(B, chunk):
        adz, ax = dz[c].abs(), x[c].abs()
        dzf = adz.reshape(-1, fout)
        A = [(dzf @ Wk[:, :, k]).reshape(-1, V, F) for k in range(3)]
        rs = dzf.sum(dim=1, keepdim=True)
        Fl = [(e_dz * wk_sum[k] + e_w * rs).reshape(-1, V, F) for k in range(3)]
        fl_dx = prop(*Fl)
        if split == "network":
            Tdz = _abs_basis(adz, lp)
            conv_fl = e_dz * Wk.sum(dim=(0, 2))[None, :] + e_w * Tdz.reshape(dzf.shape[0], -1).sum(dim=1, keepdim=True)
            fl_dx = torch.maximum(fl_dx, conv_fl.reshape(-1, V, F))
            tdz_sum += Tdz.reshape(-1, 3, fout).sum(dim=0)
            del Tdz
        b_dx[c] = g_dx * prop(*A) + fl_dx
        del A, Fl, fl_dx
        Tf = _abs_basis(ax, lp).reshape(-1, 3, F)
        con += _contract_rows(dzf, Tf)
        t_sum += Tf.sum(dim=0).T
        dz_sum += dzf.sum(dim=0)
        x_sum += ax.reshape(-1, F).sum(dim=0)
    Rn = B * V
    g_dw0 = dw_gamma_default(Rn, precision_dw, lp.deg)
    g_dw = g_dw0
    if dw_chain:
        g_dw = max(g_dw, dw_chain * R.U32 + R.SPLIT_TERM[precision_dw])
    if split == "network":
        on_x = e_dz * t_sum.reshape(1, 3 * F) + R.NET_LO * dz_sum[:, None]
        on_dz = (e_dz * torch.repeat_interleave(x_sum, 3)[None, :]
                 + R.NET_LO * tdz_sum.T[:, None, :].expand(fout, F, 3).reshape(fout, 3 * F))
        fl_dw = torch.maximum(on_x, on_dz)
    else:
        fl_dw = 2.0 ** -34 * mdz * t_sum.reshape(1, 3 * F) + 2.0 ** (lp.h - 34) * mx * dz_sum[:, None]
    out = (b_dx, g_dw * con + fl_dw, 2 * R.U32 * dz_sum)
    return out + (g_dw0 * con + fl_dw,) if with_default else out


def dw_gamma_default(n_rows: int, precision: str, deg: int) -> float:
    """The accumulation factor cheb_conv_bwd_bound holds dW to without dw_chain."""
    return R.gamma(n_rows, precision, deg) + n_rows.bit_length() * R.U32


# --------------------------------------------------------------------------------------------- BatchNorm1d over rows
def _cols(z, chunk, fn) -> list:
    """Column sums over every row, in one pass over the chunks: fn(chunk) returns a tuple of [r, F] tensors, the
    result is the list of their sums over all rows ([F] each, float64)."""
    acc = None
    for c in _chunks(z.shape[0], chunk):
        s = [t.sum(dim=0) for t in fn(c)]
        acc = s if acc is None else [a + b for a, b in zip(acc, s)]
    return acc


def _col(z, chunk, fn) -> torch.Tensor:
    """sum over every row of fn(rows of one chunk [r, F]) -> [F], float64."""
    return _cols(z, chunk, lambda c: (fn(c),))[0]


def _r(t, c) -> torch.Tensor:
    """rows [r, F] of chunk c of a [B, ..., F] tensor, as float64."""
    return t[c].to(F64).reshape(-1, t.shape[-1])


def _n_rows(z) -> int:
    return int(np.prod(z.shape[:-1]))


def _mean_var(z, chunk):
    n = _n_rows(z)
    mean = _col(z, chunk, lambda c: _r(z, c)) / n
    var = _col(z, chunk, lambda c: (_r(z, c) - mean) ** 2) / n
    return mean, var


def bn_train_fwd(z, gamma, beta, rm, rv, relu=False, eps=R.BN_EPS, momentum=R.BN_MOMENTUM, chunk=None):
    """(y, mean, biased var, new running_mean, new running_var) of fp64_ref.bn_train_fwd; z [B, ..., F]."""
    dv = z.device
    n = _n_rows(z)
    mean, var = _mean_var(z, chunk)
    g, b = t64(gamma, dv), t64(beta, dv)
    y = torch.empty(z.shape, dtype=F64, device=dv)
    inv = torch.sqrt(var + eps)
    for c in _chunks(z.shape[0], chunk):
        yc = (_r(z, c) - mean) / inv * g + b
        y[c] = (torch.clamp_min(yc, 0.0) if relu else yc).reshape(y[c].shape)
    unbiased = var * n / (n - 1) if n > 1 else var
    rm_new = (1 - momentum) * t64(rm, dv) + momentum * mean
    rv_new = (1 - momentum) * t64(rv, dv) + momentum * unbiased
    return y, mean, var, rm_new, rv_new


def _bn_fwd_cols(z, E, gamma, beta, eps, chunk):
    """The column quantities of fp64_ref.bn_train_fwd_bound (E None: zero)."""
    dv = z.device
    n, F = _n_rows(z), z.shape[-1]
    mean, var = _mean_var(z, chunk)
    sig = torch.sqrt(var + eps)
    z0 = z.reshape(-1, F)[0].to(F64)

    def er(c):
        e = R.U32 * _r(z, c).abs()
        return e if E is None else e + _r(E, c)

    def shifted(c):
        d = _r(z, c) - z0
        return er(c), d.abs(), d * d, d

    mE, D, Q2, dm = (t / n for t in _cols(z, chunk, shifted))
    mzE = _col(z, chunk, lambda c: ((_r(z, c) - mean).abs() / sig) * er(c)) / n
    a = R.stat_allowance(n, F)
    d_mean = a * D + R.U32 * mean.abs()
    d_var_local = a * Q2 + 2 * dm.abs() * a * D
    d_var = d_var_local + 2 * sig * mzE
    rel_is = d_var_local / (2 * sig ** 2) + 2 * R.U32
    g, b = t64(gamma, dv).abs(), t64(beta, dv).abs()
    return dict(n=n, mean=mean, var=var, sig=sig, mE=mE, mzE=mzE, d_mean=d_mean, d_var=d_var, rel_is=rel_is, g=g, b=b,
                er=er)


def bn_train_fwd_bound(z, E, gamma, beta, rm, rv, eps=R.BN_EPS, momentum=R.BN_MOMENTUM, chunk=None):
    """fp64_ref.bn_train_fwd_bound (E None: the exact z, E = 0)."""
    dv = z.device
    s = _bn_fwd_cols(z, E, gamma, beta, eps, chunk)
    mean, sig, g, b = s["mean"], s["sig"], s["g"], s["b"]
    sc = g / sig
    ey = torch.empty(z.shape, dtype=F64, device=dv)
    for c in _chunks(z.shape[0], chunk):
        zh = (_r(z, c) - mean).abs() / sig
        e = (sc * (s["er"](c) + s["mE"] + zh * s["mzE"]) + sc * s["d_mean"] + g * zh * s["rel_is"]
             + R.U32 * (2 * g * zh + 3 * sc * mean.abs() + 2 * b))
        ey[c] = e.reshape(ey[c].shape)
    n = s["n"]
    unb = n / (n - 1) if n > 1 else 1.0
    e_rm = momentum * (s["mE"] + s["d_mean"]) + 4 * R.U32 * ((1 - momentum) * t64(rm, dv).abs() + momentum * mean.abs())
    e_rv = momentum * unb * s["d_var"] + 4 * R.U32 * ((1 - momentum) * t64(rv, dv).abs() + momentum * unb * s["var"])
    e_is = (1 / sig) * (s["rel_is"] + s["mzE"] / sig)
    return dict(y=ey, mean=s["mE"] + s["d_mean"], invstd=e_is, rm=e_rm, rv=e_rv)


def bn_eval_fwd(z, gamma, beta, rm, rv, relu=False, eps=R.BN_EPS, chunk=None):
    dv = z.device
    g, b, m, v = (t64(a, dv) for a in (gamma, beta, rm, rv))
    y = torch.empty(z.shape, dtype=F64, device=dv)
    for c in _chunks(z.shape[0], chunk):
        yc = (z[c].to(F64) - m) / torch.sqrt(v + eps) * g + b
        y[c] = torch.clamp_min(yc, 0.0) if relu else yc
    return y


def bn_eval_fwd_bound(z, E, gamma, beta, rm, rv, bias, eps=R.BN_EPS, chunk=None):
    """fp64_ref.bn_eval_fwd_bound."""
    dv = z.device
    g, b, m, v, bias = (t64(a, dv) for a in (gamma, beta, rm, rv, bias))
    sc = g.abs() / torch.sqrt(v + eps)
    bm = (bias - m).abs()
    out = torch.empty(z.shape, dtype=F64, device=dv)
    for c in _chunks(z.shape[0], chunk):
        zc = z[c].to(F64)
        y = ((zc - m) / torch.sqrt(v + eps) * g + b).abs()
        out[c] = sc * E[c].to(F64) + R.U32 * (4 * (zc - bias).abs() * sc + 3 * bm * sc + 2 * b.abs() + 2 * y)
    return out


def _bwd_cols(z, g_a, gamma, beta, relu, eps, mask, chunk):
    dv = z.device
    n = _n_rows(z)
    mean, var = _mean_var(z, chunk)
    invstd = 1.0 / torch.sqrt(var + eps)
    gam, bet = t64(gamma, dv), t64(beta, dv)

    def parts(c):
        zh = (_r(z, c) - mean) * invstd
        pre = zh * gam + bet
        gr = _r(g_a, c)
        if mask is not None:
            gr = torch.where(mask[c].reshape(gr.shape), gr, 0.0)
        elif relu:
            gr = torch.where(pre > 0, gr, 0.0)
        return zh, pre, gr

    def sums(c):
        zh, _, g = parts(c)
        return g, g * zh

    m1, m2 = (t / n for t in _cols(z, chunk, sums))
    return dict(n=n, mean=mean, invstd=invstd, gam=gam, parts=parts, m1=m1, m2=m2)


def bn_train_bwd(z, g_a, gamma, beta, relu=False, eps=R.BN_EPS, mask=None, chunk=None):
    """(g_z, dgamma, dbeta, pre) of fp64_ref.bn_train_bwd; z, g_a (and mask) [B, ..., F]."""
    s = _bwd_cols(z, g_a, gamma, beta, relu, eps, mask, chunk)
    n = s["n"]
    g_z = torch.empty(z.shape, dtype=F64, device=z.device)
    pre_out = torch.empty(z.shape, dtype=F64, device=z.device)
    for c in _chunks(z.shape[0], chunk):
        zh, pre, g = s["parts"](c)
        g_z[c] = (s["gam"] * s["invstd"] * (g - s["m1"] - zh * s["m2"])).reshape(g_z[c].shape)
        pre_out[c] = pre.reshape(pre_out[c].shape)
    return g_z, s["m2"] * n, s["m1"] * n, pre_out


def bn_train_bwd_bound(z, g_a, gamma, beta, relu=False, eps=R.BN_EPS, mask=None, chunk=None):
    """fp64_ref.bn_train_bwd_bound: (g_z [z's shape], dgamma [F], dbeta [F])."""
    dv = z.device
    s = _bwd_cols(z, g_a, gamma, beta, relu, eps, mask, chunk)
    n, F = s["n"], z.shape[-1]
    st = _bn_fwd_cols(z, None, gamma, beta, eps, chunk)
    st_is = (1 / st["sig"]) * (st["rel_is"] + st["mzE"] / st["sig"])
    st_mean = st["mE"] + st["d_mean"]
    mean, invstd, gam, m1, m2 = s["mean"], s["invstd"], s["gam"], s["m1"], s["m2"]
    a = gam.abs() * invstd
    e_a = gam.abs() * st_is + R.U32 * a
    al = R.stat_allowance(n, F)

    def e_zh(c, zh):
        return (_r(z, c) - mean).abs() * st_is + invstd * st_mean + 2 * R.U32 * zh.abs()

    def sums(c):
        zh, _, g = s["parts"](c)
        ag = g.abs()
        return ag, ag * zh.abs(), ag * e_zh(c, zh)

    sum_ag, sum_agzh, sum_agezh = _cols(z, chunk, sums)
    dgam, dbet = m2 * n, m1 * n
    e_m1 = al * sum_ag / n + R.U32 * m1.abs()
    e_m2 = al * sum_agzh / n + sum_agezh / n + R.U32 * m2.abs()
    e_gz = torch.empty(z.shape, dtype=F64, device=dv)
    for c in _chunks(z.shape[0], chunk):
        zh, _, g = s["parts"](c)
        ag = g.abs()
        ezh = e_zh(c, zh)
        g_z = gam * invstd * (g - m1 - zh * m2)
        e = (e_a * (g - m1 - zh * m2).abs() + a * (e_m1 + m2.abs() * ezh + zh.abs() * e_m2)
             + R.U32 * (5 * a * (ag + m1.abs() + (zh * m2).abs())
                        + 4 * a * invstd * m2.abs() * (_r(z, c).abs() + mean.abs()) + 2 * g_z.abs()))
        e_gz[c] = e.reshape(e_gz[c].shape)
    e_dbeta = al * sum_ag + R.U32 * dbet.abs()
    e_dgamma = al * sum_agzh + sum_agezh + R.U32 * dgam.abs()
    return e_gz, e_dgamma, e_dbeta


def col_sum_bound(g, chunk=None) -> torch.Tensor:
    """fp64_ref.col_sum_bound over the rows of g [B, ..., F]."""
    n, F = _n_rows(g), g.shape[-1]
    rl = 256 // min(F, 256)
    m = min(n, -(-R.STAT_ROWS // rl))
    sa, ss = _cols(g, chunk, lambda c: (_r(g, c).abs(), _r(g, c)))
    return (m + rl) * R.U32 * sa + R.U32 * ss.abs()


# --------------------------------------------------------------------------------------------- network glue
def unpool(x) -> torch.Tensor:
    return torch.repeat_interleave(t64(x), 2, dim=1)


def unpool_t(g) -> torch.Tensor:
    g = t64(g)
    B, V, F = g.shape
    return g.reshape(B, V // 2, 2, F).sum(dim=2)


def _resample(x, M, chunk):
    out = torch.empty(x.shape[:-1] + (M.shape[0],), dtype=F64, device=x.device)
    for c in _chunks(x.shape[0], chunk):
        out[c] = x[c].to(F64) @ M.T
    return out


def channel_resample(x, fout: int, chunk=None) -> torch.Tensor:
    if x.shape[-1] == fout:
        return t64(x)
    return _resample(x, t64(R.resample_matrix(x.shape[-1], fout), x.device), chunk)


def channel_resample_t(g, fin: int, chunk=None) -> torch.Tensor:
    if g.shape[-1] == fin:
        return t64(g)
    return _resample(g, t64(R.resample_matrix(fin, g.shape[-1]), g.device).T, chunk)


def channel_resample_bound(x, fout: int, chunk=None) -> torch.Tensor:
    fin = x.shape[-1]
    if fin == fout:
        return torch.zeros(x.shape, dtype=F64, device=x.device)
    M, M32 = R.resample_matrix(fin, fout), R.resample_matrix(fin, fout, np.float32)
    return _resample(x.abs(), t64(np.abs(M - M32) + 3 * R.U32 * np.abs(M), x.device), chunk)


def channel_resample_t_bound(g, fin: int, chunk=None) -> torch.Tensor:
    fout = g.shape[-1]
    if fin == fout:
        return torch.zeros(g.shape, dtype=F64, device=g.device)
    M, M32 = R.resample_matrix(fin, fout), R.resample_matrix(fin, fout, np.float32)
    taps = int((M32 != 0).sum(axis=0).max())
    return _resample(g.abs(), t64((np.abs(M - M32) + (taps + 1) * R.U32 * np.abs(M)).T, g.device), chunk)


def thin_head_fused_bound(y_in, E_in, L, W, chunk=None) -> torch.Tensor:
    """fp64_ref.thin_head_fused_bound."""
    E_in = t64(E_in)
    dv = E_in.device
    lp, aW = lap(L, dv), t64(W, dv).abs()
    B, V, _ = E_in.shape
    out = torch.empty(B, V, aW.shape[0], dtype=F64, device=dv)
    for c in _chunks(B, chunk):
        out[c] = (_flat(_abs_basis(E_in[c], lp)) @ aW.T).reshape(-1, V, aW.shape[0])
    return out


def fc(a0, W, b, precision: str):
    """The fc (test_gpu_network_fp64.fc_ref): (float64 a0 W^T + b, its bound); a0 [B, K]."""
    a0 = t64(a0)
    dv = a0.device
    W, b = t64(W, dv), t64(b, dv)
    ref = a0 @ W.T + b
    bound = R.gamma(a0.shape[1], precision) * (a0.abs() @ W.abs().T) + R.U32 * (b.abs() + ref.abs())
    if precision == "fp16x3":
        bound = bound + (2.0 ** -34 * float(a0.abs().max()) * W.abs().sum(dim=1)[None, :]
                         + R.NET_LO / R.NET_W_SCALE * a0.abs().sum(dim=1, keepdim=True))
    return ref, bound


def bound_ratio(y, y64, bound, chunk=None) -> float:
    """fp64_ref.bound_ratio: max |y - y64| / bound over every element (inf where y is not finite)."""
    worst = 0.0
    n = y.shape[0] if y.dim() else 1
    for c in _chunks(n, chunk):
        yc = y[c].to(F64)
        if not bool(torch.isfinite(yc).all()):
            return math.inf
        r = ((yc - y64[c].to(F64)).abs() / bound[c].to(F64).clamp_min(1e-300)).max() if yc.numel() else 0.0
        worst = max(worst, float(r))
    return worst
