"""Float64 reference of PoseNet's train-mode forward and backward with the dropout masks injected, the element-wise
bound an implementation built from the library's kernels is held to (same precision model as fp64_ref), and the dropout
rule of include/p2m_b200.h restated in numpy (Philox4x32-10 and the keep test).

The bound is first order and carried through the whole chain.  Within one operation it is fp64_ref's; from one
operation to the next the errors of different elements are taken as independent with mean zero, like the rounding
errors inside fp64_ref.gamma: a sum of them grows as the root of the sum of squares.  What is carried along is thus an
error scale per element, and the bound is C_FINAL times the scale at the end, applied once.  (Worst-case absolute-value
propagation multiplies by ||W||_1 ~ sqrt(H) per layer, and a safety factor inside every sum compounds to the eighth
power: either says nothing after eight layers.)"""
from __future__ import annotations

import numpy as np

import fp64_ref as R

U32 = R.U32
C_RSS = 1.0               # a sum of independent propagated errors: sqrt(sum of squares)
C_FINAL = 6.0             # bound = C_FINAL * the propagated error scale


def _rss(E, W):
    """Bound on sum_k e_ik W_kj for independent errors |e_ik| <= E_ik."""
    return C_RSS * np.sqrt((E * E) @ (W * W))


# --------------------------------------------------------------------------------------------- the dropout rule
def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11).  ctr: four uint32 arrays (or ints), key: two.  Returns four uint32 arrays."""
    c = [np.asarray(v, np.uint64) & np.uint64(0xFFFFFFFF) for v in ctr]
    k = [int(v) & 0xFFFFFFFF for v in key]
    m0, m1, mask = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k[0]), p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k[1]),
             p0 & mask]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return [v.astype(np.uint32) for v in c]


def dropout_multiplier(seed, layer: int, n: int, p: float) -> np.ndarray:
    """The multiplier (0, or float32 1 / (1 - p)) of each of the n elements of dropout layer `layer`, as float64."""
    p = np.float32(p)
    if p <= 0:
        return np.ones(n)
    if p >= 1:
        return np.zeros(n)
    s0, s1 = (int(v) & 0xFFFFFFFFFFFFFFFF for v in seed)
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    words = philox4x32_10((q & np.uint64(0xFFFFFFFF), q >> np.uint64(32), layer, s1 & 0xFFFFFFFF),
                          (s0 & 0xFFFFFFFF, s0 >> 32))
    bits = np.stack(words, axis=1).reshape(-1)[:n]
    threshold = min(int(np.floor((1.0 - float(p)) * 2.0 ** 32)), 2 ** 32 - 1)
    keep_scale = np.float32(1) / (np.float32(1) - p)
    return np.where(bits < threshold, float(keep_scale), 0.0)


def dropout_masks(seed, p: float, B: int, H: int, num_stage: int):
    """[2 num_stage] multipliers [B, H]: layer d = 2 stage + {0 after bn1, 1 after bn2}."""
    return [dropout_multiplier(seed, d, B * H, p).reshape(B, H) for d in range(2 * num_stage)]


# --------------------------------------------------------------------------------------------- forward + backward
def _gemm(a, ea, Wt, eW, prec, over_batch=False):
    """a [m, k] @ Wt [k, n] and its bound when a is within ea and Wt within eW of the exact operands.  over_batch: the
    sum runs over the batch, where the errors of one channel share that channel's statistics (mean, invstd) and are
    not independent: they add linearly."""
    y = a @ Wt
    prop = ea @ np.abs(Wt) + np.abs(a) @ eW if over_batch else _rss(ea, Wt) + _rss(a, eW)
    e = R.gamma(a.shape[1], prec) * (np.abs(a) @ np.abs(Wt)) + prop
    if prec == "fp16x3":
        e = e + R.floor_matmul(a, Wt)
    return y, e


def _col_sum(g, eg):
    """Sum over the batch: see _gemm's over_batch."""
    return g.sum(axis=0), eg.sum(axis=0) + R.stat_allowance(*g.shape) * np.abs(g).sum(axis=0) + U32 * np.abs(g.sum(axis=0))


def _bn_fwd(z, ez, f, pre, mult):
    """drop(relu(bn(z))) with batch statistics: the activation, its bound, and what the backward needs."""
    g, b, rm, rv = (f[pre + k] for k in ("weight", "bias", "running_mean", "running_var"))
    h, mean, var, rm_new, rv_new = R.bn_train_fwd(z, g, b, rm, rv)
    bd = R.bn_train_fwd_bound(z, np.zeros_like(z), g, b, rm, rv)      # the layer's own roundings
    n = z.shape[0]
    sig = np.sqrt(var + R.BN_EPS)
    zh = np.abs(z - mean) / sig
    # the incoming error e moves y by gamma / sigma (e - mean(e) - zhat mean(zhat e)): the two means are sums
    m_e, m_ze = C_RSS * np.sqrt((ez * ez).sum(axis=0)) / n, C_RSS * np.sqrt((zh * ez * zh * ez).sum(axis=0)) / n
    eh = bd["y"] + np.abs(g) / sig * (ez + m_e + zh * m_ze)
    unb = n / (n - 1)
    a = np.maximum(h, 0.0) * mult
    ea = eh * mult + U32 * np.abs(a)
    ctx = dict(z=z, ez=ez + U32 * np.abs(z), h=h, eh=eh, mean=mean, sig=sig, gamma=g, mult=mult,
               e_mean=bd["mean"] + m_e, e_is=bd["invstd"] + m_ze / sig ** 2)
    stats = dict(rm=rm_new, rv=rv_new, e_rm=bd["rm"] + R.BN_MOMENTUM * m_e,
                 e_rv=bd["rv"] + R.BN_MOMENTUM * unb * 2 * sig * m_ze)
    return a, ea, ctx, stats


def _bn_bwd(c, ga, ega):
    """Gradient through drop, ReLU and the train-mode BatchNorm of context c: (g_z, bound, dgamma, bound, dbeta, bound).
    An activation whose pre-ReLU value is within its own forward bound of zero may have the other sign in fp32: its
    gradient is allowed to be there or not."""
    z, mean, sig, gam, mult = c["z"], c["mean"], c["sig"], c["gamma"], c["mult"]
    n = z.shape[0]
    on, flip = c["h"] > 0, np.abs(c["h"]) <= c["eh"]
    gp = ga * mult * on
    egp = ega * mult * (on | flip) + np.abs(ga) * mult * flip + U32 * np.abs(gp)
    zh = (z - mean) / sig
    ezh = (c["ez"] + c["e_mean"]) / sig + np.abs(z - mean) * c["e_is"] + 2 * U32 * np.abs(zh)
    dbeta, e_dbeta = _col_sum(gp, egp)
    dgamma, e_dgamma = _col_sum(gp * zh, egp * np.abs(zh) + np.abs(gp) * ezh + U32 * np.abs(gp * zh))
    m1, m2, em1, em2 = dbeta / n, dgamma / n, e_dbeta / n, e_dgamma / n
    sc = gam / sig
    gz = sc * (gp - m1 - zh * m2)
    asc = np.abs(sc)
    egz = (asc * (egp + em1 + np.abs(zh) * em2 + ezh * np.abs(m2)) + np.abs(gz) * (c["e_is"] * sig + 4 * U32)
           + 8 * U32 * asc * (np.abs(gp) + np.abs(m1) + np.abs(zh * m2))
           + 4 * U32 * asc / sig * np.abs(m2) * (np.abs(z) + np.abs(mean)))       # g_z = a g' + b z + c: b z against c
    return gz, egz, dgamma, e_dgamma, dbeta, e_dbeta


def forward_backward(sd, x, num_stage: int, masks, d_out, precision: str = "fp16x3", last_precision: str = "fp32"):
    """sd: state_dict name -> array (running statistics BEFORE the step).  masks: dropout_masks(...) (or any list of
    [B, H] multipliers).  Returns (values, bounds): dicts with 'out', 'dx', 'grad.<parameter name>',
    '<bn>.running_mean', '<bn>.running_var'."""
    f = {k: np.asarray(v, np.float64) for k, v in sd.items()}
    x, d_out = np.asarray(x, np.float64), np.asarray(d_out, np.float64)
    val, bnd = {}, {}
    zero = np.zeros_like
    y, e = _gemm(x, zero(x), f["w1.weight"].T, zero(f["w1.weight"].T), "fp32")
    y = y + f["w1.bias"]
    e = e + U32 * np.abs(y)
    tape = []
    for s in range(num_stage):
        p = f"linear_stages.{s}."
        Wa, Wb = f[p + "w1.weight"], f[p + "w2.weight"]
        a1, ea1, c1, st1 = _bn_fwd(y, e, f, p + "batch_norm1.", masks[2 * s])
        z, ez = _gemm(a1, ea1, Wa.T, zero(Wa.T), precision)
        z = z + f[p + "w1.bias"]
        ez = ez + U32 * np.abs(z)
        a2, ea2, c2, st2 = _bn_fwd(z, ez, f, p + "batch_norm2.", masks[2 * s + 1])
        o, eo = _gemm(a2, ea2, Wb.T, zero(Wb.T), precision)
        y = y + o + f[p + "w2.bias"]
        e = e + eo + 2 * U32 * (np.abs(y) + np.abs(o))
        tape.append((a1, ea1, c1, a2, ea2, c2))
        for name, st in (("batch_norm1.", st1), ("batch_norm2.", st2)):
            val[p + name + "running_mean"], bnd[p + name + "running_mean"] = st["rm"], st["e_rm"]
            val[p + name + "running_var"], bnd[p + name + "running_var"] = st["rv"], st["e_rv"]
    W2 = f["w2.weight"]
    out, eout = _gemm(y, e, W2.T, zero(W2.T), last_precision)
    val["out"], bnd["out"] = out + f["w2.bias"], eout + U32 * np.abs(out + f["w2.bias"])

    # backward; the thin layers run in fp32, both operands of a tensor-core dW enter the fp16 split range-normalised
    def put(name, v, b):
        val["grad." + name], bnd["grad." + name] = v, b

    put("w2.bias", *_col_sum(d_out, zero(d_out)))
    put("w2.weight", *_gemm(d_out.T, zero(d_out.T), y, e, "fp32", over_batch=True))
    g, eg = _gemm(d_out, zero(d_out), W2, zero(W2), "fp32")
    for s in reversed(range(num_stage)):
        p = f"linear_stages.{s}."
        a1, ea1, c1, a2, ea2, c2 = tape[s]
        put(p + "w2.bias", *_col_sum(g, eg))
        put(p + "w2.weight", *_gemm(g.T, eg.T, a2, ea2, precision, over_batch=True))
        ga2, ega2 = _gemm(g, eg, f[p + "w2.weight"], zero(f[p + "w2.weight"]), precision)
        gz, egz, dgam, e_dgam, dbet, e_dbet = _bn_bwd(c2, ga2, ega2)
        put(p + "batch_norm2.weight", dgam, e_dgam)
        put(p + "batch_norm2.bias", dbet, e_dbet)
        put(p + "w1.bias", *_col_sum(gz, egz))
        put(p + "w1.weight", *_gemm(gz.T, egz.T, a1, ea1, precision, over_batch=True))
        ga1, ega1 = _gemm(gz, egz, f[p + "w1.weight"], zero(f[p + "w1.weight"]), precision)
        gy, egy, dgam, e_dgam, dbet, e_dbet = _bn_bwd(c1, ga1, ega1)
        put(p + "batch_norm1.weight", dgam, e_dgam)
        put(p + "batch_norm1.bias", dbet, e_dbet)
        g = g + gy
        eg = eg + egy + U32 * np.abs(g)
    put("w1.bias", *_col_sum(g, eg))
    put("w1.weight", *_gemm(g.T, eg.T, x, zero(x), "fp32", over_batch=True))
    val["dx"], bnd["dx"] = _gemm(g, eg, f["w1.weight"], zero(f["w1.weight"]), "fp32")
    return val, {k: C_FINAL * v for k, v in bnd.items()}
