"""A float64 restatement of one RMSprop step (torch.optim.RMSprop, include/p2m_b200.h p2m_rmsprop_step) and the
element-wise bound of one step computed in a floating-point format of unit roundoff u.

The kernel's operation order, per element (every line one of torch's foreach ops; a + c b is one fma in the kernel and
may be two roundings in torch, so it is counted as two here, which bounds both):

    g   = g + wd p                                   (wd != 0)       2 roundings
    s   = s alpha ;  s = s + (1 - alpha) (g g)                       4
    ga  = ga + (1 - alpha) (g - ga)                  (centred)       3
    v   = s - ga ga                                  (centred)       2
    avg = sqrt(v) + eps                                              2
    q   = g / avg                                                    1
    buf = buf mu + q ;  p = p + (-lr) buf            (momentum)      4
    p   = p + (-lr) q                                (otherwise)     2

Each quantity x is carried as (x, e): its value in exact arithmetic and a bound on |computed - exact|.  A rounding of a
result whose exact value is x and whose unrounded computed value is within e of it adds at most u (|x| + e) + eta (eta
the format's smallest subnormal, for results in the subnormal range); an operation on inexact operands propagates
their bounds exactly to first order and with the product term:

    a + b    e_a + e_b
    a b      |a| e_b + |b| e_a + e_a e_b             (c a for a constant c of the format: |c| e_a)
    a / b    (e_a + |a / b| e_b) / (|b| - e_b)
    sqrt(a)  min(sqrt(e_a), e_a / (sqrt(a) + sqrt(max(a - e_a, 0))))

so an error in s reaches avg at half its relative size, and p's bound is u |p| from the last rounding plus
lr |g| / avg times the relative bound of q (the roundings of g, s, the square root, eps, the division and the
multiplication by lr).  With zero input bounds this is the bound of one step from exact inputs; with the bounds of the
previous step as input bounds it accumulates along a trajectory (the two fp32 implementations then differ by at most
twice the accumulated bound).  The hyperparameters are exact constants of the format: the fp32-rounded values for the
kernel (fp32_hparams), the Python floats for a float64 step.
"""
from __future__ import annotations

import torch

U32, ETA32 = 2.0 ** -24, 2.0 ** -149
U64, ETA64 = 2.0 ** -53, 2.0 ** -1074
OPTION_GRID = [dict(weight_decay=wd, momentum=mu, centered=c) for wd in (0.0, 0.1) for mu in (0.0, 0.9)
               for c in (False, True)]


def fp32_hparams(lr, alpha=0.99, eps=1e-8, weight_decay=0.0, momentum=0.0, centered=False):
    """The constants the kernel multiplies by: each hyperparameter rounded to fp32, 1 - alpha computed in double first
    (torch passes value=1 - alpha from Python)."""
    f = lambda x: float(torch.tensor(float(x), dtype=torch.float32))
    return dict(lr=f(lr), alpha=f(alpha), one_minus_alpha=f(1.0 - alpha), eps=f(eps), weight_decay=f(weight_decay),
                momentum=f(momentum), centered=centered, use_momentum=momentum > 0, use_wd=weight_decay != 0)


def f64_hparams(lr, alpha=0.99, eps=1e-8, weight_decay=0.0, momentum=0.0, centered=False):
    """The same as float64 constants (torch.optim.RMSprop in float64)."""
    return dict(lr=float(lr), alpha=float(alpha), one_minus_alpha=1.0 - alpha, eps=float(eps),
                weight_decay=float(weight_decay), momentum=float(momentum), centered=centered,
                use_momentum=momentum > 0, use_wd=weight_decay != 0)


class _E:
    """A value in exact arithmetic (float64 tensor) with the bound of its computed counterpart."""

    def __init__(self, v, e, u, eta):
        self.v, self.e, self.u, self.eta = v, e, u, eta

    def _new(self, v, e, rounded=True):
        return _E(v, e + (self.u * (v.abs() + e) + self.eta if rounded else 0.0), self.u, self.eta)

    def __add__(self, o):
        return self._new(self.v + o.v, self.e + o.e)

    def __sub__(self, o):
        return self._new(self.v - o.v, self.e + o.e)

    def __mul__(self, o):
        if isinstance(o, float):
            return self._new(self.v * o, abs(o) * self.e)
        return self._new(self.v * o.v, self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e)

    def __truediv__(self, o):
        q = self.v / o.v
        return self._new(q, (self.e + q.abs() * o.e) / (o.v.abs() - o.e))

    def sqrt(self):
        v = self.v.clamp_min(0).sqrt()
        below = (self.v - self.e).clamp_min(0).sqrt()
        e = torch.minimum(self.e.sqrt(), self.e / (v + below).clamp_min(1e-300))
        return self._new(v, e)

    def plus_const(self, c):
        return self._new(self.v + c, self.e)


def step(p, g, s, buf=None, ga=None, *, hp, u=U32, eta=ETA32, err=None):
    """One step of float64 tensors (p, g, s and, where the options use them, buf / ga: the state before the step) with
    hyperparameters hp (fp32_hparams / f64_hparams).  err: input bounds {"p", "s", "buf", "ga"} (absent: 0; g is
    exact).  Returns (values, bounds): dicts with keys p, s and buf / ga where used, after the step."""
    err = err or {}
    z = torch.zeros_like(p)
    E = lambda x, k: _E(x, err.get(k, z), u, eta)
    P, S, G = E(p, "p"), E(s, "s"), _E(g, z, u, eta)
    if hp["use_wd"]:
        G = G + P * hp["weight_decay"]
    S = S * hp["alpha"]
    S = S + (G * G) * hp["one_minus_alpha"]
    out = {}
    V = S
    if hp["centered"]:
        A = E(ga, "ga")
        A = A + (G - A) * hp["one_minus_alpha"]
        V = S - A * A
        out["ga"] = A
    avg = V.sqrt().plus_const(hp["eps"])
    Q = G / avg
    if hp["use_momentum"]:
        B = E(buf, "buf") * hp["momentum"] + Q
        P = P + B * (-hp["lr"])
        out["buf"] = B
    else:
        P = P + Q * (-hp["lr"])
    out["p"], out["s"] = P, S
    return {k: x.v for k, x in out.items()}, {k: x.e for k, x in out.items()}


def exceed(got, ref, bound, slack=1.0 + 2.0 ** -20):
    """Elements where |got - ref| > slack * bound (slack covers the float64 rounding of ref and bound); both float64."""
    return ((got.double() - ref).abs() > bound * slack).sum().item()
