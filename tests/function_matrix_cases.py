"""The function matrix: every table distortion function at the parameters and distances where its kernels branch.

Shared by tests/golden/make_function_matrix_golden.py (which runs the reference on these cases and stores
tests/golden/function_matrix.npz) and by the tests that read that fixture.  A case is a function with fixed scalar
parameters (exponent, threshold, alpha, gamma) and, per point, a distance d and the per-edge parameters (weight or
deviation, and the second weight array of WeightedQuadratic).  `build(ns, case, par0, par1)` constructs the case
from the `penalties` / `losses` modules of either the reference or pymde_b200, which share class names and
constructor signatures.

Points (all fp32 numbers; the fp64 columns of the fixture evaluate the same numbers in fp64):
  * d log-spaced over 1e-6 .. 1e4, plus 0.0625 (the MUFU series threshold), 0.25, 0.4 and 0.49 (inside the range a
    wrong series threshold would reach);
  * d = 0;
  * d exactly at every threshold (penalty Huber: d = threshold; Logistic: d = threshold; loss Huber: |d - delta| =
    threshold), d = delta and d = delta (1 +- 2^-20) for every loss;
  * d where d^e (penalties) or |d - delta|^e (loss Power) overflows or underflows fp32, and d = delta + 100, where
    exp(|d - delta|) overflows fp32 (loss Logistic);
  * InvPower and LogRatio: d where d d^e or d^2e leaves the normal fp32 range while d^e does not, and where
    |w| / d^e overflows (`_band_d`).
Penalty weights include 0 and -0.0 (the reference's `weights >= 0` puts both on the attractive side of PushAndPull)
and negative values; deviations are dyadic, so delta +- threshold is exact in fp32.
"""
import functools

import numpy as np

EXPONENTS = (0.5, 1.0, 1.5, 2.0, 3.0, 0.7, 2.5)  # every pow_pair branch, and powf
W_ANY = (0.5, 1.0, 2.0, 0.0, -0.0)
W_REP = (-0.5, -1.0, -2.0, 0.0, -0.0)
W_PP = (1.0, 2.0, -1.0, 0.0, -0.0, -0.5)
DEVS = (0.125, 0.5, 1.0, 3.0, 10.0)
W2 = (0.5, 1.0, 2.0)

_F32_MAX = float(np.finfo(np.float32).max)


def _f32(x):
    return float(np.float32(x))


GRID = tuple(_f32(x) for x in np.concatenate([10.0 ** np.linspace(-6, 4, 41), [0.0625, 0.25, 0.4, 0.49]]))
LOSS_GRID = tuple(_f32(x) for x in np.concatenate([10.0 ** np.linspace(-6, 4, 21), [0.0625, 0.25, 0.4, 0.49]]))


class Case(object):
    """family 'pen' | 'loss' | 'pp'; make(ns, par0, par1) -> distortion function."""

    def __init__(self, name, family, make, weights=None, exponent=None, kinks=(), thresholds=(), par1=False,
                 scalar=False):
        self.name, self.family, self.make = name, family, make
        self.weights = weights
        self.exponent = exponent
        self.kinks = tuple(kinks)            # penalty d values that are branch points
        self.thresholds = tuple(thresholds)  # loss Huber thresholds: d = delta +- threshold
        self.par1 = par1                     # WeightedQuadratic with explicit weights
        self.scalar = scalar                 # one weight for every edge (a 1-element tensor)


def _overflow_d(e):
    """d (fp32) with d^e > fp32 max, and d with d^e < the smallest fp32 subnormal; only exponents > 1 have them."""
    if e is None or e <= 1.0:
        return ()
    big = 2.0 ** (130.0 / e)
    small = 2.0 ** (-152.0 / e)
    return tuple(_f32(x) for x in (big, small) if x < _F32_MAX)


def _band_d(e, weights):
    """InvPower and LogRatio: d where a product of powers of d such as d d^e or d^2e underflows, becomes subnormal or
    overflows in fp32 while d^e itself does not, and d where |w| / d^e overflows (d^e ~ |w| 2^-128).  Forms of f' that
    multiply or divide in another order than the reference's chain rule turn finite there when the reference is not,
    or the other way round."""
    out = [2.0 ** (k / c) for k in (-152.0, -140.0, -130.0, 130.0) for c in (e + 1.0, 2.0 * e)]
    out += [(abs(w) * 2.0 ** -128) ** (1.0 / e) for w in weights if w != 0]
    return tuple(sorted({_f32(x) for x in out if x < _F32_MAX and _f32(x) > 0.0}))


def points(case):
    """(d, par0, par1 or None) as fp32 arrays."""
    d, a, b = [], [], []
    if case.family in ("pen", "pp"):
        W = case.weights
        specials = (0.0,) + tuple(_f32(k) for k in case.kinks) + _overflow_d(case.exponent)
        for k, x in enumerate(GRID):
            d.append(x)
            a.append(W[k % len(W)])
        for x in specials:
            for w in W:
                d.append(x)
                a.append(w)
        if case.scalar:
            a = [W[0]] * len(d)
    else:
        for dev in DEVS:
            specials = [0.0, dev, dev * (1 + 2.0 ** -20), dev * (1 - 2.0 ** -20), dev + 100.0]
            for t in case.thresholds:
                specials += [dev + t] + ([dev - t] if dev - t >= 0 else [])
            for x in _overflow_d(case.exponent):
                specials.append(dev + x)
            for x in LOSS_GRID + tuple(specials):
                d.append(_f32(x))
                a.append(dev)
        if case.par1:
            b = [W2[k % len(W2)] for k in range(len(d))]
    f32 = np.float32
    return (np.array(d, f32), np.array(a, f32), np.array(b, f32) if b else None)


_IMPLIED_EXP = {"Quadratic": 2.0, "Cubic": 3.0}


def _cases():
    out = []

    def pen(name, cls, weights=W_ANY, kinks=(), **kw):
        # kw: constructor keywords; `exponent` also places the overflow points
        def make(ns, par0, par1):
            return getattr(ns.penalties, cls)(par0, **kw)
        out.append(Case(name, "pen", make, weights, kw.get("exponent", _IMPLIED_EXP.get(cls)), kinks))

    pen("pen_linear", "Linear")
    pen("pen_quadratic", "Quadratic")
    pen("pen_cubic", "Cubic")
    for e in EXPONENTS:
        pen("pen_power_%g" % e, "Power", exponent=e)
    for t in (0.25, 0.5, 2.0):
        pen("pen_huber_%g" % t, "Huber", kinks=(t,), threshold=t)
    for t in (-1.0, 0.3, 2.0):
        for al in (0.5, 3.0, 20.0):
            # both libraries refuse a negative threshold in the constructor; the formula takes any value, so the
            # threshold is set afterwards (z = alpha (d + 1) > 0 at every d)
            def make(ns, par0, par1, t=t, al=al):
                f = ns.penalties.Logistic(par0, max(t, 0.0), al)
                f.threshold = t
                return f
            out.append(Case("pen_logistic_%g_%g" % (t, al), "pen", make, W_ANY, None,
                            kinks=((t,) if t >= 0 else ()) + (max(t, 0.0) + 40.0 / al,)))
    for e in EXPONENTS:
        pen("pen_log1p_%g" % e, "Log1p", exponent=e)
        pen("pen_log_%g" % e, "Log", weights=W_REP, exponent=e)
        pen("pen_invpower_%g" % e, "InvPower", weights=W_REP, kinks=_band_d(e, W_REP), exponent=e)
        pen("pen_logratio_%g" % e, "LogRatio", weights=W_REP, kinks=_band_d(e, W_REP), exponent=e)

    def scalar(name, cls, w, **kw):
        def make(ns, par0, par1):
            import torch
            return getattr(ns.penalties, cls)(torch.tensor([float(w)], dtype=par0.dtype, device=par0.device), **kw)
        out.append(Case(name, "pen", make, (w,), kw.get("exponent"), scalar=True))

    scalar("pen_quadratic_scalar_w", "Quadratic", 2.0)
    scalar("pen_log1p_scalar_w", "Log1p", 0.5, exponent=1.5)

    def pp(name, att, rep, ea=None, er=None):
        def make(ns, par0, par1):
            P = ns.penalties
            A = getattr(P, att) if ea is None else functools.partial(getattr(P, att), exponent=ea)
            R = getattr(P, rep) if er is None else functools.partial(getattr(P, rep), exponent=er)
            return P.PushAndPull(par0, A, R)
        out.append(Case(name, "pp", make, W_PP, None))

    pp("pp_log1p_log", "Log1p", "Log")                     # the recipe default: MUFU kernels unless precise
    pp("pp_log1p_logratio", "Log1p", "LogRatio")           # the reference's own default
    pp("pp_quadratic_invpower", "Quadratic", "InvPower")
    pp("pp_log1p2_log2", "Log1p", "Log", 2.0, 2.0)         # Log1p / Log ids with other exponents: no MUFU form
    pp("pp_log1p3_log05", "Log1p", "Log", 3.0, 0.5)
    pp("pp_huber_logratio", "Huber", "LogRatio")           # run-time table on every path

    def loss(name, cls, thresholds=(), par1=False, **kw):
        def make(ns, par0, par1_):
            if par1:
                return getattr(ns.losses, cls)(par0, par1_, **kw)
            return getattr(ns.losses, cls)(par0, **kw)
        out.append(Case(name, "loss", make, None, kw.get("exponent", _IMPLIED_EXP.get(cls)), thresholds=thresholds,
                        par1=par1))

    loss("loss_absolute", "Absolute")
    loss("loss_quadratic", "Quadratic")
    loss("loss_weighted_quadratic", "WeightedQuadratic")
    loss("loss_weighted_quadratic_w", "WeightedQuadratic", par1=True)
    for t in (0.25, 0.5, 2.0):
        loss("loss_huber_%g" % t, "Huber", thresholds=(t,), threshold=t)
    loss("loss_cubic", "Cubic")
    for e in EXPONENTS:
        loss("loss_power_%g" % e, "Power", exponent=e)
    loss("loss_logistic", "Logistic")
    loss("loss_fractional", "Fractional")
    for g in (1.0, 10.0, 100.0):
        loss("loss_soft_fractional_%g" % g, "SoftFractional", gamma=g)
    return out


CASES = _cases()
BY_NAME = {c.name: c for c in CASES}


def build(ns, case, par0, par1=None):
    """The case's distortion function from the `penalties` / `losses` modules of `ns`, on par0's device and dtype."""
    return case.make(ns, par0, par1)
