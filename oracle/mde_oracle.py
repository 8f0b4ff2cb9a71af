"""TEST INFRASTRUCTURE ONLY -- CPU restatement (numpy) of the reference's MDE hot path.

This file restates, in closed form, the algorithm of cvxgrp/pymde v0.2.1 for the
edge-parallel average-distortion path and the solver wrapped around it.  It is the
checker for the CUDA path in `pymde_b200/`; only `tests/`, `__graft_entry__.smoke()`
and `bench.py`'s cpu_baseline / `--impl reference` leg may import it.  The product
never routes through it.

Parity is PINNED: `tests/golden/make_golden.py` imports the unmodified reference in
the build container and stores its outputs (values, gradients, projections, full
L-BFGS trajectories) as fixtures under `tests/golden/`; `tests/test_oracle_*.py`
check this restatement against every one of them, and against the reference's own
known-answer tests (pymde/test_optim.py:75-93, :97-118, :57-71; pymde/test_util.py:20-71).

Reference map (all paths relative to the reference repo):
  distortion functions  pymde/functions/penalties.py:112-400, pymde/functions/losses.py:61-239
  average distortion    pymde/average_distortion.py:36-80
  constraints           pymde/constraints.py:94-200, pymde/util.py:129-171
  L-BFGS step           pymde/lbfgs.py:390-590      strong Wolfe  pymde/lbfgs.py:16-253
  solve driver          pymde/optim.py:69-184

The reference has no closed-form derivatives (it back-propagates through torch ops);
the derivatives below are those closed forms, including the reference's conventions
at the non-smooth points (sign(0) = 0, tie of max() -> averaged gradient).
"""
import math

import numpy as np

# --------------------------------------------------------------------------------------
# function ids: shared vocabulary with include/mde_b200.h (MDE_FN_*)
# --------------------------------------------------------------------------------------
P_LINEAR, P_QUADRATIC, P_CUBIC, P_POWER, P_HUBER = 1, 2, 3, 4, 5
P_LOGISTIC, P_LOG1P, P_LOG, P_INVPOWER, P_LOGRATIO = 6, 7, 8, 9, 10
L_ABSOLUTE, L_QUADRATIC, L_WEIGHTED_QUADRATIC, L_HUBER, L_CUBIC = 20, 21, 22, 23, 24
L_POWER, L_LOGISTIC, L_FRACTIONAL, L_SOFT_FRACTIONAL = 25, 26, 27, 28


class FnSpec(object):
    """A distortion function in table form.

    fn_att / fn_rep : function ids; for everything except PushAndPull they are equal.
    par0            : (p,) weights (penalties) or deviations (losses)
    par1            : (p,) second per-edge array (WeightedQuadratic weights) or None
    att, rep        : scalar triples (exponent | threshold | gamma, alpha, unused)
    Selection rule for PushAndPull (penalties.py:390): weight >= 0 -> attractive.
    """

    def __init__(self, fn_att, par0, att=(0.0, 0.0, 0.0), fn_rep=None, rep=None, par1=None):
        self.fn_att = int(fn_att)
        self.fn_rep = int(fn_att if fn_rep is None else fn_rep)
        self.par0 = np.asarray(par0)
        self.par1 = None if par1 is None else np.asarray(par1)
        self.att = tuple(float(a) for a in att)
        self.rep = self.att if rep is None else tuple(float(a) for a in rep)
        self.push_pull = fn_rep is not None


def _sign(x):
    return np.sign(x)


def _eval_one(fn, sc, d, a, b, dt):
    """Return (f(d), f'(d)) for one function id. `a` = par0, `b` = par1. Follows the
    formulas of penalties.py / losses.py; derivative = what torch autograd yields."""
    s0 = dt(sc[0])
    s1 = dt(sc[1])
    one = dt(1.0)
    with np.errstate(all="ignore"):
        if fn == P_LINEAR:  # penalties.py:112-120
            return a * d, a * np.ones_like(d)
        if fn == P_QUADRATIC:  # :123-131  w * d^2: a zero weight times an overflowed d^2 is NaN
            return a * (d * d), dt(2.0) * a * d
        if fn == P_CUBIC:  # :163-171
            return a * (d * d * d), dt(3.0) * a * d * d
        if fn == P_POWER:  # :191-202
            return a * np.power(d, s0), a * s0 * np.power(d, s0 - one)
        if fn == P_HUBER:  # :205-243  (s0 = threshold)
            lt = d < s0
            f = np.where(lt, a * dt(0.5) * d * d, a * s0 * (d - dt(0.5) * s0))
            fp = np.where(lt, a * d, a * s0 * np.ones_like(d))
            return f, fp
        if fn == P_LOGISTIC:  # :246-266  (s0 = threshold, s1 = alpha)
            z = s1 * (d - s0)
            f = a * np.logaddexp(dt(0.0), z)
            fp = a * s1 / (one + np.exp(-z))
            return f, fp
        if fn == P_LOG1P:  # :310-321  (s0 = exponent)
            de = np.power(d, s0)
            return a * np.log1p(de), a * s0 * np.power(d, s0 - one) / (one + de)
        if fn == P_LOG:  # :324-337
            de = np.power(d, s0)
            f = a * np.log(-np.expm1(-de))
            fp = a * s0 * np.power(d, s0 - one) / np.expm1(de)
            return f, fp
        if fn == P_INVPOWER:  # :340-353
            aw = np.abs(a)
            de = np.power(d, s0)
            fp = -aw * s0 * np.power(d, -s0 - one)
            # the reference's chain rule -((|w| / x) / x) (e d^(e-1)), x = d^e, is not finite where an intermediate
            # overflows or meets inf * 0 (NaN at d = 0 for e > 1); where it is finite and the closed form is not (a zero
            # weight times d^(-e-1) = inf), its value is the reference's
            chain = -((aw / de) / de) * (s0 * np.power(d, s0 - one))
            return aw / de, np.where(np.isfinite(chain) & np.isfinite(fp), fp, chain)
        if fn == P_LOGRATIO:  # :356-369
            de = np.power(d, s0)
            y = de / (one + de)
            fp = a * s0 / (d * (one + de))
            # the reference's chain rule ((w / y) / (1 + x) - (w / y) x / (1 + x)^2) (e d^(e-1)), x = d^e, is NaN
            # where x is 0 (inf * 0) or overflows (y = inf / inf)
            gy = a / y
            chain = (gy / (one + de) - gy * de / ((one + de) * (one + de))) * (s0 * np.power(d, s0 - one))
            return a * np.log(y), np.where(np.isfinite(chain) & np.isfinite(fp), fp, chain)
        # losses: a = deviations
        r = np.abs(a - d)
        sg = _sign(d - a)
        if fn == L_ABSOLUTE:  # losses.py:166-174
            return r, sg
        if fn == L_QUADRATIC:  # :61-69
            return r * r, dt(2.0) * (d - a)
        if fn == L_WEIGHTED_QUADRATIC:  # :72-87
            return b * r * r, dt(2.0) * b * (d - a)
        if fn == L_HUBER:  # :101-125 (s0 = threshold)
            lt = r < s0
            f = np.where(lt, r * r, s0 * (dt(2.0) * r - s0))
            fp = np.where(lt, dt(2.0) * (d - a), dt(2.0) * s0 * sg)
            return f, fp
        if fn == L_CUBIC:  # :128-136
            return r * r * r, dt(3.0) * r * r * sg
        if fn == L_POWER:  # :139-148
            return np.power(r, s0), s0 * np.power(r, s0 - one) * sg
        if fn == L_LOGISTIC:  # :177-186  (naive log(1+exp(r)), as written in the reference)
            er = np.exp(r)
            return np.log(one + er), er / (one + er) * sg
        if fn == L_FRACTIONAL:  # :189-200
            u = a / d
            v = d / a
            f = np.maximum(u, v) - one
            du = -a / (d * d)
            dv = one / a
            fp = np.where(v > u, dv, np.where(u > v, du, dt(0.5) * (du + dv)))
            return f, fp
        if fn == L_SOFT_FRACTIONAL:  # :203-229 (s0 = gamma)
            u = s0 * a / d
            v = s0 * d / a
            mx = np.maximum(u, v)
            lse = mx + np.log(np.exp(u - mx) + np.exp(v - mx))
            lse = np.where(np.isinf(mx), mx, lse)  # torch.logsumexp returns +inf, not NaN
            # the reference forms 1/gamma and log(2) as fp32 tensors whatever the input dtype
            inv_gamma = dt(np.float32(1.0) / np.float32(sc[0]))
            shift = dt(np.float32(np.log(np.float32(2.0))) + np.float32(sc[0]))  # fp32 sum
            f = inv_gamma * (lse - shift)
            pu = np.exp(u - lse)
            pv = np.exp(v - lse)
            fp = (inv_gamma * s0) * (pu * (-a / (d * d)) + pv * (one / a))
            return f, fp
    raise ValueError("unknown function id %r" % (fn,))


def eval_function(spec, d, dtype=np.float64):
    """(f_k(d_k), f'_k(d_k)) for every edge k."""
    dt = np.dtype(dtype).type
    d = np.asarray(d, dtype=dtype)
    a = np.asarray(spec.par0, dtype=dtype)
    if a.ndim == 0 or a.size == 1:
        a = np.broadcast_to(a.reshape(()), d.shape)
    b = None if spec.par1 is None else np.asarray(spec.par1, dtype=dtype)
    if not spec.push_pull:
        return _eval_one(spec.fn_att, spec.att, d, a, b, dt)
    pos = a >= 0  # penalties.py:390
    f = np.empty_like(d)
    fp = np.empty_like(d)
    fa, fpa = _eval_one(spec.fn_att, spec.att, d[pos], a[pos], None, dt)
    fr, fpr = _eval_one(spec.fn_rep, spec.rep, d[~pos], a[~pos], None, dt)
    f[pos], fp[pos] = fa, fpa
    f[~pos], fp[~pos] = fr, fpr
    return f, fp


# --------------------------------------------------------------------------------------
# average distortion: value and gradient  (average_distortion.py:36-80)
# --------------------------------------------------------------------------------------
def edge_distances(X, edges):
    diff = X[edges[:, 0]] - X[edges[:, 1]]  # :42
    return np.sqrt((diff * diff).sum(axis=1)), diff  # :46


def average_distortion(X, edges, spec, want_grad=True, dtype=np.float64, p_total=None):
    """E = (1/p) sum_k f_k(||x_i - x_j||) and dE/dX.

    g_k = f'_k(d_k) / (p d_k), non-finite g_k -> 1.0 (average_distortion.py:55-62);
    grad = scatter_add(lhs, g*diff) - scatter_add(rhs, g*diff) (:70-79).
    `p_total` overrides the divisor (edge shards of a larger problem)."""
    dt = np.dtype(dtype).type
    X = np.asarray(X, dtype=dtype)
    edges = np.asarray(edges)
    p = edges.shape[0] if p_total is None else p_total
    d, diff = edge_distances(X, edges)
    f, fp = eval_function(spec, d, dtype)
    value = f.sum(dtype=np.float64) / p
    if not want_grad:
        return dtype(value) if dtype is not np.float64 else value, None
    with np.errstate(all="ignore"):
        g = (fp * (dt(1.0) / dt(p))) / d
    g[~np.isfinite(g)] = dt(1.0)
    datx = g[:, None] * diff
    n, m = X.shape
    grad = np.zeros((n, m), dtype=np.float64)
    for c in range(m):
        grad[:, c] = np.bincount(edges[:, 0], weights=datx[:, c], minlength=n) - np.bincount(
            edges[:, 1], weights=datx[:, c], minlength=n
        )
    return value, grad.astype(dtype)


# --------------------------------------------------------------------------------------
# constraints (constraints.py:94-200, util.py:129-171)
# --------------------------------------------------------------------------------------
class Centered(object):
    name = "centered"

    def project(self, Z):  # constraints.py:106-111
        return Z - Z.mean(axis=0, dtype=np.float64).astype(Z.dtype)

    def tangent(self, X, Z):  # :102-104  identity
        return Z


class Standardized(object):
    name = "standardized"

    def project(self, Z):  # :194-195 -> util.py:129-171: de-mean, thin SVD, sqrt(n) U V^T
        Z = Z - Z.mean(axis=0, dtype=np.float64).astype(Z.dtype)
        U, _, Vh = np.linalg.svd(Z.astype(np.float64), full_matrices=False)
        return (math.sqrt(Z.shape[0]) * (U @ Vh)).astype(Z.dtype)

    def tangent(self, X, Z):  # :186-192   Z - (1/n) X (Z^T X)
        n = X.shape[0]
        gtx = Z.astype(np.float64).T @ X.astype(np.float64)
        return (Z - (1.0 / n) * (X.astype(np.float64) @ gtx)).astype(Z.dtype)


class Anchored(object):
    name = "anchored"

    def __init__(self, anchors, values):  # constraints.py:114-164
        self.anchors = np.asarray(anchors)
        self.values = np.asarray(values)

    def project(self, Z):
        Z = Z.copy()
        Z[self.anchors] = self.values.astype(Z.dtype)
        return Z

    def tangent(self, X, Z):
        Z = Z.copy()
        Z[self.anchors] = 0
        return Z


# --------------------------------------------------------------------------------------
# strong-Wolfe line search (lbfgs.py:16-253) on scalars only.
#
# With max_iter=1 per LBFGS.step (optim.py:108-122) the gradient returned by the line
# search is discarded (lbfgs.py:547-549 assigns it, nothing reads it before the next
# step re-reads X.grad at :434), so the bracket needs only (t, f, g.d) triples.
# Scalars follow the reference's types: f and t are Python floats (doubles) until an
# interpolation returns a 0-dim fp32 tensor; directional derivatives are fp32 tensors.
# `sdt` is the dtype used for those tensor-typed scalars (np.float32 mirrors the
# reference; np.float64 is the exact arbiter).
# --------------------------------------------------------------------------------------
def _cubic_interpolate(x1, f1, g1, x2, f2, g2, bounds, sdt):  # lbfgs.py:16-41
    if bounds is not None:
        xmin_bound, xmax_bound = bounds
    else:
        xmin_bound, xmax_bound = (x1, x2) if x1 <= x2 else (x2, x1)
    with np.errstate(all="ignore"):
        d1 = sdt(g1) + sdt(g2) - sdt(3 * (f1 - f2) / (x1 - x2))
        d2_square = sdt(d1 * d1 - sdt(g1) * sdt(g2))
        if d2_square >= 0:
            d2 = sdt(np.sqrt(d2_square))
            if x1 <= x2:
                min_pos = sdt(x2) - sdt(x2 - x1) * sdt((g2 + d2 - d1) / (g2 - g1 + 2 * d2))
            else:
                min_pos = sdt(x1) - sdt(x1 - x2) * sdt((g1 + d2 - d1) / (g1 - g2 + 2 * d2))
            # python min(max(a, b), c) semantics incl. NaN behaviour (:39)
            lo = min_pos if not (xmin_bound > min_pos) else xmin_bound
            return lo if not (xmax_bound < lo) else xmax_bound
        return (xmin_bound + xmax_bound) / 2.0


class SolverError(Exception):
    pass


def strong_wolfe(obj_func, t, f, gtd, d_norm, c1=1e-4, c2=0.9, tolerance_change=1e-9,
                 max_ls=25, sdt=np.float32):
    """obj_func(t) -> (f_new: float, gtd_new, grad_is_finite: bool).  Returns
    (f_new, t, ls_func_evals).  Mirrors lbfgs.py:44-253 decision for decision."""
    f_new = gtd_new = None
    for _ in range(10):  # :59-69  back off while the trial point is outside the domain
        f_new, gtd_new, finite = obj_func(t)
        if np.isnan(f_new) or np.isinf(f_new) or not finite:
            t = t * 0.5
        else:
            break
    if np.isnan(f_new):
        raise SolverError("Function evaluation returned NaN.")
    if np.isinf(f_new):
        raise SolverError("Function evaluation returned inf.")
    if not finite:
        raise SolverError("Gradient evaluation returned NaN/inf.")
    ls_func_evals = 1

    t_prev, f_prev, gtd_prev = 0, f, gtd
    done = False
    ls_iter = 0
    bracket = bracket_f = bracket_gtd = None
    while ls_iter < max_ls:  # :87-133 bracketing
        if f_new > sdt(f + sdt(sdt(c1 * t) * gtd)) or (ls_iter > 1 and f_new >= f_prev):
            bracket, bracket_f, bracket_gtd = [t_prev, t], [f_prev, f_new], [gtd_prev, gtd_new]
            break
        if abs(gtd_new) <= -c2 * gtd:
            bracket, bracket_f, bracket_gtd = [t], [f_new], [gtd_new]
            done = True
            break
        if gtd_new >= 0:
            bracket, bracket_f, bracket_gtd = [t_prev, t], [f_prev, f_new], [gtd_prev, gtd_new]
            break
        min_step = t + 0.01 * (t - t_prev)
        max_step = t * 10
        tmp = t
        t = _cubic_interpolate(t_prev, f_prev, gtd_prev, t, f_new, gtd_new,
                               (min_step, max_step), sdt)
        t_prev, f_prev, gtd_prev = tmp, f_new, gtd_new
        f_new, gtd_new, _ = obj_func(t)
        ls_func_evals += 1
        ls_iter += 1

    if ls_iter == max_ls:  # :136-139
        bracket, bracket_f, bracket_gtd = [0, t], [f, f_new], [gtd, gtd_new]

    insuf_progress = False
    low_pos, high_pos = (0, 1) if bracket_f[0] <= bracket_f[-1] else (1, 0)
    while not done and ls_iter < max_ls:  # :147-224 zoom
        if abs(bracket[1] - bracket[0]) * d_norm < tolerance_change:
            break
        t = _cubic_interpolate(bracket[0], bracket_f[0], bracket_gtd[0],
                               bracket[1], bracket_f[1], bracket_gtd[1], None, sdt)
        bmax, bmin = max(bracket), min(bracket)
        eps = 0.1 * (bmax - bmin)
        if min(bmax - t, t - bmin) < eps:
            if insuf_progress or t >= bmax or t <= bmin:
                if abs(t - bmax) < abs(t - bmin):
                    t = bmax - eps
                else:
                    t = bmin + eps
                insuf_progress = False
            else:
                insuf_progress = True
        else:
            insuf_progress = False

        f_new, gtd_new, _ = obj_func(t)
        ls_func_evals += 1
        ls_iter += 1

        if np.isnan(f_new) or (f_new > sdt(f + sdt(sdt(c1 * t) * gtd))
                               or f_new >= bracket_f[low_pos]):
            bracket[high_pos], bracket_f[high_pos], bracket_gtd[high_pos] = t, f_new, gtd_new
            low_pos, high_pos = (0, 1) if bracket_f[0] <= bracket_f[1] else (1, 0)
        else:
            if abs(gtd_new) <= -c2 * gtd:
                done = True
            elif gtd_new * (bracket[high_pos] - bracket[low_pos]) >= 0:
                bracket[high_pos] = bracket[low_pos]
                bracket_f[high_pos] = bracket_f[low_pos]
                bracket_gtd[high_pos] = bracket_gtd[low_pos]
            bracket[low_pos], bracket_f[low_pos], bracket_gtd[low_pos] = t, f_new, gtd_new

    line_search_failed = bool(np.isnan(f_new))  # :230
    if low_pos < len(bracket):
        t = bracket[low_pos]
        f_new = bracket_f[low_pos]
    else:  # IndexError branch :235-237 (single-point bracket with low_pos == 1)
        t = 1.0
        line_search_failed = True
    if line_search_failed:  # :239-246
        while t > 1e-8:
            t = t * 0.8
            f_new, gtd_new, _ = obj_func(t)
            ls_func_evals += 1  # (the reference does not count these; harmless)
            if np.isnan(f_new):
                continue
            elif f_new < sdt(f + sdt(sdt(c1 * t) * gtd)):
                break
    if np.isnan(f_new):  # :247-249
        t = 0.0
        f_new, gtd_new, _ = obj_func(t)
    return f_new, t, ls_func_evals


# --------------------------------------------------------------------------------------
# projected L-BFGS solve (optim.py:69-184 driving lbfgs.py:390-590 with max_iter=1)
# --------------------------------------------------------------------------------------
class SolveStats(object):
    def __init__(self):
        self.average_distortions = []
        self.residual_norms = []
        self.step_size_percents = []
        self.step_lengths = []
        self.func_evals = 0

    @property
    def iterations(self):
        return len(self.average_distortions)


def embed(X0, edges, spec, constraint, eps=1e-5, max_iter=300, memory_size=10,
          dtype=np.float32, value_and_grad=None, trace=None):
    """Restatement of MDE.embed -> optim.lbfgs.  Returns (X, SolveStats).

    `trace`, if given, is called after every iteration with a dict of the solver state the device solver's debug
    view reports at a pause (X, g, g_prev, d, the stored pairs S and Y oldest first, H_diag, n_iter, func_evals);
    it changes nothing the solve computes.

    State kept between iterations mirrors lbfgs.py:581-588.  Note the reference quirk
    (SURVEY section 7.5): the gradient used by iteration k+1 is X.grad as left by the LAST
    closure evaluation of iteration k's line search, while the loss is the ACCEPTED
    trial's loss (`_cached_loss`, lbfgs.py:550)."""
    dt = np.dtype(dtype).type
    sdt = dt
    X = np.array(X0, dtype=dtype)
    stats = SolveStats()

    if value_and_grad is None:
        def value_and_grad(Xe):  # optim.py:100-105
            v, g = average_distortion(Xe, edges, spec, True, dtype)
            stats.func_evals += 1
            return float(dt(v)), constraint.tangent(Xe, g)

    state = {"n_iter": 0}
    cached_loss = None
    grad = None
    for _ in range(max_iter):
        norm_X = dt(np.sqrt((X.astype(np.float64) ** 2).sum()))  # optim.py:129-130
        # ---- LBFGS.step, lbfgs.py:390 ----
        if state["n_iter"] > 0:  # :418-426
            loss = cached_loss
        else:
            loss, grad = value_and_grad(X)
        stats.average_distortions.append(loss)  # callback, optim.py:94-96
        stats.residual_norms.append(float(dt(np.sqrt((grad.astype(np.float64) ** 2).sum()))))
        flat_grad = grad.reshape(-1).copy()

        state["n_iter"] += 1
        if state["n_iter"] == 1:  # :461-466
            d = -flat_grad
            old_dirs, old_stps, ro = [], [], []
            H_diag = dt(1.0)
        else:  # :467-507
            d, t_prev = state["d"], state["t"]
            old_dirs, old_stps, ro, H_diag = (state["old_dirs"], state["old_stps"],
                                              state["ro"], state["H_diag"])
            y = flat_grad - state["prev_flat_grad"]
            s = d * dt(t_prev)
            ys = dt(np.dot(y.astype(np.float64), s.astype(np.float64)))
            if ys > 1e-10:
                if len(old_dirs) == memory_size:
                    old_dirs.pop(0)
                    old_stps.pop(0)
                    ro.pop(0)
                old_dirs.append(y)
                old_stps.append(s)
                ro.append(dt(1.0) / ys)
                H_diag = ys / dt(np.dot(y.astype(np.float64), y.astype(np.float64)))
            num_old = len(old_dirs)
            al = [None] * num_old
            q = -flat_grad
            for i in range(num_old - 1, -1, -1):
                al[i] = dt(np.dot(old_stps[i].astype(np.float64), q.astype(np.float64))) * ro[i]
                q = q - al[i] * old_dirs[i]
            d = r = q * H_diag
            for i in range(num_old):
                be_i = dt(np.dot(old_dirs[i].astype(np.float64), r.astype(np.float64))) * ro[i]
                r = r + (al[i] - be_i) * old_stps[i]
            d = r
        prev_flat_grad = flat_grad.copy()

        if state["n_iter"] == 1:  # :521-524
            inv = dt(1.0) / dt(np.abs(flat_grad.astype(np.float64)).sum())
            t = inv if inv < 1.0 else 1.0
        else:
            t = 1
        gtd = dt(np.dot(flat_grad.astype(np.float64), d.astype(np.float64)))  # :527

        x_init = X.copy()
        d_mat = d.reshape(X.shape)
        d_norm = dt(np.abs(d).max())

        def obj_func(tt):  # _directional_evaluate, :368-376
            nonlocal grad
            Xe = constraint.project((x_init + dt(tt) * d_mat).astype(dtype))
            v, g = value_and_grad(Xe)
            grad = g
            gflat = g.reshape(-1)
            gd = dt(np.dot(gflat.astype(np.float64), d.astype(np.float64)))
            return v, gd, bool(np.isfinite(gflat).all())

        loss_new, t, _ = strong_wolfe(obj_func, t, loss, gtd, d_norm, sdt=sdt)
        # :550 `torch.tensor(loss)` is an fp32 tensor whatever dtype the problem runs in
        cached_loss = float(np.float32(loss_new))
        X = (x_init + dt(t) * d_mat).astype(dtype)  # :551 (not projected here)
        state.update(d=d, t=t, old_dirs=old_dirs, old_stps=old_stps, ro=ro, H_diag=H_diag,
                     prev_flat_grad=prev_flat_grad)
        # ---- back in optim.lbfgs ----
        X = constraint.project(X)  # optim.py:135-136
        h = float(t)
        pc = 100.0 * h * float(dt(np.sqrt((d.astype(np.float64) ** 2).sum()))) / float(norm_X)
        stats.step_size_percents.append(pc)
        stats.step_lengths.append(h)
        stop = stats.residual_norms[-1] <= eps  # :165
        if not stop and h == 0:  # :172-173 -> reset, lbfgs.py:378-388
            state = {"n_iter": 0}
        if trace is not None:
            trace(_trace_point(X, grad, prev_flat_grad, d, state, stats.func_evals))
        if stop:
            break
    return X, stats


def _trace_point(X, grad, prev_flat_grad, d, state, func_evals):
    """What the device solver's debug view (mde_solver_debug_lbfgs) reads at a pause, as copies."""
    held = state["n_iter"] > 0
    shape = X.shape
    return {"X": X.copy(), "g": grad.reshape(shape).copy(), "g_prev": prev_flat_grad.reshape(shape).copy(),
            "d": d.reshape(shape).copy(),
            "S": [s.reshape(shape).copy() for s in state["old_stps"]] if held else [],
            "Y": [y.reshape(shape).copy() for y in state["old_dirs"]] if held else [],
            "H_diag": float(state["H_diag"]) if held else 1.0, "n_iter": state["n_iter"],
            "func_evals": func_evals}


# --------------------------------------------------------------------------------------
# helpers to build a FnSpec from a reference (or pymde_b200) distortion-function object
# --------------------------------------------------------------------------------------
_PEN = {"Linear": P_LINEAR, "Quadratic": P_QUADRATIC, "Cubic": P_CUBIC, "Power": P_POWER,
        "Huber": P_HUBER, "Logistic": P_LOGISTIC, "Log1p": P_LOG1P, "Log": P_LOG,
        "InvPower": P_INVPOWER, "LogRatio": P_LOGRATIO}
_LOSS = {"Absolute": L_ABSOLUTE, "Quadratic": L_QUADRATIC,
         "WeightedQuadratic": L_WEIGHTED_QUADRATIC, "Huber": L_HUBER, "Cubic": L_CUBIC,
         "Power": L_POWER, "Logistic": L_LOGISTIC, "Fractional": L_FRACTIONAL,
         "SoftFractional": L_SOFT_FRACTIONAL}


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _scalars(f):
    name = type(f).__name__
    if hasattr(f, "exponent"):
        return (float(_np(f.exponent)), 0.0, 0.0)
    if hasattr(f, "gamma"):
        return (float(_np(f.gamma)), 0.0, 0.0)
    if name == "Logistic" and hasattr(f, "alpha"):
        return (float(f.threshold), float(f.alpha), 0.0)
    if hasattr(f, "threshold"):
        return (float(f.threshold), 0.0, 0.0)
    return (0.0, 0.0, 0.0)


def spec_from_function(f):
    """Translate a distortion-function module (reference or pymde_b200) into a FnSpec."""
    name = type(f).__name__
    mod = type(f).__module__
    if name == "PushAndPull":
        a, r = f.attractive_penalty, f.repulsive_penalty
        return FnSpec(_PEN[type(a).__name__], _np(f.weights), _scalars(a),
                      fn_rep=_PEN[type(r).__name__], rep=_scalars(r))
    if "losses" in mod:
        par1 = _np(f.weights) if name == "WeightedQuadratic" else None
        return FnSpec(_LOSS[name], _np(f.deviations), _scalars(f), par1=par1)
    return FnSpec(_PEN[name], _np(f.weights), _scalars(f))
