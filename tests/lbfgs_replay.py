"""Replay of a projected L-BFGS solve in fp64, pause by pause (no GPU import).

A solve is recorded as the state read at the pause after every iteration (the device solver's debug view,
`DeviceSolver.debug_lbfgs()`, or the oracle's `embed(trace=...)`), and `replay()` checks that consecutive pauses follow
the rules of pymde/lbfgs.py:390-590 and pymde/optim.py:69-184.  Notation: (k) means "read at the pause after k
iterations".  g^(k) is the gradient buffer there (the last evaluation of iteration k-1: the reference's stale-gradient
quirk), g_prev^(k) and d^(k) the gradient and direction of iteration k-1, t_{k-1} = step_lengths[k-1] its step, and
X_k the iterate.  Every check uses the solver's own vectors, so fp32 drift between two trajectories never builds up:

  direction      d^(k) = explicit two-loop recursion (lbfgs.py:488-507) on g_prev^(k), the pairs and H_diag of
                 iteration k-1, in fp64 (relative infinity norm); d^(k) = -g_prev^(k) bit for bit while no pair is held
  n_iter         one more per iteration, back to 0 exactly when the accepted step was 0 (a reset, optim.py:172-173)
  bookkeeping    g_prev^(k) == g^(k-1) bit for bit (after a reset: the fresh evaluation at X_{k-1})
  history        the candidate pair of iteration k-1, s = fl32(d^(k-1) fl32(t_{k-2})), y = fl32(g^(k-1) - g_prev^(k-1)),
                 is appended bit for bit iff y.s > 1e-10 (the oldest pair evicted when the history was full, the others
                 unchanged and in order), H_diag = fl32(y.s) / fl32(y.y); otherwise history and H_diag are unchanged;
                 a reset leaves nothing held.  The direction is checked on the pairs the iteration used, so also at a
                 pause that follows a reset
  move           X_k = fp64 projection of X_{k-1} + t_{k-1} d^(k) (exact mean, fp64 polar factor, exact anchor rows)
  statistics     average_distortions[k] = fp64 value at X_k, residual_norms[k] = ||g^(k)||, step_size_percents and
                 the first step length by their formulas; where iteration k-1 took one evaluation, g^(k) = the fp64
                 tangent-projected gradient at X_k
  line search    Armijo for every accepted step, the strong curvature condition where the search took one evaluation

The tolerances come from the fp32 oracle's own trace of the same cases; see `TOL`.
"""
import numpy as np

from oracle import mde_oracle as O

C1, C2 = 1e-4, 0.9  # strong-Wolfe constants (lbfgs.py:44)
YS_MIN = 1e-10      # curvature threshold of the history update (lbfgs.py:474)
EPS32 = float(np.finfo(np.float32).eps)

# name -> tolerance.  Where the fp32 oracle's trace shows an error against this replay, the tolerance is 10 x its
# worst error over every case of tests/test_gpu_lbfgs_replay.py (run through the oracle on the CPU, docs5 included) and
# of tests/test_lbfgs_replay_cpu.py; the comment gives that worst error and its case.  Where the oracle shows none,
# because it evaluates the same fp32 formula as the solver, the tolerance is the fp32 rounding a different summation
# order can cause, stated with it.
TOL = {
    "direction": 3.9e-5,  # relative infinity norm of d - two-loop; oracle 3.93e-6 (Centered, m = 1, memory 32)
    "h_diag": 1e-5,       # relative, H_diag against fl32(y.s) / fl32(y.y); oracle 0: y.s and y.y summed in another
    #                       order move the quotient by a few ulp (1e-5 = 80 ulp)
    "move": 1.1e-6,       # infinity norm of X_k - projection, relative to its infinity norm; oracle 1.07e-7
    #                       (Standardized, m = 2, memory 32)
    "average": 1.0e-6,    # relative; oracle 1.04e-7 (docs5)
    "residual": 5.8e-7,   # relative; oracle 5.83e-8 (Standardized, m = 40, memory 32)
    "gradient": 2.7e-6,   # absolute, times max |fp64 gradient| (the gradient at X_0 sets a floor on the scale);
    #                       oracle 2.72e-7 (Centered, m = 8, memory 32)
    "percent": 1.0e-6,    # relative; oracle 9.99e-8 (Centered, m = 3, memory 10)
    "first_step": 1e-6,   # relative; oracle 0: |g|_1 summed in another order moves 1/|g|_1 by an ulp or two
    "armijo": 2 * EPS32,  # excess over the Armijo bound relative to |f|; oracle 8.4e-12: the reference tests the
    #                       condition in fp32, so one rounding of f either way
    "curvature": 1e-5,    # excess over the curvature bound relative to |g_prev.d|; oracle 0: fp32 dots summed in
    #                       another order
}


def explicit_two_loop(g, S, Y, H_diag):
    """lbfgs.py:488-507 with explicit vectors (float64)."""
    q = -np.array(g, dtype=np.float64)
    h = len(S)
    al = [0.0] * h
    ro = [1.0 / float(Y[i] @ S[i]) for i in range(h)]
    for i in range(h - 1, -1, -1):
        al[i] = float(S[i] @ q) * ro[i]
        q -= al[i] * Y[i]
    r = q * H_diag
    for i in range(h):
        be = float(Y[i] @ r) * ro[i]
        r += (al[i] - be) * S[i]
    return r


# --------------------------------------------------------------------------------------
# problems (numpy only: the GPU tests build the same problems as pymde_b200 objects)
# --------------------------------------------------------------------------------------
def knn_graph(n, k, seed, scale=1.0):
    """k-NN-like attractive edges plus as many random repulsive ones (the generator of test_gpu_solver._knn_problem);
    PushAndPull(Log1p, Log) weights +-scale."""
    rng = np.random.default_rng(seed)
    i = np.repeat(np.arange(n), k)
    j = (i + rng.integers(1, 50, n * k)) % n
    att = np.unique(np.sort(np.stack([i, j], 1), axis=1), axis=0)
    rep = rng.integers(0, n, (len(att), 2))
    rep = rep[rep[:, 0] != rep[:, 1]]
    rep = np.unique(np.sort(rep, axis=1), axis=0)
    key = lambda e: e[:, 0].astype(np.int64) * n + e[:, 1]
    rep = rep[~np.isin(key(rep), key(att))]
    edges = np.concatenate([att, rep]).astype(np.int64)
    w = (scale * np.concatenate([np.ones(len(att)), -np.ones(len(rep))])).astype(np.float32)
    return edges, w


def push_pull_spec(w):
    return O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))


def initial_point(n, m, constraint, seed):
    """A feasible X_0, except under Centered: there it is shifted off centre by half a unit per column, so that the
    first retraction removes a mean that matters (later ones only remove rounding: the objective is translation
    invariant, its gradient sums to zero)."""
    X0 = np.random.default_rng(seed + 7919).standard_normal((n, m)).astype(np.float32)
    X0 = constraint.project(X0.astype(np.float64))
    if getattr(constraint, "name", "") == "centered":
        X0 = X0 + 0.5
    return X0.astype(np.float32)


class Problem(object):
    """What the replay evaluates in fp64: the objective and the constraint."""

    def __init__(self, edges, spec, constraint):
        self.edges, self.spec, self.constraint = edges, spec, constraint

    def value_and_grad(self, X):
        X = np.asarray(X, dtype=np.float64)
        v, g = O.average_distortion(X, self.edges, self.spec, True, np.float64)
        return v, self.constraint.tangent(X, g)

    def project(self, Z):
        return self.constraint.project(np.asarray(Z, dtype=np.float64))


def oracle_trace(problem, X0, memory, iters):
    """(pauses, stats) of the fp32 oracle on `problem`, in the form replay() takes."""
    pauses = [{"X": np.array(X0, dtype=np.float32), "func_evals": 0}]
    _, st = O.embed(X0, problem.edges, problem.spec, problem.constraint, eps=0.0, max_iter=iters,
                    memory_size=memory, dtype=np.float32, trace=pauses.append)
    for p in pauses[1:]:
        p["S"] = np.array(p["S"], dtype=np.float32).reshape(-1, *X0.shape)
        p["Y"] = np.array(p["Y"], dtype=np.float32).reshape(-1, *X0.shape)
        p["count"] = len(p["S"])
    stats = {"average": np.array(st.average_distortions), "residual": np.array(st.residual_norms),
             "percent": np.array(st.step_size_percents), "steplen": np.array(st.step_lengths)}
    return pauses, stats


# --------------------------------------------------------------------------------------
# the replay
# --------------------------------------------------------------------------------------
def _f64(a):
    return np.asarray(a, dtype=np.float64).reshape(-1)


def _rel_inf(a, ref):
    a, ref = _f64(a), _f64(ref)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-300))


class Replay(object):
    def __init__(self, problem, memory, tol, strict):
        self.problem, self.memory, self.tol, self.strict = problem, memory, dict(TOL, **(tol or {})), strict
        self.worst = {k: 0.0 for k in self.tol}
        self.accepted = self.rejected = self.evicted = self.resets = 0

    def near(self, name, err, k, what=""):
        """Record a tolerance-checked error; fail (when strict) above the tolerance."""
        err = float(err)
        if not np.isfinite(err):
            raise AssertionError("%s at pause %d is not finite %s" % (name, k, what))
        self.worst[name] = max(self.worst[name], err)
        if self.strict and err > self.tol[name]:
            raise AssertionError("%s at pause %d: error %.3g > tolerance %.3g %s" % (name, k, err, self.tol[name], what))

    def exact(self, ok, k, what):
        if not ok:
            raise AssertionError("pause %d: %s" % (k, what))


def replay(pauses, stats, problem, memory, tol=None, strict=True, eps=0.0):
    """Check the pauses 0..N of one solve (see the module docstring).  pauses[0] holds X_0 and func_evals = 0 only;
    pauses[k >= 1] hold X, g, g_prev, d (n, m), S, Y (count, n, m) oldest first, count, H_diag, n_iter, func_evals
    (fp32 arrays as the solver stored them).  `stats` holds the arrays average, residual, percent, steplen of at least
    N entries; `eps` is the solve's residual tolerance.  Returns the Replay (worst error per quantity, counts of
    accepted, rejected and evicted pairs and of resets); raises AssertionError on a violation."""
    R = Replay(problem, memory, tol, strict)
    cons = problem.constraint
    N = len(pauses) - 1
    avg, res, pct, stp = (np.asarray(stats[k], dtype=np.float64) for k in ("average", "residual", "percent", "steplen"))
    assert min(len(avg), len(res), len(pct), len(stp)) >= N, "statistics shorter than the trace"
    f64 = {}  # k -> (value, gradient) at X_k

    def at(k):
        if k not in f64:
            f64[k] = problem.value_and_grad(pauses[k]["X"])
        return f64[k]

    def gscale(gref):  # near convergence the gradient is rounding noise of terms as large as those at X_0
        return max(np.abs(gref).max(), np.abs(at(0)[1]).max())

    kept = (lambda a, b: len(a) == len(b) and all(np.array_equal(u, v) for u, v in zip(a, b)))
    for k in range(1, N + 1):
        P, Q = pauses[k - 1], pauses[k]
        X0, X1 = np.asarray(P["X"]), np.asarray(Q["X"])
        g, gp, d = (np.asarray(Q[n], dtype=np.float32) for n in ("g", "g_prev", "d"))
        t = stp[k - 1]
        p_iter = P.get("n_iter", 0)  # pause 0: a new solve holds nothing
        fresh = p_iter == 0  # iteration k-1 began with an evaluation at X_{k-1} (first iteration / after a reset)
        ls_evals = Q["func_evals"] - P["func_evals"] - (1 if fresh else 0)
        R.exact(ls_evals >= 1, k, "iteration %d took %d line-search evaluations" % (k - 1, ls_evals))

        # ---- n_iter: one more per iteration (lbfgs.py:440), back to 0 after a step of 0 (optim.py:165-173) ----
        reset = t == 0 and not res[k - 1] <= eps
        R.exact(Q["n_iter"] == (0 if reset else p_iter + 1), k, "n_iter %d after %d and a step of %r: expected %s"
                % (Q["n_iter"], p_iter, t, "a reset to 0" if reset else "no reset, %d" % (p_iter + 1)))
        R.resets += int(reset)

        # ---- gradient bookkeeping ----
        if fresh:  # g_prev^(k) is the evaluation at X_{k-1}
            gref = at(k - 1)[1]
            R.near("gradient", np.abs(_f64(gp) - _f64(gref)).max() / gscale(gref), k, "(fresh evaluation)")
        else:
            R.exact(np.array_equal(gp, P["g"]), k, "g_prev is not the gradient buffer of the previous pause")

        # ---- history rule: the pairs iteration k-1 used (read at pause k unless it ended in a reset) ----
        if fresh:
            used = ([], [], 1.0)
        else:
            s = (np.asarray(P["d"], dtype=np.float32) * np.float32(stp[k - 2])).astype(np.float32)
            y = (np.asarray(P["g"], dtype=np.float32) - np.asarray(P["g_prev"], dtype=np.float32)).astype(np.float32)
            ys, yy = float(_f64(y) @ _f64(s)), float(_f64(y) @ _f64(y))
            band = abs(ys - YS_MIN) <= 1e-5 * np.linalg.norm(_f64(s)) * np.linalg.norm(_f64(y))
            full = P["count"] == memory
            S_acc = list(P["S"][1:] if full else P["S"]) + [s]
            Y_acc = list(P["Y"][1:] if full else P["Y"]) + [y]
            h_acc = float(np.float32(ys) / np.float32(yy))
            if not band:
                accept = ys > YS_MIN
            elif not reset:  # at the threshold fp32 summation order decides: take what the solver did
                accept = kept(Q["S"], S_acc) and kept(Q["Y"], Y_acc)
            else:
                accept = None  # unknowable: the reset cleared the history
            if accept is None:
                used = None
            elif accept:
                used = (S_acc, Y_acc, h_acc if reset else float(Q["H_diag"]))
            else:
                used = (list(P["S"]), list(P["Y"]), float(P["H_diag"]))
            if accept is not None and not reset:
                if accept and not (kept(Q["S"], S_acc) and kept(Q["Y"], Y_acc)):
                    newest = Q["count"] >= 1 and np.array_equal(Q["S"][-1], s) and np.array_equal(Q["Y"][-1], y)
                    R.exact(False, k, "accepted pair (y.s = %.3g) not appended as the rule says: count %d -> %d, "
                            "newest pair %s, %s" % (ys, P["count"], Q["count"],
                                                    "is the candidate" if newest else "is NOT the candidate",
                                                    "full: oldest must be evicted" if full else "not full"))
                if accept:
                    R.near("h_diag", abs(Q["H_diag"] - h_acc) / abs(h_acc), k)
                else:
                    R.exact(kept(Q["S"], P["S"]) and kept(Q["Y"], P["Y"]) and Q["H_diag"] == P["H_diag"], k,
                            "rejected pair (y.s = %.3g) changed the history or H_diag" % ys)
            if accept:
                R.accepted += 1
                R.evicted += int(full)
            elif accept is not None:
                R.rejected += 1
        if reset:
            R.exact(Q["count"] == 0 and Q["H_diag"] == 1.0, k, "history not empty after a reset: count %d, H_diag %r"
                    % (Q["count"], Q["H_diag"]))

        # ---- direction, from the pairs iteration k-1 used ----
        if used is not None:
            S_u, Y_u, H_u = used
            if not S_u:
                R.exact(H_u == 1.0 and np.array_equal(d, -gp), k, "d != -g_prev with no pair held")
            else:
                dref = explicit_two_loop(_f64(gp), [_f64(v) for v in S_u], [_f64(v) for v in Y_u], H_u)
                R.near("direction", _rel_inf(d, dref), k, "(count %d)" % len(S_u))

        # ---- move ----
        Z = np.asarray(X0, dtype=np.float64) + float(np.float32(t)) * np.asarray(d, dtype=np.float64)
        if getattr(cons, "name", "") == "anchored":
            R.exact(np.array_equal(X1[cons.anchors], cons.values.astype(np.float32)), k, "anchor rows moved")
        Pz = problem.project(Z)
        R.near("move", np.abs(np.asarray(X1, dtype=np.float64) - Pz).max() / np.abs(Pz).max(), k)

        # ---- statistics ----
        if k == 1:
            R.near("residual", abs(res[0] - np.linalg.norm(_f64(gp))) / np.linalg.norm(_f64(gp)), 0)
            R.near("average", abs(avg[0] - at(0)[0]) / abs(at(0)[0]), 0)
        if k < min(len(avg), len(res)):
            R.near("residual", abs(res[k] - np.linalg.norm(_f64(g))) / np.linalg.norm(_f64(g)), k)
            R.near("average", abs(avg[k] - at(k)[0]) / abs(at(k)[0]), k)
        dn, xn = np.linalg.norm(_f64(d)), np.linalg.norm(_f64(X0))
        R.near("percent", abs(pct[k - 1] - 100.0 * t * dn / xn) / max(abs(pct[k - 1]), 1e-300), k)
        if fresh and ls_evals == 1:
            g1 = float(np.float32(np.abs(_f64(gp)).sum()))
            inv = float(np.float32(1.0) / np.float32(g1))
            R.near("first_step", abs(t - min(inv, 1.0)) / min(inv, 1.0), k)
        if ls_evals == 1 and t > 0:
            gref = at(k)[1]
            R.near("gradient", np.abs(_f64(g) - _f64(gref)).max() / gscale(gref), k)

        # ---- line search ----
        gtd = float(_f64(gp) @ _f64(d))
        R.exact(gtd < 0, k, "d is not a descent direction (g_prev.d = %.3g)" % gtd)
        if k < len(avg):
            f0, f1 = avg[k - 1], avg[k]
            R.near("armijo", max(0.0, f1 - (f0 + C1 * t * gtd)) / abs(f0), k)
        if ls_evals == 1 and t > 0:
            gtd1 = float(_f64(g) @ _f64(d))
            R.near("curvature", max(0.0, abs(gtd1) - C2 * abs(gtd)) / abs(gtd), k)
    return R
