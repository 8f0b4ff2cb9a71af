"""Host-stepped projected L-BFGS for problems the device-resident solver does not take:
user-defined constraints (any `Constraint` subclass) unless PYMDE_B200_CONSTRAINT=device|graph|hook
asks for the device-resident solver (and always on edge-sharded problems), memory_size > 32,
use_line_search=False or use_cached_loss=False, embedding dimensions past the evaluation kernels' caps, and Python
callables as distortion functions on edge-sharded problems or under PYMDE_B200_EXTERNAL=generic
(other callables, and opted-in constraints, run on the device-resident solver, pymde_b200/external.py).

Same algorithm as pymde/optim.py:69-184 + pymde/lbfgs.py (history update :461-507, strong
Wolfe :44-253, cached loss :418-426, stale-gradient quirk); tensors stay on the CUDA device,
the objective still goes through the fused CUDA kernel via `MDE.average_distortion`; only the
control flow and the small vector algebra are host-driven torch ops."""
import time

import torch

from . import util


def _cubic(x1, f1, g1, x2, f2, g2, bounds=None):
    if bounds is not None:
        lo, hi = bounds
    else:
        lo, hi = (x1, x2) if x1 <= x2 else (x2, x1)
    d1 = g1 + g2 - 3 * (f1 - f2) / (x1 - x2)
    sq = d1 * d1 - g1 * g2
    if sq >= 0:
        d2 = sq ** 0.5
        if x1 <= x2:
            pos = x2 - (x2 - x1) * ((g2 + d2 - d1) / (g2 - g1 + 2 * d2))
        else:
            pos = x1 - (x1 - x2) * ((g1 + d2 - d1) / (g1 - g2 + 2 * d2))
        return min(max(pos, lo), hi)
    return (lo + hi) / 2.0


def _wolfe(phi, t, f, gtd, d_norm, c1=1e-4, c2=0.9, tol=1e-9, max_ls=25):
    """phi(t) -> (loss: float, g.d: float, finite: bool).  Returns (loss, t)."""
    nan = lambda v: v != v
    for _ in range(10):
        f_new, gtd_new, ok = phi(t)
        if nan(f_new) or f_new in (float("inf"), float("-inf")) or not ok:
            t *= 0.5
        else:
            break
    else:
        raise util.SolverError("Function or gradient evaluation returned NaN/inf.")
    t_prev, f_prev, gtd_prev = 0.0, f, gtd
    done, it = False, 0
    br = None
    while it < max_ls:
        if f_new > f + c1 * t * gtd or (it > 1 and f_new >= f_prev):
            br = [[t_prev, t], [f_prev, f_new], [gtd_prev, gtd_new]]
            break
        if abs(gtd_new) <= -c2 * gtd:
            br = [[t], [f_new], [gtd_new]]
            done = True
            break
        if gtd_new >= 0:
            br = [[t_prev, t], [f_prev, f_new], [gtd_prev, gtd_new]]
            break
        lo, hi = t + 0.01 * (t - t_prev), t * 10
        tn = _cubic(t_prev, f_prev, gtd_prev, t, f_new, gtd_new, (lo, hi))
        t_prev, f_prev, gtd_prev = t, f_new, gtd_new
        t = tn
        f_new, gtd_new, _ = phi(t)
        it += 1
    if it == max_ls:
        br = [[0.0, t], [f, f_new], [gtd, gtd_new]]
    bt, bf, bg = br
    insuf = False
    low, high = (0, 1) if bf[0] <= bf[-1] else (1, 0)
    while not done and it < max_ls:
        if abs(bt[1] - bt[0]) * d_norm < tol:
            break
        t = _cubic(bt[0], bf[0], bg[0], bt[1], bf[1], bg[1])
        bmax, bmin = max(bt), min(bt)
        eps = 0.1 * (bmax - bmin)
        if min(bmax - t, t - bmin) < eps:
            if insuf or t >= bmax or t <= bmin:
                t = bmax - eps if abs(t - bmax) < abs(t - bmin) else bmin + eps
                insuf = False
            else:
                insuf = True
        else:
            insuf = False
        f_new, gtd_new, _ = phi(t)
        it += 1
        if nan(f_new) or f_new > f + c1 * t * gtd or f_new >= bf[low]:
            bt[high], bf[high], bg[high] = t, f_new, gtd_new
            low, high = (0, 1) if bf[0] <= bf[1] else (1, 0)
        else:
            if abs(gtd_new) <= -c2 * gtd:
                done = True
            elif gtd_new * (bt[high] - bt[low]) >= 0:
                bt[high], bf[high], bg[high] = bt[low], bf[low], bg[low]
            bt[low], bf[low], bg[low] = t, f_new, gtd_new
    failed = nan(f_new)
    if low < len(bt):
        t, f_new = bt[low], bf[low]
    else:
        t, failed = 1.0, True
    if failed:
        while t > 1e-8:
            t *= 0.8
            f_new, gtd_new, _ = phi(t)
            if nan(f_new):
                continue
            if f_new < f + c1 * t * gtd:
                break
    if nan(f_new):
        t = 0.0
        f_new, gtd_new, _ = phi(t)
    return f_new, t


def lbfgs_generic(X, objective_fn, constraint, eps, max_iter, memory_size, use_line_search, use_cached_loss,
                  verbose, print_every, snapshot_every, logger):
    from .optim import SolveStats
    start_time = time.time()
    if X.device.type != "cuda":
        raise ValueError("pymde_b200 solves on CUDA tensors only")
    avgs, resids, pcts, times, snaps = [], [], [], [], []
    evals = [0]
    grad = [None]

    def closure(Xe):
        Xe = Xe.detach().requires_grad_(True)
        v = objective_fn(Xe)
        v.backward()
        g = Xe.grad
        with torch.no_grad():
            g = constraint.project_onto_tangent_space(Xe.detach(), g, inplace=True)
        evals[0] += 1
        grad[0] = g
        return float(v.detach())

    state = None
    cached = None
    digits = len(str(max_iter))
    start = time.time()
    with torch.no_grad():
        for iteration in range(max_iter):
            if snapshot_every is not None and iteration % snapshot_every == 0:
                snaps.append(X.detach().cpu().clone())
            norm_X = float(X.norm())
            if state is not None and use_cached_loss:
                loss = cached
            else:
                with torch.enable_grad():
                    loss = closure(X)
            avgs.append(loss)
            g = grad[0].reshape(-1)
            resids.append(float(g.norm()))
            if state is None:
                d = -g
                S, Y, ro, H = [], [], [], 1.0
            else:
                d, t_prev, S, Y, ro, H, g_prev = state
                y = g - g_prev
                s = d * t_prev
                ys = float(y.dot(s))
                if ys > 1e-10:
                    if len(S) == memory_size:
                        S.pop(0), Y.pop(0), ro.pop(0)
                    S.append(s), Y.append(y), ro.append(1.0 / ys)
                    H = ys / float(y.dot(y))
                q = -g
                al = [0.0] * len(S)
                for i in range(len(S) - 1, -1, -1):
                    al[i] = float(S[i].dot(q)) * ro[i]
                    q = q - al[i] * Y[i]
                r = q * H
                for i in range(len(S)):
                    be = float(Y[i].dot(r)) * ro[i]
                    r = r + (al[i] - be) * S[i]
                d = r
            g_prev = g.clone()
            t = min(1.0, 1.0 / float(g.abs().sum())) if state is None else 1.0
            gtd = float(g.dot(d))
            x0 = X.clone()
            dmat = d.view_as(X)

            def phi(tt):
                Xe = constraint.project_onto_constraint(x0 + tt * dmat, inplace=True)
                with torch.enable_grad():
                    v = closure(Xe)
                gf = grad[0].reshape(-1)
                return v, float(gf.dot(d)), bool(torch.isfinite(gf).all())

            if use_line_search:
                loss_new, t = _wolfe(phi, t, loss, gtd, float(d.abs().max()))
                cached = loss_new
            X.copy_(constraint.project_onto_constraint(x0 + t * dmat, inplace=True))
            state = (d, t, S, Y, ro, H, g_prev)
            times.append(time.time() - start)
            pc = 100.0 * t * float(d.norm()) / norm_X
            pcts.append(pc)
            if verbose and ((iteration % print_every == 0) or (iteration == max_iter - 1)):
                logger.info("iteration %0*d | distortion %6f | residual norm %g | step length %g | "
                            "percent change %g" % (digits, iteration, avgs[-1], resids[-1], t, pc))
            if resids[-1] <= eps:
                if verbose:
                    logger.info("Converged in %03d iterations, with residual norm %g" % (iteration + 1, resids[-1]))
                break
            elif t == 0:
                state = None
    stats = SolveStats(avgs, resids, pcts, time.time() - start_time, times, snaps, snapshot_every)
    stats.func_evals = evals[0]
    return X, stats
