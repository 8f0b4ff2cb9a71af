"""The device-resident L-BFGS solver (csrc/mde_solver.cu), iteration by iteration, against the fp64 replay of
tests/lbfgs_replay.py: the solve is paused after every iteration (run(1)), the solver's own L-BFGS state is read
(DeviceSolver.debug_lbfgs) and every pause is checked against the previous one -- direction, gradient bookkeeping,
history update bit for bit, the move, the statistics and the line-search conditions.

History sizes 1..32 cover every boundary of the head kernel's 10-pair slices (memory 11-32 runs 2-4 slices) and each
solve runs N = 2 memory + 12 iterations, so that the history wraps at least once.  The constraints and widths reach
fused centering (m = 1, 2, 4), the separate centering kernel (m = 3), the Jacobi (m = 2) and Newton-Schulz (m = 40)
retractions, Anchored, and the wide distortion kernel (m = 8).  Pausing must not perturb the solve: the cases on the
default layout at m <= 4, whose gradient is bit-reproducible (DESIGN section 5), also run run(N) in one call and must
end bit-identical -- the paused solve builds each history pair in the resume pass, the uninterrupted one speculatively
in the step that evaluated it, and only bitwise equality carries the replay's verdict over to the uninterrupted path.

Problems: PushAndPull(Log1p, Log) on a k-NN-like graph, n = 3000, built from seeds in tests/lbfgs_replay.py; eps = 0.
Tolerances: lbfgs_replay.TOL (derived from the fp32 oracle's trace of these same cases, as stated there).
Worst device errors over the cases, measured on an H100 80GB HBM3 at a 700 W power limit (tolerance in brackets):
direction 2.0e-6 (3.9e-5; Centered m = 1), H_diag 4.5e-7 (1e-5), move 4.7e-7 (1.1e-6; Standardized m = 40,
Newton-Schulz), average distortion 1.1e-7 (1.0e-6), residual 1.3e-7 (5.8e-7), gradient 6.8e-7 (2.7e-6; Centered
m = 3), step percent 1.6e-7 (1.0e-6), first step 8.7e-8 (1e-6), Armijo excess 6.1e-8 (2.4e-7; docs5), curvature
excess 0 (1e-5); docs5 resets its history 49 times.  The file runs in about 25 s on that card."""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O
from tests import lbfgs_replay as L

pytestmark = pytest.mark.gpu

N_ROWS = 3000
SWEEP = [1, 2, 9, 10, 11, 19, 20, 21, 31, 32]
MATRIX = [("centered", 1), ("centered", 4), ("centered", 3), ("standardized", 2), ("standardized", 40),
          ("anchored", 2), ("centered", 8)]


def _case(cname, m, scale=1.0):
    """(pymde_b200 MDE, X0 on the device, fp64 Problem)."""
    import pymde_b200 as pm
    edges, w = L.knn_graph(N_ROWS, 6, 11, scale)
    if cname == "centered":
        ocons, cons = O.Centered(), pm.Centered()
    elif cname == "standardized":
        ocons, cons = O.Standardized(), pm.Standardized()
    else:
        anchors = np.arange(0, N_ROWS, N_ROWS // 7)[:7]
        values = np.random.default_rng(5).standard_normal((len(anchors), m)).astype(np.float32)
        ocons = O.Anchored(anchors, values)
        cons = pm.Anchored(torch.tensor(anchors, device="cuda"), torch.tensor(values, device="cuda"))
    X0 = L.initial_point(N_ROWS, m, ocons, 3)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(N_ROWS, m, torch.tensor(edges, device="cuda"), f, cons)
    return mde, torch.tensor(X0, device="cuda"), L.Problem(edges, L.push_pull_spec(w), ocons)


def paused_solve(mde, X0, memory, iters):
    """Run `iters` iterations one at a time; (pauses, stats) as lbfgs_replay.replay takes them."""
    solver = mde._solver(mde.constraint, memory, iters + 1)
    solver.begin(X0, 0.0, iters + 1)  # one more than is run: the solve is paused, not finished, after the last one
    with pytest.raises(Exception):
        solver.debug_lbfgs()  # not paused yet
    pauses = [{"X": X0.cpu().numpy(), "func_evals": 0}]
    for k in range(1, iters + 1):
        done, _ = solver.run(1)
        assert done == k
        r = solver.debug_lbfgs()
        p = {n: r[n].numpy().copy() for n in ("g", "g_prev", "d", "S", "Y")}
        p.update(count=r["count"], H_diag=r["H_diag"], n_iter=r["n_iter"], func_evals=solver.stats(k)[4],
                 X=solver.x_view().cpu().numpy())
        pauses.append(p)
    avg, res, pct, stp, fe = solver.stats(iters)
    return pauses, {"average": avg, "residual": res, "percent": pct, "steplen": stp, "func_evals": fe}


def whole_solve(mde, X0, memory, iters):
    solver = mde._solver(mde.constraint, memory, iters + 1)
    solver.begin(X0, 0.0, iters + 1)
    done, _ = solver.run(iters)
    assert done == iters
    avg, res, pct, stp, fe = solver.stats(iters)
    return solver.x_view().cpu().numpy(), {"average": avg, "residual": res, "percent": pct, "steplen": stp,
                                           "func_evals": fe}


def _check(cname, m, memory, scale=1.0, iters=None):
    mde, X0, prob = _case(cname, m, scale)
    iters = iters or 2 * memory + 12
    pauses, stats = paused_solve(mde, X0, memory, iters)
    R = L.replay(pauses, stats, prob, memory)
    if m <= 4:
        X, whole = whole_solve(mde, X0, memory, iters)
        assert np.array_equal(X, pauses[-1]["X"]), "pausing after every iteration changed X"
        for name in ("average", "residual", "percent", "steplen", "func_evals"):
            assert np.array_equal(whole[name], stats[name]), "pausing after every iteration changed " + name
    return R, pauses


@pytest.mark.parametrize("memory", SWEEP)
def test_history_sizes_replay_exactly(memory):
    """Centered, m = 2 (centering fused into the vector kernel, column sums tracked per history slot)."""
    R, _ = _check("centered", 2, memory)
    assert R.evicted >= memory + 1, "the history must wrap"


@pytest.mark.parametrize("memory", [10, 32])
@pytest.mark.parametrize("cname,m", MATRIX)
def test_constraints_and_widths_replay_exactly(cname, m, memory):
    R, pauses = _check(cname, m, memory)
    assert R.evicted >= 1


def test_rejected_pairs_keep_steepest_descent():
    """Weights scaled by 1e-4: y.s < 1e-10 from the first pair on, so every pair is rejected, count stays 0 and
    d = -g_prev with H_diag = 1 at every pause."""
    R, pauses = _check("centered", 2, 10, scale=1e-4)
    assert R.accepted == 0 and R.rejected == len(pauses) - 2
    assert all(p["count"] == 0 and p["H_diag"] == 1.0 for p in pauses[1:])


def test_converging_problem_replays_exactly(golden):
    """docs5 (Quadratic, Standardized, n = 5) for 60 iterations at eps = 0: it converges, its line searches end at
    t = 0 and the solver resets its history (optim.py:172-173) at almost every iteration -- n_iter, the direction
    (d = -g_prev after each reset) and the rest hold through the resets."""
    from tests.test_gpu_solver import build
    import pymde_b200 as pm
    g = golden["trajectories"]
    mde, X0 = build(pm, "docs5", g)
    prob = L.Problem(g["docs5/edges"], O.FnSpec(O.P_QUADRATIC, g["docs5/par0"]), O.Standardized())
    pauses, stats = paused_solve(mde, X0, 10, 60)
    R = L.replay(pauses, stats, prob, 10)
    assert R.resets >= 40  # the fp32 oracle resets 50 times on this problem
    X, whole = whole_solve(mde, X0, 10, 60)
    assert np.array_equal(X, pauses[-1]["X"])
    for name in ("average", "residual", "steplen", "func_evals"):
        assert np.array_equal(whole[name], stats[name]), name


def test_history_sizes_route_to_the_device_solver():
    """memory_size <= 32 runs on the device solver, 33 on the host-stepped one."""
    mde, _, _ = _case("centered", 2)
    assert mde._fused_ok(mde.constraint, 32)
    assert not mde._fused_ok(mde.constraint, 33)
