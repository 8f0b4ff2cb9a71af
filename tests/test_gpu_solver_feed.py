"""mde_solver_run keeps the step queue fed from the device's progress word and takes a clean stop from it without
synchronising: the solve it runs is the one a single run(N) runs, bit for bit, however the N iterations are split over
calls; iters_done and converged are exact; a non-finite loss still raises SolverError; and no step is enqueued after
the device pauses at the requested iteration count."""
import ctypes as C

import numpy as np
import pytest
import torch

import bench

pytestmark = pytest.mark.gpu
KERNELS_PER_STEP = 3  # Centered at m = 2: head, vector and owner kernels
BIG = 8  # steps of the multi-step graph


def c2_problem(n=20000, k=15):
    import pymde_b200 as pm
    dev = torch.device("cuda", 0)
    edges, w = bench.c2_edges(0, n=n, k=k) if n != bench.N_ITEMS else bench.c2_edges(0)
    X0 = bench.initial_iterate(1, n=n)
    f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, bench.EMBED_DIM, torch.tensor(edges, device=dev), f, pm.Centered(), device=dev)
    return mde, torch.tensor(X0, device=dev)


def run_steps(solver):
    from pymde_b200 import _lib
    launched, ran = C.c_int64(0), C.c_int64(0)
    _lib.check(_lib.load().mde_solver_debug_run_steps(solver.handle, C.byref(launched), C.byref(ran)))
    return launched.value, ran.value


def solve(mde, X0, chunks, cap):
    solver = mde._solver(mde.constraint, 10, cap)
    solver.begin(X0, 0.0, cap)
    done = 0
    for c in chunks:
        before = done
        done, conv = solver.run(c)
        assert done == min(before + c, cap) and not conv
    avg, res, pct, stp, fe = solver.stats(done)
    return done, solver.x_view().clone(), (avg.copy(), res.copy(), pct.copy(), stp.copy()), fe


def test_split_runs_are_bit_identical_to_one_run():
    mde, X0 = c2_problem()
    N = 40
    ref = solve(mde, X0, (N,), N)
    for chunks in ((1,) * N, (3, 8, 9, 20), (7, 1, 32)):
        got = solve(mde, X0, chunks, N)
        assert got[0] == N and got[3] == ref[3]
        assert torch.equal(got[1], ref[1]), chunks
        for a, b in zip(got[2], ref[2]):
            np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("iters", [1, 7, 8, 9, 20, 97])
def test_iters_done_is_exact_and_no_surplus_step(iters):
    from pymde_b200 import _lib
    lib = _lib.load()
    mde, X0 = c2_problem()
    solver = mde._solver(mde.constraint, 10, 2 * iters + 1)
    solver.begin(X0, 0.0)
    for call in (1, 2):  # a fresh solve, then a resumed one
        l0 = int(lib.mde_launch_count())
        done, conv = solver.run(iters)
        assert done == call * iters and not conv
        launched, ran = run_steps(solver)
        assert int(lib.mde_launch_count()) - l0 == launched * KERNELS_PER_STEP + 1  # (+ the resume kernel)
        assert ran >= iters and launched == ran, (launched, ran)


def test_convergence_stops_the_feed():
    import pymde_b200 as pm
    n = 200
    edges = pm.all_edges(n)
    mde = pm.MDE(n, 2, edges.cuda(), pm.penalties.Quadratic(torch.ones(edges.shape[0])), pm.Standardized())
    X0 = mde.constraint.project_onto_constraint(torch.randn(n, 2, generator=torch.Generator().manual_seed(0)).cuda())
    solver = mde._solver(mde.constraint, 10, 500)
    solver.begin(X0, 1e-4)
    done, conv = solver.run(500)
    assert conv and 0 < done < 500
    launched, ran = run_steps(solver)
    # convergence cannot be foreseen: up to the two eight-step graphs kept queued run gated after it
    assert 0 <= launched - ran <= 2 * BIG, (launched, ran)
    assert solver.run(10) == (done, True)  # a converged solve does not resume


def test_non_finite_loss_raises_solver_error():
    import pymde_b200 as pm
    n = 50
    edges = pm.all_edges(n).cuda()
    mde = pm.MDE(n, 2, edges, pm.penalties.Log(-torch.ones(edges.shape[0], device="cuda")), pm.Centered())
    solver = mde._solver(mde.constraint, 10, 20)
    solver.begin(torch.zeros(n, 2, device="cuda"), 0.0)
    with pytest.raises(pm.util.SolverError):
        solver.run(20)


def test_benchmark_windows_enqueue_no_surplus_step():
    """bench.py's shape: the full C2 workload, warm-up, then run(20) windows."""
    mde, X0 = c2_problem(bench.N_ITEMS)
    solver = mde._solver(mde.constraint, 10, 200)
    solver.begin(X0, 0.0)
    solver.run(10)
    for w in range(5):
        done, _ = solver.run(20)
        assert done == 10 + 20 * (w + 1)
        launched, ran = run_steps(solver)
        assert launched == ran, (w, launched, ran)
