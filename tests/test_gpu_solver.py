"""GPU parity tests of the device-resident projected L-BFGS (mde_solver_*) through MDE.embed:
against the reference's own embed() trajectories (tests/golden/trajectories.npz) and the numpy
oracle, plus size-independent invariants of the constraint sets."""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O

pytestmark = pytest.mark.gpu

TRAJ = ["quad_std", "pp_cen", "pp_std", "cycle_abs", "huber_std", "docs5"]


def build(pm, key, g):
    par0 = torch.tensor(g[key + "/par0"], device="cuda")
    pen, los = pm.penalties, pm.losses
    f, c = {
        "quad_std": (lambda: pen.Quadratic(par0), pm.Standardized()),
        "pp_cen": (lambda: pen.PushAndPull(par0, pen.Log1p, pen.Log), pm.Centered()),
        "pp_std": (lambda: pen.PushAndPull(par0, pen.Log1p, pen.Log), pm.Standardized()),
        "cycle_abs": (lambda: los.Absolute(par0), pm.Centered()),
        "huber_std": (lambda: los.Huber(par0, 0.5), pm.Standardized()),
        "docs5": (lambda: pen.Quadratic(par0), pm.Standardized()),
    }[key]
    X0 = torch.tensor(g[key + "/X0"], device="cuda")
    n, m = X0.shape
    return pm.MDE(n, m, torch.tensor(g[key + "/edges"], device="cuda"), f(), c), X0


@pytest.mark.parametrize("key", TRAJ)
def test_embed_follows_reference_trajectory(golden, key):
    import pymde_b200 as pm
    g = golden["trajectories"]
    mde, X0 = build(pm, key, g)
    X = mde.embed(X=X0, max_iter=int(g[key + "/max_iter"]), eps=float(g[key + "/eps"]))
    st = mde.solve_stats
    ref = g[key + "/average_distortions"]
    # iteration 0 is a plain evaluation at X0: per-evaluation parity, 1e-5 relative (north_star)
    np.testing.assert_allclose(st.average_distortions[0], ref[0], rtol=1e-5)
    np.testing.assert_allclose(st.residual_norms[0], g[key + "/residual_norms"][0], rtol=1e-4)
    # the first iterations track the reference within fp32 summation-order noise
    k = min(5, len(ref), st.iterations)
    np.testing.assert_allclose(st.average_distortions[:k], ref[:k], rtol=1e-3)
    np.testing.assert_allclose(st.step_size_percents[0], g[key + "/step_size_percents"][0], rtol=5e-3)
    final = mde.average_distortion(X).item()
    if key in ("quad_std", "docs5"):  # problems that converge: final value within 1e-5 relative
        np.testing.assert_allclose(final, g[key + "/final_value"], rtol=1e-5)
    else:  # non-converged after 40 iterations: within the reference's own run-to-run spread
        np.testing.assert_allclose(final, g[key + "/final_value"], rtol=1e-2)
    # value reported == loss at the start of the last iteration (SURVEY Appendix B.4)
    assert mde.value == st.average_distortions[-1]
    assert X.data_ptr() == mde.X.data_ptr()


@pytest.mark.parametrize("key", TRAJ)
def test_embed_matches_fp32_oracle(golden, key):
    """Same inputs through the numpy restatement in fp32: iteration counts and early losses agree."""
    import pymde_b200 as pm
    from tests.test_oracle_golden import _spec_for_traj
    g = golden["trajectories"]
    mde, X0 = build(pm, key, g)
    mde.embed(X=X0, max_iter=12, eps=float(g[key + "/eps"]))
    spec, cons = _spec_for_traj(key, g[key + "/par0"])
    _, st = O.embed(g[key + "/X0"], g[key + "/edges"], spec, cons, eps=float(g[key + "/eps"]), max_iter=12,
                    dtype=np.float32)
    k = min(4, st.iterations, mde.solve_stats.iterations)
    np.testing.assert_allclose(mde.solve_stats.average_distortions[:k], st.average_distortions[:k], rtol=1e-3)
    np.testing.assert_allclose(mde.solve_stats.residual_norms[:k], st.residual_norms[:k], rtol=2e-2, atol=1e-6)


def _knn_problem(pm, n, k, m, seed, constraint):
    from tests.lbfgs_replay import knn_graph
    edges, w = knn_graph(n, k, seed)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    return pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, constraint), edges, w


def test_embed_follows_fp32_oracle_over_30_iterations(golden):
    """docs5 for 30 iterations (eps = 1e-7) against the numpy restatement in fp32 on the same inputs: the first 10
    average distortions within 1e-4 relative, the final ones within 1e-2.  Iteration counts are not compared: whether
    the residual ever reaches eps is decided by rounding (the fp64 oracle converges at iteration 12, the fp32 one runs
    all 30)."""
    import pymde_b200 as pm
    from tests.test_oracle_golden import _spec_for_traj
    g = golden["trajectories"]
    mde, X0 = build(pm, "docs5", g)
    mde.embed(X=X0, max_iter=30, eps=1e-7)
    ours = list(mde.solve_stats.average_distortions)
    spec, cons = _spec_for_traj("docs5", g["docs5/par0"])
    _, st = O.embed(g["docs5/X0"], g["docs5/edges"], spec, cons, eps=1e-7, max_iter=30, dtype=np.float32)
    ref = list(st.average_distortions)
    k = min(10, len(ours), len(ref))
    np.testing.assert_allclose(ours[:k], ref[:k], rtol=1e-4)
    np.testing.assert_allclose(ours[-1], ref[-1], rtol=1e-2)


def test_solver_create_accepts_only_the_step_driver(golden):
    """opts.mode must be 2: the retired drivers 0 and 1 are unsupported, anything else is invalid."""
    import ctypes as C
    import pymde_b200 as pm
    from pymde_b200 import _lib, util
    g = golden["trajectories"]
    mde, _ = build(pm, "docs5", g)
    layout = mde._layout()
    lib = _lib.load()
    expected = {0: _lib.MDE_E_UNSUPPORTED, 1: _lib.MDE_E_UNSUPPORTED, 3: _lib.MDE_E_INVALID, -1: _lib.MDE_E_INVALID,
                2: 0}
    for mode, rc_expected in expected.items():
        opts = _lib.mde_solver_opts_t()
        opts.constraint = int(mde.constraint._solver_id)
        opts.memory_size, opts.max_iter, opts.world_size, opts.mode = 10, 4, 1, mode
        handle = C.c_void_p()
        rc = lib.mde_solver_create(C.byref(handle), layout.handle, int(mde.n_items), int(mde.embedding_dim),
                                   C.byref(opts), util.stream_ptr(layout.device))
        if handle:
            lib.mde_solver_destroy(handle)
        assert rc == rc_expected, (mode, rc)


@pytest.mark.parametrize("cname", ["centered", "standardized"])
def test_embed_invariants_medium(cname):
    import pymde_b200 as pm
    cons = pm.Centered() if cname == "centered" else pm.Standardized()
    n, m = 20000, 2
    mde, edges, w = _knn_problem(pm, n, 8, m, 1, cons)
    pm.seed(0)
    X = mde.embed(max_iter=60, eps=1e-6)
    st = mde.solve_stats
    assert st.iterations == 60 and len(st.residual_norms) == 60 and len(st.step_size_percents) == 60
    assert torch.isfinite(X).all()
    assert st.average_distortions[-1] < st.average_distortions[0]
    # line search accepts only decreasing losses (Armijo) -> monotone sequence
    assert all(b <= a + 1e-6 * abs(a) for a, b in zip(st.average_distortions, st.average_distortions[1:]))
    np.testing.assert_allclose(X.mean(0).cpu().numpy(), 0, atol=1e-5)
    if cname == "standardized":
        X64 = X.double()
        np.testing.assert_allclose((X64.T @ X64 / n).cpu().numpy(), np.eye(m), atol=1e-4)
    # final loss agrees with the oracle's evaluation of the returned embedding
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    v_ref, _ = O.average_distortion(X.cpu().double().numpy(), edges, spec, False)
    np.testing.assert_allclose(mde.average_distortion(X).item(), v_ref, rtol=1e-5)
    assert st.func_evals >= st.iterations


def test_converges_and_stops_early():
    import pymde_b200 as pm
    n = 200
    edges = pm.all_edges(n)
    mde = pm.MDE(n, 2, edges.cuda(), pm.penalties.Quadratic(torch.ones(edges.shape[0])), pm.Standardized())
    pm.seed(0)
    mde.embed(max_iter=500, eps=1e-4)
    assert mde.solve_stats.iterations < 500
    assert mde.residual_norm <= 1e-4
    # all-pairs unit-weight quadratic + standardized: every standardized X has the same value 2*m*n/(n-1)
    np.testing.assert_allclose(mde.average_distortion(mde.X).item(), 2.0 * 2 * n / (n - 1), rtol=1e-4)


def test_anchored_constraint_keeps_anchors():
    import pymde_b200 as pm
    rng = np.random.default_rng(3)
    n, m = 300, 2
    mde0, edges, w = _knn_problem(pm, n, 5, m, 2, pm.Centered())
    anchors = torch.tensor([0, 5, 17], device="cuda")
    values = torch.tensor(rng.standard_normal((3, m)).astype(np.float32), device="cuda")
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, pm.Anchored(anchors, values))
    pm.seed(0)
    X = mde.embed(max_iter=30)
    np.testing.assert_allclose(X[anchors].cpu().numpy(), values.cpu().numpy(), atol=0)
    assert mde.solve_stats.average_distortions[-1] < mde.solve_stats.average_distortions[0]


@pytest.mark.parametrize("key", ["quad", "pp"])
def test_anchored_follows_reference_trajectory(golden, key):
    """Anchored against fixtures generated by the unmodified reference (tests/golden/anchored.npz)."""
    import pymde_b200 as pm
    g = golden["anchored"]
    dev = "cuda"
    w = torch.tensor(g[key + "/par0"], device=dev)
    f = pm.penalties.Quadratic(w) if key == "quad" else pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log)
    anchors = torch.tensor(g["anchors"], device=dev)
    values = torch.tensor(g["values"], device=dev)
    n, m = g[key + "/X0"].shape
    mde = pm.MDE(n, m, torch.tensor(g[key + "/edges"], device=dev), f, pm.Anchored(anchors, values))
    X = mde.embed(X=torch.tensor(g[key + "/X0"], device=dev), max_iter=int(g[key + "/max_iter"]), eps=1e-6)
    st = mde.solve_stats
    ref = g[key + "/f32/average_distortions"]
    np.testing.assert_allclose(st.average_distortions[0], ref[0], rtol=1e-5)
    np.testing.assert_allclose(st.residual_norms[0], g[key + "/f32/residual_norms"][0], rtol=1e-4)
    k = min(5, len(ref), st.iterations)
    np.testing.assert_allclose(st.average_distortions[:k], ref[:k], rtol=1e-3)
    assert torch.equal(X[anchors], values)
    final = mde.average_distortion(X).item()
    if key == "quad":  # convex in the free rows: the reference (fp32 and fp64) and this solver meet at the optimum
        np.testing.assert_allclose(final, float(g["quad/f64/final_value"]), rtol=1e-5)
    else:
        np.testing.assert_allclose(final, float(g["pp/f32/final_value"]), rtol=1e-2)


def test_custom_constraint_and_callable_use_generic_solver():
    import pymde_b200 as pm

    class Sphere(pm.constraints.Constraint):
        def name(self):
            return "sphere"

        def initialization(self, n_items, embedding_dim, device=None):
            X = torch.randn((int(n_items), int(embedding_dim)), device="cuda")
            return X / X.norm(dim=1)[:, None]

        def project_onto_constraint(self, Z, inplace=True):
            return Z.div_(Z.norm(dim=1)[:, None]) if inplace else Z / Z.norm(dim=1)[:, None]

        def project_onto_tangent_space(self, X, Z, inplace=True):
            dual = (Z * X).sum(1)
            return Z.sub_(dual[:, None] * X) if inplace else Z - dual[:, None] * X

    n, m = 400, 3
    mde0, edges, w = _knn_problem(pm, n, 5, m, 4, pm.Centered())
    wt = torch.tensor(np.abs(w), device="cuda")
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), pm.penalties.Quadratic(wt), Sphere())
    pm.seed(0)
    X = mde.embed(max_iter=25)
    np.testing.assert_allclose(X.norm(dim=1).cpu().numpy(), 1.0, atol=1e-5)
    assert mde.solve_stats.average_distortions[-1] < mde.solve_stats.average_distortions[0]
    mde2 = pm.MDE(n, m, torch.tensor(edges, device="cuda"), lambda d: wt * d.pow(2), pm.Centered())
    mde2.embed(max_iter=10)
    assert mde2.solve_stats.average_distortions[-1] < mde2.solve_stats.average_distortions[0]


def test_solver_error_where_the_reference_raises():
    """All items on one point with a repulsive Log penalty: the loss is +inf at every trial step, the line
    search backs off 10 times and the reference raises SolverError (pymde/lbfgs.py:59-80)."""
    import pymde_b200 as pm
    n = 50
    edges = pm.all_edges(n).cuda()
    f = pm.penalties.Log(-torch.ones(edges.shape[0], device="cuda"))
    mde = pm.MDE(n, 2, edges, f, pm.Centered())
    with pytest.raises(pm.util.SolverError):
        mde.embed(X=torch.zeros(n, 2, device="cuda"), max_iter=5)


@pytest.mark.parametrize("m", [40, 128])
def test_wide_standardized_runs_on_the_device_solver(m):
    """Standardized with 32 < embedding_dim <= 256 runs on the device-resident solver (tiled Gram + Newton-Schulz
    retraction, csrc/mde_project_wide.cu): the constraint holds at the end, the loss decreases monotonically, and the
    first iterations agree with the host-stepped solver (cuSOLVER eigh retraction) on the same problem."""
    import pymde_b200 as pm
    n = 600 if m == 40 else 3000
    mde0, edges, w = _knn_problem(pm, n, 6, 2, 5, pm.Centered())
    f = pm.penalties.Quadratic(torch.tensor(np.abs(w), device="cuda"))
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, pm.Standardized())
    assert mde._fused_ok(mde.constraint, 10)
    pm.seed(0)
    X0 = mde.constraint.initialization(n, m)
    X = mde.embed(X=X0.clone(), max_iter=15)
    st = mde.solve_stats
    X64 = X.double()
    np.testing.assert_allclose((X64.T @ X64 / n).cpu().numpy(), np.eye(m), atol=2e-4)
    np.testing.assert_allclose(X.mean(0).cpu().numpy(), 0, atol=1e-5)
    d = st.average_distortions
    assert d[-1] < d[0] and all(b <= a + 1e-6 * abs(a) for a, b in zip(d, d[1:]))
    # first iterations against the oracle (fp64 SVD retraction, same L-BFGS / strong-Wolfe restatement)
    spec = O.FnSpec(O.P_QUADRATIC, np.abs(w).astype(np.float32), (0, 0, 0))
    _, ost = O.embed(X0.cpu().numpy(), edges, spec, O.Standardized(), max_iter=4, dtype=np.float32)
    np.testing.assert_allclose(d[:4], ost.average_distortions[:4], rtol=1e-3)


def test_verbose_and_snapshots_follow_the_reference_cadence(capsys):
    import pymde_b200 as pm
    mde, edges, w = _knn_problem(pm, 500, 5, 2, 6, pm.Centered())
    pm.seed(0)
    mde.embed(max_iter=20, snapshot_every=5, verbose=True, print_every=10)
    st = mde.solve_stats
    assert len(st.snapshots) == 4 and st.snapshots[0].device.type == "cpu"  # iterations 0,5,10,15 (optim.py:127-128)
    assert st.iterations == 20 and len(st.times) == 20


@pytest.mark.parametrize("m,cname", [(20, "centered"), (8, "standardized"), (5, "centered"), (33, "centered")])
def test_wide_embeddings_follow_the_oracle(m, cname):
    """Group-per-edge kernel + generic projections (m >= 5; Jacobi retraction for Standardized) inside the device
    solver, against the fp32 oracle trajectory on the same inputs."""
    import pymde_b200 as pm
    rng = np.random.default_rng(m)
    n = 150
    mde0, edges, w = _knn_problem(pm, n, 4, 2, 10 + m, pm.Centered())
    cons, ocons = (pm.Centered(), O.Centered()) if cname == "centered" else (pm.Standardized(), O.Standardized())
    X0 = rng.standard_normal((n, m)).astype(np.float32)
    X0 = ocons.project(X0).astype(np.float32)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, cons)
    mde.embed(X=torch.tensor(X0, device="cuda"), max_iter=8, eps=1e-7)
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    _, st = O.embed(X0, edges, spec, ocons, eps=1e-7, max_iter=8, dtype=np.float32)
    k = 4
    np.testing.assert_allclose(mde.solve_stats.average_distortions[:k], st.average_distortions[:k], rtol=2e-3)
    np.testing.assert_allclose(mde.solve_stats.residual_norms[0], st.residual_norms[0], rtol=1e-4)
    assert mde.solve_stats.average_distortions[-1] < mde.solve_stats.average_distortions[0]


def test_one_solver_serves_embeds_with_different_max_iter(golden):
    """max_iter only sizes statistics: the cached device solver (and its CUDA graphs) is reused, and a solve
    capped at k iterations is the prefix of a longer one (docs5 is evaluated without atomics races)."""
    import pymde_b200 as pm
    g = golden["trajectories"]
    mde, X0 = build(pm, "docs5", g)
    mde.embed(X=X0.clone(), max_iter=4, eps=0.0)
    s4 = mde.solve_stats
    solver = mde.__dict__["_device_solver"][1]
    mde.embed(X=X0.clone(), max_iter=9, eps=0.0)
    s9 = mde.solve_stats
    assert mde.__dict__["_device_solver"][1] is solver
    assert s4.iterations == 4 and s9.iterations == 9
    assert list(s9.average_distortions[:4]) == list(s4.average_distortions)
    assert list(s9.residual_norms[:4]) == list(s4.residual_norms)


def test_pause_and_resume_is_exact(golden):
    """run(3) + run(4) + run(5) == run(12): pausing at an iteration boundary does not perturb the solve."""
    import pymde_b200 as pm
    g = golden["trajectories"]
    res = []
    for chunks in ((12,), (3, 4, 5)):
        mde, X0 = build(pm, "docs5", g)
        solver = mde._solver(mde.constraint, 10, 64)
        solver.begin(X0, 0.0, 12)
        done = 0
        for c in chunks:
            done, conv = solver.run(c)
        assert done == 12
        avg, resid, pct, stp, fe = solver.stats(done)
        res.append((avg.copy(), resid.copy(), stp.copy(), fe, solver.x_view().clone()))
    np.testing.assert_array_equal(res[0][0], res[1][0])
    np.testing.assert_array_equal(res[0][1], res[1][1])
    np.testing.assert_array_equal(res[0][2], res[1][2])
    assert res[0][3] == res[1][3]
    assert torch.equal(res[0][4], res[1][4])
    # a further run() after the cap is a no-op
    d2, _ = solver.run(5)
    assert d2 == 12
