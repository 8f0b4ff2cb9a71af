"""GPU: distortion functions that are plain torch callables, solved on the device-resident L-BFGS solver
(pymde_b200/external.py, mde_solver_create_external) in its two modes -- the callable captured as a CUDA graph
inside the solver's step graphs, and the callable called back at every evaluation -- against the reference's own
embed() trajectories, the host-stepped solver and the autograd path."""
import numpy as np
import pytest
import torch

from tests.test_gpu_solver import TRAJ, _knn_problem

pytestmark = pytest.mark.gpu

MODES = ["graph", "hook"]


# the reference's penalties and losses (pymde/functions/penalties.py, losses.py) as plain torch callables, written
# with torch.where instead of boolean-mask assignment so that they can be captured
def _log1p(w, d):
    return w * torch.log1p(d.pow(1.5))


def _log(w, d):
    return w * torch.log(-torch.expm1(-d))


def torch_function(key, par0):
    if key in ("quad_std", "docs5"):
        return lambda d: par0 * d.pow(2)
    if key in ("pp_cen", "pp_std"):
        return lambda d: torch.where(par0 >= 0, _log1p(par0, d), _log(par0, d))
    if key == "cycle_abs":
        return lambda d: (par0 - d).abs()
    if key == "huber_std":
        def huber(d, t=0.5):
            diff = (par0 - d).abs()
            return torch.where(diff < t, diff.pow(2), t * (2 * diff - t))
        return huber
    raise KeyError(key)


def build(pm, key, g):
    par0 = torch.tensor(g[key + "/par0"], device="cuda")
    cons = pm.Centered() if key in ("pp_cen", "cycle_abs") else pm.Standardized()
    X0 = torch.tensor(g[key + "/X0"], device="cuda")
    n, m = X0.shape
    return pm.MDE(n, m, torch.tensor(g[key + "/edges"], device="cuda"), torch_function(key, par0), cons), X0


def solver_of(mde):
    cur = mde.__dict__["_device_solver"]
    return None if cur is None else cur[1]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("key", TRAJ)
def test_callable_follows_reference_trajectory(golden, key, mode, monkeypatch):
    """The assertions of test_embed_follows_reference_trajectory, with the function as a torch callable."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", mode)
    g = golden["trajectories"]
    mde, X0 = build(pm, key, g)
    X = mde.embed(X=X0, max_iter=int(g[key + "/max_iter"]), eps=float(g[key + "/eps"]))
    assert solver_of(mde).external_mode == mode
    st = mde.solve_stats
    ref = g[key + "/average_distortions"]
    np.testing.assert_allclose(st.average_distortions[0], ref[0], rtol=1e-5)
    np.testing.assert_allclose(st.residual_norms[0], g[key + "/residual_norms"][0], rtol=1e-4)
    k = min(5, len(ref), st.iterations)
    np.testing.assert_allclose(st.average_distortions[:k], ref[:k], rtol=1e-3)
    np.testing.assert_allclose(st.step_size_percents[0], g[key + "/step_size_percents"][0], rtol=5e-3)
    final = mde.average_distortion(X).item()
    rtol = 1e-5 if key in ("quad_std", "docs5") else 1e-2
    np.testing.assert_allclose(final, g[key + "/final_value"], rtol=rtol)
    assert mde.value == st.average_distortions[-1]


def _weights(w):
    return torch.tensor(np.abs(w), device="cuda")


def test_routing_graph_hook_and_generic(monkeypatch):
    import pymde_b200 as pm
    n, m = 400, 2
    _, edges, w = _knn_problem(pm, n, 5, m, 4, pm.Centered())
    E = torch.tensor(edges, device="cuda")
    wt = _weights(w)
    pos = torch.tensor(w, device="cuda") >= 0

    def run(f, cons=None):
        mde = pm.MDE(n, m, E, f, cons if cons is not None else pm.Centered())
        pm.seed(0)
        mde.embed(max_iter=10)
        st = mde.solve_stats
        assert st.average_distortions[-1] < st.average_distortions[0]
        return mde

    assert solver_of(run(lambda d: wt * d.pow(2))).external_mode == "graph"

    def masked(d):  # boolean-mask assignment, as the reference's own PushAndPull: synchronises with the host
        out = torch.empty_like(d)
        out[pos] = wt[pos] * torch.log1p(d[pos].pow(1.5))
        out[~pos] = -wt[~pos] * torch.log(-torch.expm1(-d[~pos]))
        return out

    assert solver_of(run(masked)).external_mode == "hook"
    noisy = run(lambda d: wt * d.pow(2) * (1.0 + 1e-3 * torch.rand_like(d)))
    assert solver_of(noisy).external_mode == "hook"
    # a table function reports no external mode
    table = run(pm.penalties.Quadratic(wt))
    assert solver_of(table).external_mode is None

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

    assert solver_of(run(lambda d: wt * d.pow(2), Sphere())) is None
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", "generic")
    assert solver_of(run(lambda d: wt * d.pow(2))) is None
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", "graph")
    with pytest.raises(ValueError):
        run(masked)


@pytest.mark.parametrize("m,cname", [(1, "centered"), (2, "anchored"), (3, "standardized"), (4, "centered"),
                                     (40, "standardized")])
def test_callable_runs_on_the_device_solver(m, cname):
    """Anchored, every narrow width and the wide Standardized retraction (m = 40) take callables on the device."""
    import pymde_b200 as pm
    n = 300
    _, edges, w = _knn_problem(pm, n, 6, 2, 7 + m, pm.Centered())
    wt = torch.tensor(w, device="cuda")
    f = lambda d: torch.where(wt >= 0, _log1p(wt, d), _log(wt, d))
    if cname == "anchored":
        anchors = torch.tensor([0, 5, 17], device="cuda")
        values = torch.tensor(np.random.default_rng(3).standard_normal((3, m)).astype(np.float32), device="cuda")
        cons = pm.Anchored(anchors, values)
    else:
        cons = pm.Centered() if cname == "centered" else pm.Standardized()
    if m == 40:
        wa = _weights(w)
        f = lambda d: wa * d.pow(2)
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, cons)
    pm.seed(0)
    X = mde.embed(max_iter=15)
    assert solver_of(mde).external_mode == "graph"
    d = mde.solve_stats.average_distortions
    assert d[-1] < d[0] and all(b <= a + 1e-6 * abs(a) for a, b in zip(d, d[1:]))
    if cname == "anchored":
        assert torch.equal(X[anchors], values)
    if cname == "standardized":
        X64 = X.double()
        np.testing.assert_allclose((X64.T @ X64 / n).cpu().numpy(), np.eye(m), atol=2e-4)


@pytest.mark.parametrize("mode", MODES)
def test_iteration_zero_matches_the_generic_solver_and_autograd(mode, monkeypatch):
    import pymde_b200 as pm
    n, m = 2000, 2
    _, edges, w = _knn_problem(pm, n, 8, m, 11, pm.Centered())
    wt = torch.tensor(w, device="cuda")
    f = lambda d: torch.where(wt >= 0, _log1p(wt, d), _log(wt, d))
    X0 = torch.tensor(np.random.default_rng(5).standard_normal((n, m)).astype(np.float32), device="cuda")
    X0 -= X0.mean(0)
    res = {}
    for arm in (mode, "generic"):
        monkeypatch.setenv("PYMDE_B200_EXTERNAL", arm)
        mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, pm.Centered())
        mde.embed(X=X0.clone(), max_iter=3)
        res[arm] = mde.solve_stats
    assert solver_of(mde) is None
    dev, gen = res[mode], res["generic"]
    np.testing.assert_allclose(dev.average_distortions[0], gen.average_distortions[0], rtol=1e-6)
    np.testing.assert_allclose(dev.residual_norms[0], gen.residual_norms[0], rtol=1e-5)
    # the autograd path (MDE.average_distortion through _ExternalAverageDistortion); Centered: no tangent projection
    X = X0.clone().requires_grad_(True)
    v = mde.average_distortion(X)
    v.backward()
    np.testing.assert_allclose(dev.average_distortions[0], v.item(), rtol=1e-6)
    np.testing.assert_allclose(dev.residual_norms[0], X.grad.norm().item(), rtol=1e-5)


def _sparse_problem(pm, f_of_w, seed=21):
    n, m = 3000, 2
    _, edges, w = _knn_problem(pm, n, 6, m, seed, pm.Centered())
    wt = torch.tensor(w, device="cuda")
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f_of_w(wt), pm.Centered())
    X0 = torch.tensor(np.random.default_rng(seed).standard_normal((n, m)).astype(np.float32), device="cuda")
    return mde, X0 - X0.mean(0), wt


def _pp(wt):
    return lambda d: torch.where(wt >= 0, _log1p(wt, d), _log(wt, d))


def test_reproducible_and_the_same_in_both_modes(monkeypatch):
    """Default layout of a sparse graph (owner-ordered scatter, no float atomics): two solves give the same bits,
    and the graph and hook modes compute the same bits."""
    import pymde_b200 as pm
    out = {}
    for mode in MODES:
        monkeypatch.setenv("PYMDE_B200_EXTERNAL", mode)
        mde, X0, _ = _sparse_problem(pm, _pp)
        runs = []
        for _ in range(2):
            X = mde.embed(X=X0.clone(), max_iter=25, eps=0.0).clone()
            st = mde.solve_stats
            runs.append((X, list(st.average_distortions), list(st.residual_norms), list(st.step_size_percents)))
        assert mde._layout().lib.mde_edges_kind(mde._layout().handle) == 0
        assert solver_of(mde).external_mode == mode
        assert torch.equal(runs[0][0], runs[1][0])
        assert runs[0][1:] == runs[1][1:]
        out[mode] = runs[0]
    assert torch.equal(out["graph"][0], out["hook"][0])
    assert out["graph"][1:] == out["hook"][1:]


@pytest.mark.parametrize("mode", MODES)
def test_in_place_change_of_the_weights_is_seen(mode, monkeypatch):
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", mode)
    mde, X0, wt = _sparse_problem(pm, _pp)
    mde.embed(X=X0.clone(), max_iter=8, eps=0.0)
    wt.mul_(2)
    X = mde.embed(X=X0.clone(), max_iter=8, eps=0.0).clone()
    fresh, _, _ = _sparse_problem(pm, lambda w: _pp(w * 2))
    Xf = fresh.embed(X=X0.clone(), max_iter=8, eps=0.0)
    assert torch.equal(X, Xf)
    assert list(mde.solve_stats.average_distortions) == list(fresh.solve_stats.average_distortions)


def test_rebound_closure_variable_is_seen_at_the_next_embed():
    import pymde_b200 as pm
    state = {}
    mde, X0, wt = _sparse_problem(pm, lambda w: (lambda d: state["w"] * d.pow(2)))
    state["w"] = wt.abs()
    mde.embed(X=X0.clone(), max_iter=3, eps=0.0)
    v1 = mde.solve_stats.average_distortions[0]
    state["w"] = 3 * wt.abs()
    mde.embed(X=X0.clone(), max_iter=3, eps=0.0)
    np.testing.assert_allclose(mde.solve_stats.average_distortions[0], 3 * v1, rtol=1e-6)


@pytest.mark.parametrize("mode", MODES)
def test_solver_error_where_the_reference_raises(mode, monkeypatch):
    """test_gpu_solver.py::test_solver_error_where_the_reference_raises with the Log penalty as a callable:
    +inf at coincident points, so every trial of the line search is non-finite."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", mode)
    n = 50
    edges = pm.all_edges(n).cuda()
    w = -torch.ones(edges.shape[0], device="cuda")
    mde = pm.MDE(n, 2, edges, lambda d: _log(w, d), pm.Centered())
    with pytest.raises(pm.util.SolverError):
        mde.embed(X=torch.zeros(n, 2, device="cuda"), max_iter=5)
    assert solver_of(mde).external_mode == mode


@pytest.mark.parametrize("mode", MODES)
def test_edges_of_length_zero_take_the_guard(mode, monkeypatch):
    """fpp / d is 0 / 0 on an edge of length 0; it is replaced by 1 (times a zero difference) as on the autograd
    path, so the solve stays finite."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", mode)
    n, m = 200, 2
    _, edges, w = _knn_problem(pm, n, 4, m, 13, pm.Centered())
    wt = _weights(w)
    X0 = torch.tensor(np.random.default_rng(13).standard_normal((n, m)).astype(np.float32), device="cuda")
    i, j = int(edges[0, 0]), int(edges[0, 1])
    X0[j] = X0[i]
    X0 -= X0.mean(0)
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), lambda d: wt * d.pow(2), pm.Centered())
    assert mde.distances(X0)[0].item() == 0.0
    mde.embed(X=X0.clone(), max_iter=5)
    st = mde.solve_stats
    assert np.isfinite(st.average_distortions).all() and np.isfinite(st.residual_norms).all()
    X = X0.clone().requires_grad_(True)
    v = mde.average_distortion(X)
    v.backward()
    assert torch.isfinite(X.grad).all()
    np.testing.assert_allclose(st.average_distortions[0], v.item(), rtol=1e-6)
    np.testing.assert_allclose(st.residual_norms[0], X.grad.norm().item(), rtol=1e-5)


def test_the_library_refuses_graphs_it_cannot_embed():
    """A graph with a node the solver cannot add as a child (an event record) is MDE_E_UNSUPPORTED."""
    import ctypes as C
    import pymde_b200 as pm
    from pymde_b200 import _lib, util
    n, m = 200, 2
    _, edges, w = _knn_problem(pm, n, 4, m, 17, pm.Centered())
    wt = _weights(w)
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), lambda d: wt * d.pow(2), pm.Centered())
    layout = mde._layout()
    p = layout.p
    d = torch.ones(p, device="cuda")
    fpp = torch.zeros(p, device="cuda")
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    ev = torch.cuda.Event(external=True)
    with torch.cuda.graph(graph):
        fpp.copy_(d * 2)
        ev.record()
        loss.copy_(d.sum(dtype=torch.float64).reshape(1))
    lib = _lib.load()
    opts = _lib.mde_solver_opts_t()
    opts.constraint, opts.memory_size, opts.max_iter, opts.mode, opts.world_size = 0, 10, 4, 2, 1
    x = _lib.mde_external_t()
    x.d, x.fpp, x.loss, x.graph = d.data_ptr(), fpp.data_ptr(), loss.data_ptr(), graph.raw_cuda_graph()
    handle = C.c_void_p()
    rc = lib.mde_solver_create_external(C.byref(handle), layout.handle, n, m, C.byref(opts), C.byref(x),
                                        util.stream_ptr(layout.device))
    assert rc == _lib.MDE_E_UNSUPPORTED and not handle
    x.graph = None  # neither a graph nor a hook
    assert lib.mde_solver_create_external(C.byref(handle), layout.handle, n, m, C.byref(opts), C.byref(x),
                                          util.stream_ptr(layout.device)) == _lib.MDE_E_INVALID
