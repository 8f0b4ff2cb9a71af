"""GPU: user-defined constraints (Constraint subclasses) on the device-resident L-BFGS solver
(PYMDE_B200_CONSTRAINT=device|graph|hook, pymde_b200/external.py ConstraintPart, mde_solver_create_custom): the
projections captured into the solver's step graphs or called back at every step, on staging buffers.  Built-in
constraints written as user classes against the built-ins, the reference's own _Sphere against its embed()
trajectory (tests/golden/custom_constraints.npz), inert surplus steps, routing and errors."""
import numpy as np
import pytest
import torch

from tests.test_gpu_solver import _knn_problem

pytestmark = pytest.mark.gpu

MODES = ["graph", "hook"]


def _constraint_base():
    import pymde_b200 as pm
    return pm.constraints.Constraint


class UserAnchored(_constraint_base()):
    """pymde's Anchored written as a user class (with index_copy_ / index_fill_, which capture)."""

    def __init__(self, anchors, values):
        self.anchors, self.values = anchors, values

    def name(self):
        return "user-anchored"

    def initialization(self, n_items, embedding_dim, device=None):
        X = torch.randn((int(n_items), int(embedding_dim)), device="cuda")
        return X.index_copy_(0, self.anchors, self.values)

    def project_onto_constraint(self, Z, inplace=True):
        out = Z if inplace else Z.clone()
        return out.index_copy_(0, self.anchors, self.values)

    def project_onto_tangent_space(self, X, Z, inplace=True):
        out = Z if inplace else Z.clone()
        return out.index_fill_(0, self.anchors, 0.0)


class UserCentered(_constraint_base()):
    def name(self):
        return "user-centered"

    def initialization(self, n_items, embedding_dim, device=None):
        X = torch.randn((int(n_items), int(embedding_dim)), device="cuda")
        return X - X.mean(0)

    def project_onto_constraint(self, Z, inplace=True):
        return Z.sub_(Z.mean(0)) if inplace else Z - Z.mean(0)

    def project_onto_tangent_space(self, X, Z, inplace=True):
        return Z


class Sphere(_constraint_base()):
    """The reference's _Sphere (pymde/constraints.py:203-231); `radius` may be a float or a CUDA tensor."""

    def __init__(self, radius=1.0):
        self.radius = radius

    def name(self):
        return "sphere"

    def initialization(self, n_items, embedding_dim, device=None):
        X = torch.randn((int(n_items), int(embedding_dim)), device="cuda")
        return self.radius * (X / X.norm(dim=1)[:, None])

    def project_onto_tangent_space(self, X, Z, inplace=True):
        dual = (Z * X).sum(1)
        offset = (1.0 / self.radius) * dual[:, None] * X
        return Z.sub_(offset) if inplace else Z - offset

    def project_onto_constraint(self, Z, inplace=True):
        if inplace:
            Z.div_(Z.norm(dim=1)[:, None])
            return Z.mul_(self.radius)
        return self.radius * Z / Z.norm(dim=1)[:, None]


def solver_of(mde):
    cur = mde.__dict__["_device_solver"]
    return None if cur is None else cur[1]


def _stats(mde):
    st = mde.solve_stats
    return (list(st.average_distortions), list(st.residual_norms), list(st.step_size_percents),
            list(st.step_lengths), st.func_evals)


def _sphere_problem(pm, g, cons):
    w = torch.tensor(g["sphere/par0"], device="cuda")
    f = pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log)
    X0 = torch.tensor(g["sphere/X0"], device="cuda")
    n, m = X0.shape
    return pm.MDE(n, m, torch.tensor(g["sphere/edges"], device="cuda"), f, cons), X0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("key", ["quad", "pp"])
def test_user_anchored_is_bit_identical_to_the_builtin(golden, key, mode, monkeypatch):
    """Both write the same values into the same rows, and the default layout is reproducible: the solves agree bit
    for bit.  The user class also follows the reference (anchored.npz) as test_gpu_solver's anchored test does."""
    import pymde_b200 as pm
    g = golden["anchored"]
    w = torch.tensor(g[key + "/par0"], device="cuda")
    f = pm.penalties.Quadratic(w) if key == "quad" else pm.penalties.PushAndPull(w, pm.penalties.Log1p,
                                                                                 pm.penalties.Log)
    anchors = torch.tensor(g["anchors"], device="cuda")
    values = torch.tensor(g["values"], device="cuda")
    X0 = torch.tensor(g[key + "/X0"], device="cuda")
    n, m = X0.shape
    E = torch.tensor(g[key + "/edges"], device="cuda")
    iters = int(g[key + "/max_iter"])
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", mode)
    out = {}
    for arm, cons in (("builtin", pm.Anchored(anchors, values)), ("user", UserAnchored(anchors, values))):
        mde = pm.MDE(n, m, E, f, cons)
        X = mde.embed(X=X0.clone(), max_iter=iters, eps=1e-6).clone()
        out[arm] = (X, _stats(mde))
        assert mde._layout().lib.mde_edges_kind(mde._layout().handle) == 0
        assert solver_of(mde).constraint_mode == (None if arm == "builtin" else mode)
    assert torch.equal(out["builtin"][0], out["user"][0])
    assert out["builtin"][1] == out["user"][1]
    X, (avg, res, _, _, _) = out["user"]
    ref = g[key + "/f32/average_distortions"]
    np.testing.assert_allclose(avg[0], ref[0], rtol=1e-5)
    np.testing.assert_allclose(res[0], g[key + "/f32/residual_norms"][0], rtol=1e-4)
    k = min(5, len(ref), len(avg))
    np.testing.assert_allclose(avg[:k], ref[:k], rtol=1e-3)
    assert torch.equal(X[anchors], values)
    final = mde.average_distortion(X).item()
    if key == "quad":
        np.testing.assert_allclose(final, float(g["quad/f64/final_value"]), rtol=1e-5)
    else:
        np.testing.assert_allclose(final, float(g["pp/f32/final_value"]), rtol=1e-2)


@pytest.mark.parametrize("m", [1, 3, 4])
def test_user_anchored_is_bit_identical_at_other_widths(m, monkeypatch):
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "device")
    n = 500
    _, edges, w = _knn_problem(pm, n, 6, m, 40 + m, pm.Centered())
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    rng = np.random.default_rng(m)
    anchors = torch.tensor(np.sort(rng.choice(n, 20, replace=False)), device="cuda")
    values = torch.tensor(rng.standard_normal((20, m)).astype(np.float32), device="cuda")
    X0 = torch.tensor(rng.standard_normal((n, m)).astype(np.float32), device="cuda")
    X0[anchors] = values
    out = []
    for cons in (pm.Anchored(anchors, values), UserAnchored(anchors, values)):
        mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, cons)
        out.append((mde.embed(X=X0.clone(), max_iter=30, eps=0.0).clone(), _stats(mde)))
    assert solver_of(mde).constraint_mode == "graph"
    assert torch.equal(out[0][0], out[1][0])
    assert out[0][1] == out[1][1]


@pytest.mark.parametrize("m", [1, 2, 3, 4, 8])
def test_user_centered_follows_the_builtin(m, monkeypatch):
    """Only the order of the column-mean summation differs from the built-in retraction."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "device")
    n = 600
    _, edges, w = _knn_problem(pm, n, 6, m, 60 + m, pm.Centered())
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    X0 = torch.tensor(np.random.default_rng(m).standard_normal((n, m)).astype(np.float32), device="cuda")
    X0 -= X0.mean(0)
    res = {}
    for arm, cons in (("builtin", pm.Centered()), ("user", UserCentered())):
        mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, cons)
        X = mde.embed(X=X0.clone(), max_iter=12, eps=0.0).clone()
        res[arm] = (X, mde.solve_stats)
    assert solver_of(mde).constraint_mode == "graph"
    b, u = res["builtin"][1], res["user"][1]
    np.testing.assert_allclose(u.average_distortions[0], b.average_distortions[0], rtol=1e-6)
    np.testing.assert_allclose(u.residual_norms[0], b.residual_norms[0], rtol=1e-6)
    np.testing.assert_allclose(u.average_distortions[:5], b.average_distortions[:5], rtol=1e-4)
    np.testing.assert_allclose(res["user"][0].mean(0).cpu().numpy(), 0, atol=1e-5)


@pytest.mark.parametrize("mode", MODES)
def test_sphere_follows_reference_trajectory(golden, mode, monkeypatch):
    """The reference's _Sphere(1.0) (custom_constraints.npz).  The final value lies in the band of the reference's
    runs with 1 and 4 threads, widened by 1e-2 relative (the objective is not convex; the fp32 trajectories part
    after the first iterations, as test_gpu_solver's non-convex trajectories)."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", mode)
    g = golden["custom_constraints"]
    mde, X0 = _sphere_problem(pm, g, Sphere(1.0))
    X = mde.embed(X=X0, max_iter=int(g["sphere/max_iter"]), eps=1e-5)
    assert solver_of(mde).constraint_mode == mode
    st = mde.solve_stats
    ref = g["sphere/average_distortions"]
    np.testing.assert_allclose(st.average_distortions[0], ref[0], rtol=1e-5)
    np.testing.assert_allclose(st.residual_norms[0], g["sphere/residual_norms"][0], rtol=1e-5)
    k = min(5, len(ref), st.iterations)
    np.testing.assert_allclose(st.average_distortions[:k], ref[:k], rtol=1e-3)
    np.testing.assert_allclose(st.step_size_percents[0], g["sphere/step_size_percents"][0], rtol=5e-3)
    np.testing.assert_allclose(X.norm(dim=1).cpu().numpy(), 1.0, atol=1e-5)
    finals = [float(g["sphere/final_value"]), float(g["sphere/t4/final_value"])]
    lo, hi = min(finals), max(finals)
    final = mde.average_distortion(X).item()
    assert lo - 1e-2 * abs(lo) <= final <= hi + 1e-2 * abs(hi), (final, finals)


@pytest.mark.parametrize("mode", MODES)
def test_surplus_steps_are_inert(golden, mode, monkeypatch):
    """The user's projections run in every step, also after the device paused; they work on staging buffers only, so
    solves stepped one iteration at a time (verbose, snapshots) and repeated solves on the cached solver give the
    bits of a plain embed()."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", mode)
    g = golden["custom_constraints"]
    mde, X0 = _sphere_problem(pm, g, Sphere(1.0))
    runs = []
    for kw in ({}, {"verbose": True, "print_every": 1}, {"snapshot_every": 5}, {}):
        X = mde.embed(X=X0.clone(), max_iter=25, eps=0.0, **kw).clone()
        runs.append((X, _stats(mde)))
    assert solver_of(mde).constraint_mode == mode
    assert len(mde.solve_stats.snapshots) == 0 and runs[0][1][0]
    for X, st in runs[1:]:
        assert torch.equal(X, runs[0][0])
        assert st == runs[0][1]


def test_routing(monkeypatch):
    import pymde_b200 as pm
    n, m = 400, 3
    _, edges, w = _knn_problem(pm, n, 5, m, 4, pm.Centered())
    E = torch.tensor(edges, device="cuda")
    wt = torch.tensor(np.abs(w), device="cuda")
    pos = torch.tensor(w, device="cuda") >= 0

    def run(cons, f=None):
        mde = pm.MDE(n, m, E, f if f is not None else pm.penalties.Quadratic(wt), cons)
        pm.seed(0)
        mde.embed(max_iter=10)
        st = mde.solve_stats
        assert st.average_distortions[-1] < st.average_distortions[0]
        return mde

    monkeypatch.delenv("PYMDE_B200_CONSTRAINT", raising=False)
    assert solver_of(run(Sphere())) is None                      # unset: the host-stepped solver
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "generic")
    assert solver_of(run(Sphere())) is None
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "device")
    mde = run(Sphere())
    assert solver_of(mde).constraint_mode == "graph" and solver_of(mde).external_mode is None
    np.testing.assert_allclose(mde.X.norm(dim=1).cpu().numpy(), 1.0, atol=1e-5)
    assert solver_of(run(pm.Centered())).constraint_mode is None  # built-ins route as before

    class Syncing(Sphere):  # .item() synchronises with the host
        def project_onto_constraint(self, Z, inplace=True):
            if Z.norm().item() == 0.0:
                raise ValueError("zero iterate")
            return super(Syncing, self).project_onto_constraint(Z, inplace)

    class Eigh(Sphere):  # torch.linalg.eigh on CUDA checks its status on the host
        def project_onto_tangent_space(self, X, Z, inplace=True):
            torch.linalg.eigh(X.T @ X)
            return super(Eigh, self).project_onto_tangent_space(X, Z, inplace)

    class Noisy(Sphere):  # draws random numbers
        def project_onto_constraint(self, Z, inplace=True):
            Z.add_(1e-7 * torch.randn_like(Z))
            return super(Noisy, self).project_onto_constraint(Z, inplace)

    class Event(Sphere):  # captures into an event-record node, which the library refuses
        def project_onto_constraint(self, Z, inplace=True):
            torch.cuda.Event(external=True).record()
            return super(Event, self).project_onto_constraint(Z, inplace)

    for cls in (Syncing, Eigh, Noisy, Event):
        assert solver_of(run(cls())).constraint_mode == "hook", cls.__name__

    # a callable distortion function with a custom constraint: both parts as graphs, or one of them as a hook
    smooth = lambda d: wt * d.pow(2)

    def masked(d):  # boolean-mask indexing synchronises with the host
        out = torch.empty_like(d)
        out[pos] = wt[pos] * d[pos].pow(2)
        out[~pos] = wt[~pos] * d[~pos].pow(2)
        return out

    for f, cons, modes in ((smooth, Sphere(), ("graph", "graph")), (masked, Sphere(), ("hook", "graph")),
                           (smooth, Syncing(), ("graph", "hook"))):
        s = solver_of(run(cons, f))
        assert (s.external_mode, s.constraint_mode) == modes

    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "graph")
    with pytest.raises(ValueError):
        run(Syncing())
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "hook")
    assert solver_of(run(Sphere())).constraint_mode == "hook"


class Boom(Exception):
    pass


def test_exception_in_a_hooked_constraint_is_raised_from_embed(monkeypatch):
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "hook")

    class Failing(Sphere):
        def project_onto_tangent_space(self, X, Z, inplace=True):
            raise Boom("tangent")

    n, m = 300, 3
    mde, _, _ = _knn_problem(pm, n, 5, m, 8, Failing())
    with pytest.raises(Boom):
        mde.embed(max_iter=5)
    assert solver_of(mde).constraint_mode == "hook"


@pytest.mark.parametrize("mode", MODES)
def test_non_finite_projection_raises_solver_error(mode, monkeypatch):
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", mode)

    class NaN(Sphere):
        def project_onto_constraint(self, Z, inplace=True):
            return Z.mul_(float("nan"))

    n, m = 300, 3
    mde, _, _ = _knn_problem(pm, n, 5, m, 9, NaN())
    X0 = torch.tensor(np.random.default_rng(9).standard_normal((n, m)).astype(np.float32), device="cuda")
    with pytest.raises(pm.util.SolverError):
        mde.embed(X=X0, max_iter=5)
    assert solver_of(mde).constraint_mode == mode


@pytest.mark.parametrize("mode", MODES)
def test_in_place_change_of_a_tensor_the_constraint_reads_is_seen(golden, mode, monkeypatch):
    """The radius is a device tensor: changed in place, it is seen by the next evaluation without a new capture."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", mode)
    g = golden["custom_constraints"]
    radius = torch.tensor(1.0, device="cuda")
    mde, X0 = _sphere_problem(pm, g, Sphere(radius))
    X = mde.embed(X=X0.clone(), max_iter=5, eps=0.0)
    np.testing.assert_allclose(X.norm(dim=1).cpu().numpy(), 1.0, atol=1e-5)
    radius.fill_(2.0)
    solver = solver_of(mde)
    assert solver.constraint_mode == mode
    solver.begin(2.0 * X0, 0.0, 5)  # the installed part, no new capture
    solver.run(5)
    np.testing.assert_allclose(solver.x_view().norm(dim=1).cpu().numpy(), 2.0, rtol=1e-5)
    X = mde.embed(X=2.0 * X0, max_iter=5, eps=0.0)
    np.testing.assert_allclose(X.norm(dim=1).cpu().numpy(), 2.0, rtol=1e-5)
