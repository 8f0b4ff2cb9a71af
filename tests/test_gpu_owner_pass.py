"""The owner pass of the sorted-SoA layout (kind 0, m <= 4): each node's directed entries are evaluated in one place,
summed in registers in a fixed order and written once, with no atomics and no second kernel.

- Exact sums: with small-integer X and dyadic per-edge coefficients (mde_scatter_external), every contribution and
  every partial sum is exact in fp32, so the gradient must equal the fp64 sum bit for bit, whatever the order.  The
  graph has a hub of degree >= 5 000, isolated rows, coincident rows, duplicate edges and both edge classes.
- Reproducibility: fresh layouts give the same bits, and so do two embed() runs.
- The C2-shaped evaluation is one kernel launch on a kind-0 layout.
The check of the exact-sum comparison itself (dropping one incidence entry must fail it) runs without a GPU."""
import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

_ENV = ("MDE_B200_LAYOUT", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC")


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


def _exact_graph(seed, n=6000, hub_deg=5200):
    """(edges (p, 2) int64, coefficients (p,) dyadic float32, weights (p,) with both signs, X (n, m) small integers,
    isolated rows) for m = 4; callers take X[:, :m]."""
    rng = np.random.default_rng(seed)
    isolated = rng.choice(np.arange(10, n), 40, replace=False)
    active = np.setdiff1d(np.arange(n), isolated)
    hub = 3
    parts = [np.stack([np.full(hub_deg, hub), rng.choice(active[active != hub], hub_deg, replace=False)], 1)]
    parts.append(np.stack([rng.choice(active, 30000), rng.choice(active, 30000)], 1))
    e = np.concatenate(parts).astype(np.int64)
    e = e[e[:, 0] != e[:, 1]]
    e = np.concatenate([e, e[:500], e[1000:1200, ::-1]])  # duplicate edges, in both orientations
    X = rng.integers(-8, 9, (n, 4)).astype(np.float32)
    co = rng.choice(np.setdiff1d(active, [hub]), 20, replace=False).reshape(10, 2)
    X[co[:, 1]] = X[co[:, 0]]  # coincident rows, joined by an edge
    e = np.concatenate([e, co]).astype(np.int64)
    perm = rng.permutation(len(e))
    e = e[perm]
    g = (rng.integers(-16, 17, len(e)) / 8.0).astype(np.float32)
    w = np.where(rng.random(len(e)) < 0.5, 1.0, -1.0).astype(np.float32)
    return e, g, w, X, isolated


def _exact_expected(edges, g, X, n):
    """fp64: grad[i] += g_k (x_i - x_j) at i, and the negative at j, for every edge k = (i, j)."""
    Xd = X.astype(np.float64)
    v = g.astype(np.float64)[:, None] * (Xd[edges[:, 0]] - Xd[edges[:, 1]])
    out = np.zeros_like(Xd)
    np.add.at(out, edges[:, 0], v)
    np.add.at(out, edges[:, 1], -v)
    return out


def _kind(mde):
    from pymde_b200 import _lib
    return int(_lib.load().mde_edges_kind(mde._layout().handle))


@gpu
@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_external_scatter_is_exact(m):
    import pymde_b200 as pm
    n = 6000
    e, g, w, X4, isolated = _exact_graph(100 + m, n)
    X = np.ascontiguousarray(X4[:, :m])
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, m, torch.tensor(e, device="cuda"), f, pm.Centered())
    lay = mde._layout()
    assert _kind(mde) == 0
    deg = np.bincount(e.ravel(), minlength=n)
    assert deg.max() >= 5000 and np.all(deg[isolated] == 0)
    got = lay.scatter_external(torch.tensor(X, device="cuda"), torch.tensor(g, device="cuda")).cpu().numpy()
    want = _exact_expected(e, g, X, n)
    assert np.array_equal(got.astype(np.float64), want)
    assert not np.any(got[isolated])


def test_exact_check_fails_when_an_entry_is_dropped():
    """Leaving out one endpoint's entry of one edge (here: one of the hub's) changes the expected sums, and the
    comparison above sees it."""
    n = 6000
    e, g, w, X4, isolated = _exact_graph(102, n)
    X = X4[:, :2]
    want = _exact_expected(e, g, X, n)
    k = int(np.flatnonzero((e[:, 0] == 3) & (g != 0) & np.any(X[e[:, 0]] != X[e[:, 1]], axis=1))[0])
    Xd = X.astype(np.float64)
    dropped = want.copy()
    dropped[e[k, 1]] += g[k] * (Xd[e[k, 0]] - Xd[e[k, 1]])  # the dst-end entry of edge k left out
    assert not np.array_equal(dropped, want)


def _pushpull_problem(m, seed=20):
    rng = np.random.default_rng(seed + m)
    n, p = 5000, 90000
    e = rng.integers(0, n, (2 * p, 2))
    e = np.unique(np.sort(e[e[:, 0] != e[:, 1]], axis=1), axis=0)[:p]
    hub = np.stack([np.zeros(5000, np.int64), np.arange(1, 5001) % n], 1)
    e = np.unique(np.concatenate([e, hub[hub[:, 1] != 0]]), axis=0)
    w = rng.choice([1.0, 2.0, -1.0], len(e)).astype(np.float32)
    X0 = rng.standard_normal((n, m)).astype(np.float32)
    return n, e, w, X0 - X0.mean(0)


@gpu
@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_default_layout_is_bit_reproducible(m):
    """Default switches: value, gradient and 40 embed() iterations are the same bits from fresh layouts."""
    import pymde_b200 as pm
    from pymde_b200 import _lib
    dev = torch.device("cuda", 0)
    n, e, w, X0 = _pushpull_problem(m)

    def problem():
        f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
        return pm.MDE(n, m, torch.tensor(e, device=dev), f, pm.Centered(), device=dev)

    values, grads = [], []
    for _ in range(3):
        mde = problem()
        assert _kind(mde) == 0 and _lib.load().mde_edges_deterministic(mde._layout().handle) == 0
        X = torch.tensor(X0, device=dev, requires_grad=True)
        v = mde.average_distortion(X)
        v.backward()
        values.append(v.item())
        grads.append(X.grad.clone())
    assert values[0] == values[1] == values[2]
    assert torch.equal(grads[0], grads[1]) and torch.equal(grads[0], grads[2])
    runs = []
    for _ in range(2):
        mde = problem()
        Xe = mde.embed(X=torch.tensor(X0, device=dev), max_iter=40, eps=0.0).clone()
        st = mde.solve_stats
        runs.append((Xe, list(st.average_distortions), list(st.residual_norms), list(st.step_size_percents)))
    assert torch.equal(runs[0][0], runs[1][0])
    assert runs[0][1:] == runs[1][1:]


@gpu
def test_c2_evaluation_is_one_launch():
    """The C2 problem of bench.py builds the sorted-SoA layout, and its fused evaluation is one kernel."""
    import bench
    import pymde_b200 as pm
    from pymde_b200 import _lib, util
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    edges, w = bench.c2_edges(0)
    f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(bench.N_ITEMS, bench.EMBED_DIM, torch.tensor(edges, device=dev), f, pm.Centered(), device=dev)
    lay = mde._layout()
    assert _kind(mde) == 0
    X = torch.tensor(bench.initial_iterate(0), device=dev)
    grad = torch.zeros_like(X)
    c0 = lib.mde_launch_count()
    _lib.check(lib.mde_distortion(lay.handle, X.data_ptr(), X.shape[1], grad.data_ptr(), None, util.stream_ptr(dev)))
    assert lib.mde_launch_count() - c0 == 1
    torch.cuda.synchronize()
    v, g = lay.value_and_grad(X)
    assert torch.equal(g, grad) and torch.isfinite(v)
