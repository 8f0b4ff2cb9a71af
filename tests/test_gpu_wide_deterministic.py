"""Deterministic mode at 5 <= m <= 512 (MDE_B200_DETERMINISTIC=1): the sorted-SoA layout keeps the directed entries
grouped by owner, and fused and external-coefficient evaluations at the layout's m run the wide owner kernel, which
sums every row in registers in list order and writes it once, with no atomics.  Lists longer than 256 entries are
evaluated in segments whose partial rows are added in segment order.

- The switch is honoured at every m of the range, and without it nothing changes (one launch, as before).
- Exact sums: small-integer X and dyadic coefficients make every contribution and partial sum exact in fp32, so the
  gradient must equal the fp64 sum bit for bit; the graph has a segmented hub, lists of exactly 256 and 257 entries,
  isolated rows, coincident rows and duplicate edges in both orientations.
- Both ends of an edge compute the same d, f and g: on a matching grad[i] == -grad[j] bit for bit.
- Parity with the oracle, and bit-identical values, gradients, solves and recipes from fresh layouts."""
import numpy as np
import pytest
import torch

from oracle import c_oracle, mde_oracle as O
from tests import lbfgs_replay as L
from tests.test_gpu_owner_pass import _exact_expected, _exact_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"

_ENV = ("MDE_B200_LAYOUT", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC", "PYMDE_B200_EXTERNAL", "PYMDE_B200_SPECTRAL")
SEG = 256  # entries per segment of a long list (kWideSeg)


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")


def _lib():
    from pymde_b200 import _lib
    return _lib.load()


def _is_det(mde):
    return int(_lib().mde_edges_deterministic(mde._layout().handle))


def _pushpull(n, m, edges, w, constraint=None):
    import pymde_b200 as pm
    f = pm.penalties.PushAndPull(torch.tensor(w, device=DEV), pm.penalties.Log1p, pm.penalties.Log)
    return pm.MDE(n, m, torch.tensor(edges, device=DEV), f, constraint or pm.Centered(), device=DEV)


def _fused(mde, X):
    """(value, gradient) of one fused evaluation, and the kernel launches of the evaluation itself (without the sum
    of the loss partials)."""
    from pymde_b200 import _lib as L_, util
    lib = _lib()
    lay = mde._layout()
    grad = torch.zeros_like(X)
    c0 = lib.mde_launch_count()
    L_.check(lib.mde_distortion(lay.handle, X.data_ptr(), X.shape[1], grad.data_ptr(), None, util.stream_ptr(X.device)))
    launches = int(lib.mde_launch_count() - c0)
    v, g = lay.value_and_grad(X)
    torch.cuda.synchronize()
    if _is_det(mde):  # the push kernel's float reds land in any order
        assert torch.equal(g, grad)
    return v.item(), g, launches


def _small_graph(n=3000, seed=0):
    edges, w = L.knn_graph(n, 6, seed)
    return edges, w


# --------------------------------------------------------------------------------------- the switch
@pytest.mark.parametrize("m", [5, 8, 128, 512])
def test_switch_is_honoured(m, monkeypatch):
    n = 3000
    edges, w = _small_graph(n)
    assert np.bincount(edges.ravel(), minlength=n).max() <= SEG  # no segments: one launch
    X = torch.randn(n, m, device=DEV)
    plain = _pushpull(n, m, edges, w)
    assert _is_det(plain) == 0
    v0, g0, launches = _fused(plain, X)
    assert launches == 1
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    d = _pushpull(n, m, edges, w)
    assert _is_det(d) == 1
    assert int(_lib().mde_edges_kind(d._layout().handle)) == 0
    v1, g1, launches = _fused(d, X)
    assert launches == 1
    np.testing.assert_allclose(v1, v0, rtol=1e-5)
    scale = float(g0.abs().max())
    assert float((g1 - g0).abs().max()) <= 3e-5 * scale
    # the directed entries are counted in the layout's size
    assert int(_lib().mde_edges_nbytes(d._layout().handle)) > int(_lib().mde_edges_nbytes(plain._layout().handle))


def test_segmented_hub_takes_one_more_launch(det):
    n = 3000
    edges, w = _small_graph(n)
    hub = np.stack([np.zeros(1000, np.int64), np.arange(1, 1001)], 1)
    edges = np.concatenate([edges, hub])
    w = np.concatenate([w, np.ones(1000, np.float32)])
    mde = _pushpull(n, 16, edges, w)
    assert _is_det(mde) == 1
    _, _, launches = _fused(mde, torch.randn(n, 16, device=DEV))
    assert launches == 2


# --------------------------------------------------------------------------------------- exact sums
def _wide_exact_graph(m, n=6000, seed=300):
    """_exact_graph (hub of degree >= 5 000, isolated rows, coincident rows, duplicates in both orientations) plus a
    hub of 1 200 further entries and two nodes with exactly 256 and 257 entries; X (n, m) small integers."""
    e, g, w, X4, isolated = _exact_graph(seed, n)
    rng = np.random.default_rng(seed + m)
    active = np.setdiff1d(np.arange(n), np.concatenate([isolated, [3]]))
    deg = np.bincount(e.ravel(), minlength=n)
    h1, h256, h257 = rng.choice(active[deg[active] < 200], 3, replace=False)
    others = np.setdiff1d(active, [h1, h256, h257])
    extra = [np.stack([np.full(1200, h1), rng.choice(others, 1200)], 1)]
    for node, target in ((h256, SEG), (h257, SEG + 1)):
        k = target - int(deg[node])
        extra.append(np.stack([rng.choice(others, k), np.full(k, node)], 1))
    extra = np.concatenate(extra).astype(np.int64)
    e = np.concatenate([e, extra])
    g = np.concatenate([g, (rng.integers(-16, 17, len(extra)) / 8.0).astype(np.float32)])
    w = np.concatenate([w, np.where(rng.random(len(extra)) < 0.5, 1.0, -1.0).astype(np.float32)])
    X = rng.integers(-8, 9, (n, m)).astype(np.float32)
    same = np.all(X4[e[:, 0]] == X4[e[:, 1]], axis=1)  # the coincident pairs of _exact_graph
    for i, j in e[same]:
        X[j] = X[i]
    deg = np.bincount(e.ravel(), minlength=n)
    assert deg[3] >= 5000 and deg[h1] > 4 * SEG and deg[h256] == SEG and deg[h257] == SEG + 1
    assert np.all(deg[isolated] == 0) and np.sum(np.all(X[e[:, 0]] == X[e[:, 1]], axis=1)) >= 10
    return e, g, w, X, isolated


@pytest.mark.parametrize("m", [5, 7, 8, 13, 16, 32, 33, 64, 128, 200, 256, 512])
def test_external_scatter_is_exact(m, det):
    n = 6000
    e, g, w, X, isolated = _wide_exact_graph(m, n)
    mde = _pushpull(n, m, e, w)
    assert _is_det(mde) == 1
    got = mde._layout().scatter_external(torch.tensor(X, device=DEV), torch.tensor(g, device=DEV)).cpu().numpy()
    want = _exact_expected(e, g, X, n)
    assert np.array_equal(got.astype(np.float64), want)
    assert not np.any(got[isolated])


# --------------------------------------------------------------------------------------- both ends agree
def _matching(n_pairs, m, seed):
    rng = np.random.default_rng(seed)
    nodes = rng.permutation(2 * n_pairs)
    e = nodes.reshape(n_pairs, 2).astype(np.int64)
    X = rng.standard_normal((2 * n_pairs, m)).astype(np.float32)
    X[e[:8, 1]] = X[e[:8, 0]]  # zero distance
    X[e[8:16, 1]] = X[e[8:16, 0]] + 1e-4 * rng.standard_normal((8, m)).astype(np.float32)
    return e, X


@pytest.mark.parametrize("m", [5, 16, 33, 128, 512])
@pytest.mark.parametrize("fn", ["pushpull", "huber"])
def test_both_ends_agree(m, fn, det):
    import pymde_b200 as pm
    n_pairs = 4000
    e, X = _matching(n_pairs, m, 7 + m)
    rng = np.random.default_rng(m)
    if fn == "pushpull":
        w = torch.tensor(np.where(rng.random(n_pairs) < 0.5, 1.0, -1.0).astype(np.float32), device=DEV)
        f = pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log)
    else:
        f = pm.penalties.Huber(torch.tensor(rng.uniform(0.5, 2.0, n_pairs).astype(np.float32), device=DEV), 0.8)
    mde = pm.MDE(2 * n_pairs, m, torch.tensor(e, device=DEV), f, pm.Centered(), device=DEV)
    assert _is_det(mde) == 1
    _, G, _ = _fused(mde, torch.tensor(X, device=DEV))
    G = G.cpu()
    assert torch.equal(G[e[:, 0]], -G[e[:, 1]])
    assert torch.isfinite(G).all()


# --------------------------------------------------------------------------------------- parity
def _parity_problem(m, seed=11):
    rng = np.random.default_rng(seed + m)
    n = 4000
    edges, w = L.knn_graph(n, 8, seed + m)
    hub = np.stack([np.full(700, 5), rng.choice(np.arange(6, n), 700, replace=False)], 1)
    edges = np.concatenate([edges, hub]).astype(np.int64)
    w = np.concatenate([w, np.ones(700, np.float32)])
    X = rng.standard_normal((n, m)).astype(np.float32)
    X[edges[:20, 1]] = X[edges[:20, 0]]  # distance exactly zero
    X[edges[20:40, 1]] = X[edges[20:40, 0]] + 1e-3 * rng.standard_normal((20, m)).astype(np.float32)  # near zero
    return n, edges, w, X, rng


def _check(mde, X, edges, spec):
    Xg = torch.tensor(X, device=DEV, requires_grad=True)
    v = mde.average_distortion(Xg)
    v.backward()
    rv, rg = O.average_distortion(X.astype(np.float64), edges, spec, True)
    np.testing.assert_allclose(v.item(), rv, rtol=1e-5, atol=1e-6)
    scale = max(1.0, float(np.abs(rg).max()))
    np.testing.assert_allclose(Xg.grad.cpu().numpy(), rg, rtol=3e-5, atol=3e-5 * scale)
    v2 = mde.average_distortion(Xg.detach())  # value only: the wide kernel
    np.testing.assert_allclose(v2.item(), v.item(), rtol=1e-6)


@pytest.mark.parametrize("m", [5, 16, 128])
@pytest.mark.parametrize("fn", ["pushpull", "huber_penalty", "absolute", "weighted_quadratic"])
def test_parity_with_oracle(m, fn, det):
    import pymde_b200 as pm
    n, edges, w, X, rng = _parity_problem(m)
    p = len(edges)
    E = torch.tensor(edges, device=DEV)
    if fn == "pushpull":
        f = pm.penalties.PushAndPull(torch.tensor(w, device=DEV), pm.penalties.Log1p, pm.penalties.Log)
        spec = L.push_pull_spec(w)
    elif fn == "huber_penalty":
        a = rng.uniform(0.5, 2.0, p).astype(np.float32)
        f = pm.penalties.Huber(torch.tensor(a, device=DEV), 0.7)
        spec = O.FnSpec(O.P_HUBER, a, (0.7, 0, 0))
    elif fn == "absolute":
        dev = rng.uniform(0.5, 3.0, p).astype(np.float32)
        f = pm.losses.Absolute(torch.tensor(dev, device=DEV))
        spec = O.FnSpec(O.L_ABSOLUTE, dev)
    else:
        dev = rng.uniform(0.5, 3.0, p).astype(np.float32)
        wt = rng.uniform(0.2, 2.0, p).astype(np.float32)
        f = pm.losses.WeightedQuadratic(torch.tensor(dev, device=DEV), torch.tensor(wt, device=DEV))
        spec = O.FnSpec(O.L_WEIGHTED_QUADRATIC, dev, par1=wt)
    mde = pm.MDE(n, m, E, f, pm.Centered(), device=DEV)
    assert _is_det(mde) == 1
    _check(mde, X, edges, spec)


def test_c4_slice_parity(det):
    """The C4 slice of test_gpu_configs (n = 200 000, m = 128, 3e6 edges) against the C oracle."""
    import pymde_b200 as pm
    n, m = 200_000, 128
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    i = torch.arange(n, device=DEV).repeat_interleave(8)
    j = (i + torch.randint(1, 1000, (i.numel(),), device=DEV, generator=gen)) % n
    rep = torch.randint(0, n, (i.numel(), 2), device=DEV, generator=gen)
    rep = rep[rep[:, 0] != rep[:, 1]]
    e = torch.cat([torch.stack([i, j], 1), rep])
    w = torch.cat([torch.ones(i.numel(), device=DEV), -torch.ones(rep.shape[0], device=DEV)])
    mde = pm.MDE(n, m, e, pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log), pm.Centered(), device=DEV)
    assert _is_det(mde) == 1
    X = torch.randn(n, m, device=DEV, generator=gen)
    X -= X.mean(0)
    Xg = X.clone().requires_grad_(True)
    v = mde.average_distortion(Xg)
    v.backward()
    spec = O.FnSpec(O.P_LOG1P, w.cpu().numpy(), (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    v_ref, g_ref = c_oracle.average_distortion(X.cpu().numpy(), e.cpu().numpy(), spec, True)
    np.testing.assert_allclose(v.item(), v_ref, rtol=1e-5)
    err = np.abs(Xg.grad.cpu().numpy().astype(np.float64) - g_ref).max()
    assert err <= 3e-5 * np.abs(g_ref).max(), (err, np.abs(g_ref).max())
    v2 = mde.average_distortion(Xg.detach())
    g2 = Xg.grad.clone()
    Xg.grad = None
    mde.average_distortion(Xg).backward()
    assert v2.item() == pytest.approx(v.item(), rel=1e-6) and torch.equal(Xg.grad, g2)


# --------------------------------------------------------------------------------------- reproducibility
def _repro_graph(n, seed=3):
    edges, w = L.knn_graph(n, 8, seed)
    hub = np.stack([np.zeros(1500, np.int64), np.arange(1, 1501)], 1)  # six segments
    return np.concatenate([edges, hub]), np.concatenate([w, -np.ones(1500, np.float32)])


@pytest.mark.parametrize("m", [5, 16, 128])
def test_value_and_gradient_are_bit_identical(m, det):
    n = 5000
    edges, w = _repro_graph(n)
    X = torch.randn(n, m, device=DEV, generator=torch.Generator(device=DEV).manual_seed(m))
    runs = []
    for _ in range(3):
        mde = _pushpull(n, m, edges, w)
        assert _is_det(mde) == 1
        v, g, _ = _fused(mde, X)
        runs.append((v, g))
    assert runs[0][0] == runs[1][0] == runs[2][0]
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][1], runs[2][1])


def _constraint(name, n, m):
    import pymde_b200 as pm
    if name == "centered":
        return pm.Centered()
    if name == "standardized":
        return pm.Standardized()
    anchors = np.arange(0, n, n // 7)[:7]
    values = np.random.default_rng(5).standard_normal((len(anchors), m)).astype(np.float32)
    return pm.Anchored(torch.tensor(anchors, device=DEV), torch.tensor(values, device=DEV))


@pytest.mark.parametrize("cname,m", [("centered", 8), ("standardized", 40), ("anchored", 6)])
def test_embed_is_bit_identical(cname, m, det):
    n = 5000
    edges, w = _repro_graph(n)
    runs = []
    for _ in range(3):
        cons = _constraint(cname, n, m)
        mde = _pushpull(n, m, edges, w, cons)
        assert _is_det(mde) == 1
        X0 = cons.project_onto_constraint(
            torch.randn(n, m, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4)), inplace=True)
        Xe = mde.embed(X=X0, max_iter=40, eps=0.0).clone()
        st = mde.solve_stats
        runs.append((Xe, list(st.average_distortions), list(st.residual_norms), list(st.step_size_percents)))
    for r in runs[1:]:
        assert torch.equal(runs[0][0], r[0])
        assert runs[0][1:] == r[1:]


def test_callable_function_is_bit_identical(det, monkeypatch):
    """A torch callable on the device solver's graph mode: distances and the scatter run on the layout."""
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", "graph")
    n, m = 5000, 16
    edges, w = _repro_graph(n)
    wt = torch.tensor(np.abs(w), device=DEV)
    runs = []
    for _ in range(3):
        mde = pm.MDE(n, m, torch.tensor(edges, device=DEV), lambda d: wt * d.pow(2), pm.Standardized(), device=DEV)
        assert _is_det(mde) == 1
        pm.seed(0)
        Xe = mde.embed(max_iter=25).clone()
        cur = mde.__dict__["_device_solver"]
        assert cur is not None and cur[1].external_mode == "graph"
        st = mde.solve_stats
        runs.append((Xe, list(st.average_distortions), list(st.residual_norms)))
    for r in runs[1:]:
        assert torch.equal(runs[0][0], r[0])
        assert runs[0][1:] == r[1:]


def test_paused_solve_matches_one_run(det):
    n, m, iters = 5000, 8, 30
    edges, w = _repro_graph(n)
    X0 = torch.tensor(L.initial_point(n, m, O.Centered(), 3), device=DEV)

    def solve(step):
        mde = _pushpull(n, m, edges, w)
        assert _is_det(mde) == 1
        solver = mde._solver(mde.constraint, 10, iters + 1)
        solver.begin(X0, 0.0, iters + 1)
        done = 0
        while done < iters:
            done, _ = solver.run(step)
        assert done == iters
        return solver.x_view().cpu().numpy(), [np.asarray(s) for s in solver.stats(iters)]

    X1, s1 = solve(1)
    Xa, sa = solve(iters)
    assert np.array_equal(X1, Xa)
    for a, b in zip(s1, sa):
        assert np.array_equal(a, b)


# --------------------------------------------------------------------------------------- recipes
def _blobs(n, d, seed):
    rng = np.random.default_rng(seed)
    centres = 4.0 * rng.standard_normal((6, d))
    lab = rng.integers(0, 6, n)
    return torch.tensor((centres[lab] + rng.standard_normal((n, d))).astype(np.float32))


@pytest.mark.parametrize("m", [3, 8])
def test_preserve_neighbors_is_reproducible(m, det):
    """n = 5 000 > 2 000: the spectral initialisation runs the device LOBPCG, whose operator is the external scatter
    on a layout built for m + 2 >= 5 columns."""
    import pymde_b200 as pm
    Y = _blobs(5000, 20, 1)
    out = []
    for _ in range(2):
        pm.seed(0)
        mde = pm.preserve_neighbors(Y, embedding_dim=m, verbose=False)
        assert _is_det(mde) == 1
        X_init = mde._X_init.clone()
        E = mde.embed(max_iter=60).clone()
        out.append((X_init, E, list(mde.solve_stats.average_distortions)))
    assert torch.equal(out[0][0], out[1][0])
    assert torch.equal(out[0][1], out[1][1])
    assert out[0][2] == out[1][2]
