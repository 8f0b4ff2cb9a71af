"""Deterministic mode's fixed-point gradient at m <= 4 (MDE_B200_DETERMINISTIC=1) against fp64.

The sorted-SoA layout runs distortion_quad_kernel twice: a scan for every row's largest finite |contribution| M_r,
then the accumulation of every contribution, at both of its ends, rounded at its row's 2^S_r, S_r = 61 - ceil(log2(deg_r)) - eM_r (M_r < 2^eM_r),
into int64 entries, then fx_apply_kernel (tests/det_fx.py emulates it; tests/test_det_fx_cpu.py derives the bound).  Every case here checks the
layout is deterministic and of kind 0, and that a second evaluation gives the same bits.

- External coefficients (MODE 2: callables, the LOBPCG Laplacian): the kernel's floats are reproducible on the host,
  so the gradient must equal the emulation bit for bit, and lie within the derived bound of the fp64 scatter.
- Fused functions (MODE 0): within the bound of an fp64 scatter of fp64 contributions (the function's own fp32 error
  enters as a relative term), and no more than twice the default owner kernel's Frobenius error, from 6e4 to 5e7
  edges, at a random and a near-converged X.
- Range: terms and row sums beyond 2^23 (the old 2^40 accumulator's limit), the guard's g = 1 on differences of 1e7,
  far coordinates: correct to the bound.
- Non-finite X rows and coefficients end like the default mode: the same non-finite entries, the same solver outcome.
- A C2-shaped solve agrees with the default mode and is bit-reproducible."""
import math

import numpy as np
import pytest
import torch

from tests import det_fx as D

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = D.U
_ENV = ("MDE_B200_LAYOUT", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC", "PYMDE_B200_EXTERNAL", "PYMDE_B200_SPECTRAL")
# the function's own relative error on a contribution g (x_s - x_d): the MUFU forms of the recipe default (m = 2, 3
# fused), and IEEE math (rsqrt / sqrt / division rounded once each, a few roundings in all)
KAPPA = {"mufu": 2.0 ** -16, "ieee": 2.0 ** -19}


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


def _lib():
    from pymde_b200 import _lib
    return _lib.load()


def _check_det(handle):
    assert int(_lib().mde_edges_deterministic(handle)) == 1
    assert int(_lib().mde_edges_kind(handle)) == 0


def _ext_layout(edges, n, m):
    from pymde_b200 import _lib as L_
    from pymde_b200.problem import EdgeLayout
    table = L_.mde_fn_t()
    table.fn_att = table.fn_rep = 100  # external coefficients: the layout carries the index structure only
    e = torch.as_tensor(edges, device=DEV)
    return EdgeLayout(e, n, table, torch.zeros(len(edges), device=DEV), None, DEV, embedding_dim=m)


def _scatter(lay, X, g):
    """external-coefficient gradient of a deterministic layout, evaluated twice (the same bits)"""
    _check_det(lay.handle)
    Xt, gt = torch.as_tensor(X, device=DEV), torch.as_tensor(g, device=DEV)
    a = lay.scatter_external(Xt, gt)
    b = lay.scatter_external(Xt, gt)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    return a.cpu().numpy()


def _emulated_and_bound(X, edges, g):
    """(emulated gradient, fp64 gradient, bound) of external coefficients g"""
    n = len(X)
    order, src, dst = D.sort_edges(edges)
    v = D.external_contributions(X, src, dst, np.asarray(g, np.float32)[order])
    rows, vals = D.terms(src, dst, v)
    S = D.scale_exponent(src, dst, v, D.lg_degree(src, dst, n))
    F, nan = D.accumulate(n, rows, vals, S)
    want = D.finish(F, nan, S)
    G, A = D.exact_scatter(X, edges, g)
    deg = np.bincount(np.asarray(edges).ravel(), minlength=n)
    return want, G, D.bound(n, rows, A, deg, 2 * U + U * U, S, want)


def _random_edges(n, p, seed):
    rng = np.random.default_rng(seed)
    i = rng.integers(0, n, p)
    return np.stack([i, (i + rng.integers(1, n, p)) % n], 1).astype(np.int64)


# --------------------------------------------------------------------------------------- external coefficients
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("p", [60_000, 1_550_000])
def test_external_scatter_is_the_emulation(m, p, monkeypatch):
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    n = max(2700, p // 22)
    rng = np.random.default_rng(m + p)
    edges = _random_edges(n, p, m)
    hub = np.stack([np.full(5000, 7), rng.integers(8, n, 5000)], 1)  # one row of degree > 5 000
    edges = np.concatenate([edges, hub, edges[:100]])
    X = rng.standard_normal((n, m)).astype(np.float32)
    g = (rng.standard_normal(len(edges)) * 10.0 ** rng.uniform(-6, 2, len(edges)) / len(edges)).astype(np.float32)
    got = _scatter(_ext_layout(edges, n, m), X, g)
    want, G, B = _emulated_and_bound(X, edges, g)
    assert np.all(np.abs(got - G) <= B)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("k", [-100, -40, 40, 90])
def test_external_scatter_far_from_unit_scale(k, monkeypatch):
    """Coefficients scaled by 2^k: at k = -100 the scale 2^S is beyond the float range (S > 149), at k = 90 the
    contributions reach 1e27 -- the same bits as the emulation, the gradient scaled by 2^k."""
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    n, m = 5000, 2
    rng = np.random.default_rng(k + 200)
    edges = _random_edges(n, 80_000, 3)
    X = rng.standard_normal((n, m)).astype(np.float32)
    g = (rng.uniform(0.5, 2.0, len(edges)) * 2.0 ** k).astype(np.float32)
    got = _scatter(_ext_layout(edges, n, m), X, g)
    want, G, B = _emulated_and_bound(X, edges, g)
    assert np.all(np.abs(got - G) <= B)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert np.abs(got).max() > 2.0 ** (k - 2)


@pytest.mark.parametrize("kb", [3, 4])
def test_lobpcg_laplacian_operator(kb, monkeypatch):
    """The spectral initialisation's L V at kb = 3, 4 columns with weights over 1e-3 .. 1e7."""
    from pymde_b200 import quadratic
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    n = 20_000
    rng = np.random.default_rng(kb)
    edges = _random_edges(n, 300_000, kb)
    w = (10.0 ** rng.uniform(-3, 7, len(edges))).astype(np.float32)
    V = rng.standard_normal((n, kb)).astype(np.float32)
    op = quadratic._LaplacianOperator(n, kb, torch.tensor(edges, device=DEV), torch.tensor(w, device=DEV), DEV)
    _check_det(op.layout.handle)
    a = op(torch.tensor(V, device=DEV))
    b = op(torch.tensor(V, device=DEV))
    assert torch.equal(a, b)
    got = a.cpu().numpy()
    want, G, B = _emulated_and_bound(V, edges, w)
    assert np.all(np.abs(got - G) <= B)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    LV = quadratic._laplacian(n, edges, w.astype(np.float64)) @ V.astype(np.float64)  # the host operator
    np.testing.assert_allclose(LV, G, rtol=0, atol=1e-12 * np.abs(G).max())


# --------------------------------------------------------------------------------------- fused functions
def _reference(X, e, fn, par64, p, kappa):
    """fp64 scatter of fp64 contributions: (G, the function's error budget per entry, sum |v*| per entry, every row's
    largest |v*| plus its error).  A loss's f' = 2 (d - delta) cancels near delta, so the error of the fp32 d (m + 3
    roundings) enters it absolutely."""
    Xd = X.double()
    m = Xd.shape[1]
    diff = Xd[e[:, 0]] - Xd[e[:, 1]]
    d = diff.norm(dim=1)
    extra = torch.zeros_like(d)
    if fn == "pushpull":
        fp = torch.where(par64 >= 0, par64 * 1.5 * d.sqrt() / (1 + d.pow(1.5)), par64 / torch.expm1(d))
    else:
        fp = 2.0 * (d - par64)
        extra = 2.0 * (m + 3) * U * torch.ones_like(d) / p
    g = fp / (p * d)
    g = torch.where(torch.isfinite(g), g, torch.ones_like(g))
    v = g[:, None] * diff
    av = v.abs()
    err = kappa * av + extra[:, None] * diff.abs()
    G = torch.zeros_like(Xd).index_add_(0, e[:, 0], v).index_add_(0, e[:, 1], -v)
    A = torch.zeros_like(Xd).index_add_(0, e[:, 0], av).index_add_(0, e[:, 1], av)
    Er = torch.zeros_like(Xd).index_add_(0, e[:, 0], err).index_add_(0, e[:, 1], err)
    top = (av + err).max(dim=1).values
    Mr = torch.zeros(len(Xd), dtype=torch.float64, device=Xd.device)
    Mr = Mr.scatter_reduce(0, e[:, 0], top, "amax").scatter_reduce(0, e[:, 1], top, "amax")
    return G, Er, A, Mr


def _problem(fn, n, p, m, seed):
    """(edges, function, degree, X -> _reference of the problem)"""
    import pymde_b200 as pm
    edges = _random_edges(n, p, seed)
    rng = np.random.default_rng(seed)
    if fn == "pushpull":
        w = np.where(rng.random(p) < 0.5, 1.0, -1.0).astype(np.float32)
        par = torch.tensor(w, device=DEV)
        f = pm.penalties.PushAndPull(par, pm.penalties.Log1p, pm.penalties.Log)
    else:
        par = torch.tensor(rng.uniform(0.5, 2.0, p).astype(np.float32), device=DEV)
        f = pm.losses.Quadratic(par)
    e = torch.tensor(edges, device=DEV)
    deg = torch.bincount(e.reshape(-1), minlength=n).double()
    return edges, f, deg, lambda X, kappa: _reference(X, e, fn, par.double(), p, kappa)


def _bound(Er, A, deg, Mr, result):
    """det_fx.bound with the function's error budget Er in place of 2 u + u^2, and every row's scale taken from an
    upper bound Mr of its M_r (the kernel's M_r is at most the row's largest |v*| plus its error)"""
    lg = torch.ceil(torch.log2(deg.clamp(min=1)))
    em = torch.floor(torch.log2(Mr.clamp(min=2.0 ** -1000))) + 1
    half_quantum = torch.where(Mr > 0, torch.exp2(lg + em - D.HEADROOM - 1), torch.zeros_like(Mr))
    return (Er + (deg * half_quantum)[:, None] + (U + 2.0 ** -52) * result.abs()
            + (deg[:, None] + 2) * 2.0 ** -52 * A)


def _fused(mde, X):
    lay = mde._layout()
    v, g = lay.value_and_grad(X)
    return v, g, lay


SIZES = [(2_700, 60_000), (70_000, 1_550_000), (450_000, 10_000_000), (2_200_000, 50_000_000)]


@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("size", SIZES, ids=["6e4", "1.55e6", "1e7", "5e7"])
@pytest.mark.parametrize("fn", ["pushpull", "quadratic_precise"])
def test_resolution_against_fp64(fn, size, m, monkeypatch):
    import pymde_b200 as pm
    n, p = size
    if fn == "quadratic_precise":
        monkeypatch.setenv("MDE_B200_KERNEL", "precise")
    kappa = KAPPA["mufu" if fn == "pushpull" else "ieee"]
    edges, f, deg, reference = _problem(fn, n, p, m, seed=m + n)
    E = torch.tensor(edges, device=DEV)
    default = pm.MDE(n, m, E, f, pm.Centered(), device=DEV)
    default._layout()  # layouts are built on first use, under the environment of that moment
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    det = pm.MDE(n, m, E, f, pm.Centered(), device=DEV)
    _check_det(det._layout().handle)
    monkeypatch.delenv("MDE_B200_DETERMINISTIC")
    gen = torch.Generator(device=DEV).manual_seed(m)
    X0 = torch.randn(n, m, device=DEV, generator=gen)
    X0 -= X0.mean(0)
    Xc = default.embed(X=X0.clone(), max_iter=60 if p > 10 ** 7 else 150).detach()
    for name, X in (("random", X0), ("converged", Xc)):
        _, g_def, _ = _fused(default, X)
        _, g1, lay = _fused(det, X)
        _, g2, _ = _fused(det, X)
        torch.cuda.synchronize()
        assert torch.equal(g1.view(torch.int32), g2.view(torch.int32)), name
        G, Er, A, Mr = reference(X, kappa)
        B = _bound(Er, A, deg, Mr, g1.double())
        err = (g1.double() - G).abs()
        bad = int((err > B).sum())
        assert bad == 0, (name, bad, float((err / B).max()))
        e_det = float((g1.double() - G).norm() / G.norm())
        e_def = float((g_def.double() - G).norm() / G.norm())
        assert e_det <= 2.0 * e_def, (name, e_det, e_def)
        del G, Er, A, B, err
    del default, det
    torch.cuda.empty_cache()


@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_callable_function_runs_mode_2(m, monkeypatch):
    """A Python-callable distortion function: its coefficients come from torch, the scatter is the deterministic
    external one, within the bound of an fp64 scatter of the same coefficients."""
    import pymde_b200 as pm
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    n, p = 70_000, 1_550_000
    edges = _random_edges(n, p, 40 + m)
    w = torch.ones(p, device=DEV)
    f = pm.penalties.Sigmoid(w, threshold=1.0)
    mde = pm.MDE(n, m, torch.tensor(edges, device=DEV), f, pm.Centered(), device=DEV)
    _check_det(mde._layout().handle)
    X = torch.randn(n, m, device=DEV, generator=torch.Generator(device=DEV).manual_seed(m))
    grads = []
    for _ in range(2):
        Xg = X.clone().requires_grad_(True)
        mde.average_distortion(Xg).backward()
        grads.append(Xg.grad.clone())
    assert torch.equal(grads[0], grads[1])
    # the coefficients the callable produced, g = f'(d) / (p d), in fp64; torch's fp32 g carries a few ulps (kappa)
    E = torch.tensor(edges, device=DEV)
    Xd = X.double()
    diff = Xd[E[:, 0]] - Xd[E[:, 1]]
    d = diff.norm(dim=1)
    s = torch.sigmoid(d - 1.0)
    v = (s * (1 - s) / (p * d))[:, None] * diff
    av = v.abs()
    G = torch.zeros_like(Xd).index_add_(0, E[:, 0], v).index_add_(0, E[:, 1], -v)
    A = torch.zeros_like(Xd).index_add_(0, E[:, 0], av).index_add_(0, E[:, 1], av)
    deg = torch.bincount(E.reshape(-1), minlength=n).double()
    kappa = 2.0 ** -18
    top = av.max(dim=1).values * (1 + kappa)
    Mr = torch.zeros(n, dtype=torch.float64, device=DEV)
    Mr = Mr.scatter_reduce(0, E[:, 0], top, "amax").scatter_reduce(0, E[:, 1], top, "amax")
    B = _bound(kappa * A, A, deg, Mr, grads[0].double())
    err = (grads[0].double() - G).abs()
    assert bool((err <= B).all()), float((err / B).max())


# --------------------------------------------------------------------------------------- range
def _star(vals, m=1):
    """nodes 0..k-1 joined to the hub k, x_j = 0, x_k = 1: the hub's terms are the coefficients themselves"""
    k = len(vals)
    edges = np.stack([np.arange(k), np.full(k, k)], 1).astype(np.int64)
    X = np.zeros((k + 1, m), np.float32)
    X[k] = 1.0
    return edges, X, np.asarray(vals, np.float32)


@pytest.mark.parametrize("kind", ["single_above", "single_below", "sum_above", "sum_below", "hub_crosses"])
@pytest.mark.parametrize("m", [1, 4])
def test_range_beyond_2_to_23(kind, m, monkeypatch):
    """A term and a row sum at 2^23 (1 +- 2^-10), a hub whose sum crosses 2^23 with every term below it (the 2^40
    accumulator clamped or wrapped the first, third and fifth into wrong finite numbers)."""
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    t = 2.0 ** 23
    vals = {"single_above": [t * (1 + 2 ** -10)], "single_below": [t * (1 - 2 ** -10)],
            "sum_above": [t * (1 + 2 ** -10) / 4] * 4, "sum_below": [t * (1 - 2 ** -10) / 4] * 4,
            "hub_crosses": [t / 3] * 7}[kind]
    edges, X, g = _star(vals, m)
    got = _scatter(_ext_layout(edges, len(X), m), X, g)
    want, G, B = _emulated_and_bound(X, edges, g)
    assert np.all(np.abs(got - G) <= B), (got[-1], G[-1])
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("m", [1, 2])
def test_guard_g_one_on_differences_of_1e7(m, monkeypatch):
    """Power(delta = d, exponent 0.5) at d = 1e7: f' is infinite, the guard sets g = 1 and the contribution is the
    difference vector itself, 1e7; five of them meet at the hub, 5e7 in all."""
    import pymde_b200 as pm
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    k = 5
    edges = np.stack([np.full(k, k), np.arange(k)], 1).astype(np.int64)
    X = np.zeros((k + 1, m), np.float32)
    X[:k, 0] = 1e7
    f = pm.losses.Power(torch.full((k,), 1e7, device=DEV), 0.5)
    mde = pm.MDE(k + 1, m, torch.tensor(edges, device=DEV), f, pm.Centered(), device=DEV)
    _check_det(mde._layout().handle)
    _, g1, _ = _fused(mde, torch.tensor(X, device=DEV))
    _, g2, _ = _fused(mde, torch.tensor(X, device=DEV))
    assert torch.equal(g1, g2)
    want = np.zeros((k + 1, m))
    want[k, 0] = -k * 1e7
    want[:k, 0] = 1e7
    assert np.array_equal(g1.cpu().numpy().astype(np.float64), want)


def test_preserve_distances_far_from_the_origin(monkeypatch):
    """preserve_distances at m = 2 on points with coordinates around 1e6, a Quadratic loss, evaluated at an
    embedding of the same scale: contributions 2 (d - delta) / p, within the bound of fp64."""
    import pymde_b200 as pm
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    monkeypatch.setenv("MDE_B200_KERNEL", "precise")
    rng = np.random.default_rng(5)
    n, m = 600, 2
    data = (1e6 + 3e5 * rng.standard_normal((n, 5))).astype(np.float32)
    mde = pm.preserve_distances(torch.tensor(data, device=DEV), embedding_dim=m, loss=pm.losses.Quadratic)
    _check_det(mde._layout().handle)
    X = (1e6 + 4e5 * rng.standard_normal((n, m))).astype(np.float32)
    _, g1, _ = _fused(mde, torch.tensor(X, device=DEV))
    _, g2, _ = _fused(mde, torch.tensor(X, device=DEV))
    assert torch.equal(g1, g2)
    e = mde.edges
    deg = torch.bincount(e.reshape(-1), minlength=n).double()
    delta = mde.distortion_function.deviations.to(DEV).double()
    G, Er, A, Mr = _reference(torch.tensor(X, device=DEV), e, "quadratic", delta, len(e), KAPPA["ieee"])
    err = (g1.double() - G).abs()
    assert bool((err <= _bound(Er, A, deg, Mr, g1.double())).all())
    assert float(G.abs().max()) > 1.0


# --------------------------------------------------------------------------------------- non-finite input
def _both_modes(monkeypatch, build):
    outs = []
    for det in (False, True):
        if det:
            monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
        else:
            monkeypatch.delenv("MDE_B200_DETERMINISTIC", raising=False)
        outs.append(build(det))
    monkeypatch.delenv("MDE_B200_DETERMINISTIC", raising=False)
    return outs


@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("fn", ["pushpull", "quadratic_precise"])
@pytest.mark.parametrize("m", [2, 3])
def test_non_finite_rows_of_x(bad, fn, m, monkeypatch):
    import pymde_b200 as pm
    if fn == "quadratic_precise":
        monkeypatch.setenv("MDE_B200_KERNEL", "precise")
    n = 3000
    edges, f, _, _ = _problem(fn, n, 40_000, m, seed=9)
    X = torch.randn(n, m, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    X[17] = float(bad)

    def run(det):
        mde = pm.MDE(n, m, torch.tensor(edges, device=DEV), f, pm.Centered(), device=DEV)
        if det:
            _check_det(mde._layout().handle)
        _, g, _ = _fused(mde, X)
        return g.cpu().numpy()

    g_def, g_det = _both_modes(monkeypatch, run)
    assert np.array_equal(np.isfinite(g_def), np.isfinite(g_det))
    ok = np.isfinite(g_def)
    np.testing.assert_allclose(g_det[ok], g_def[ok], rtol=1e-4, atol=1e-4 * np.abs(g_def[ok]).max())


@pytest.mark.parametrize("bad", ["nan", "inf", "-inf"])
def test_non_finite_coefficients_through_the_c_entry(bad, monkeypatch):
    """mde_scatter_external takes the coefficients as given (the Python guard is bypassed)"""
    from pymde_b200 import util
    n, m = 3000, 2
    edges = _random_edges(n, 40_000, 2)
    rng = np.random.default_rng(2)
    X = torch.tensor(rng.standard_normal((n, m)).astype(np.float32), device=DEV)
    g = torch.tensor(rng.standard_normal(len(edges)).astype(np.float32) / len(edges), device=DEV)
    g[[5, 900]] = float(bad)

    def run(det):
        lay = _ext_layout(edges, n, m)
        if det:
            _check_det(lay.handle)
        out = torch.zeros_like(X)
        rc = _lib().mde_scatter_external(lay.handle, X.data_ptr(), m, g.data_ptr(), out.data_ptr(),
                                         util.stream_ptr(X.device))
        assert rc == 0
        torch.cuda.synchronize()
        return out.cpu().numpy()

    g_def, g_det = _both_modes(monkeypatch, run)
    assert not np.isfinite(g_det).all()
    assert np.array_equal(np.isfinite(g_def), np.isfinite(g_det))


@pytest.mark.parametrize("bad", ["nan", "inf"])
def test_solver_outcome_with_a_non_finite_row(bad, monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import _lib as L_, util
    n, m = 3000, 2
    edges, f, _, _ = _problem("pushpull", n, 40_000, m, seed=11)

    def run(det):
        mde = pm.MDE(n, m, torch.tensor(edges, device=DEV), f, pm.Centered(), device=DEV)
        X0 = torch.randn(n, m, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
        X0[5] = float(bad)
        try:
            X = mde.embed(X=X0, max_iter=20)
        except (util.SolverError, L_.MdeError) as exc:
            return type(exc).__name__
        return "finite" if bool(torch.isfinite(X).all()) else "non-finite"

    out_def, out_det = _both_modes(monkeypatch, run)
    assert out_def == out_det


# --------------------------------------------------------------------------------------- solve
def test_c2_shaped_solve(monkeypatch):
    """The C2 shape (n = 70 000, 1.55e6 edges: neighbour-like attractive pairs and as many random repulsive ones),
    PushAndPull(Log1p, Log), Centered, 200 iterations: both solves finish, they follow the same trajectory at first
    (the first 8 average distortions agree to 1e-5), they end at comparable distortions (L-BFGS trajectories whose
    gradients differ in the last bits take different line-search steps after that; 0.14 % apart after 200
    iterations on an H100), and the deterministic solve is the same bits twice."""
    import pymde_b200 as pm
    from tests import lbfgs_replay as L
    n, m = 70_000, 2
    edges, w = L.knn_graph(n, 12, 70)
    assert 1.4e6 < len(edges) < 1.7e6
    E = torch.tensor(edges, device=DEV)
    f = pm.penalties.PushAndPull(torch.tensor(w, device=DEV), pm.penalties.Log1p, pm.penalties.Log)
    X0 = torch.randn(n, m, device=DEV, generator=torch.Generator(device=DEV).manual_seed(70))

    def solve(det):
        mde = pm.MDE(n, m, E, f, pm.Centered(), device=DEV)
        if det:
            _check_det(mde._layout().handle)
        X = mde.embed(X=X0.clone(), max_iter=200, eps=1e-12)
        return X, list(mde.solve_stats.average_distortions), mde.solve_stats.iterations

    (X_def, h_def, it_def), (X_det, h_det, it_det) = _both_modes(monkeypatch, solve)
    assert it_def == 200 and it_det == 200
    rel = abs(h_det[-1] - h_def[-1]) / abs(h_def[-1])
    print("final average distortion: default %.9g, deterministic %.9g, relative difference %.3g"
          % (h_def[-1], h_det[-1], rel))
    np.testing.assert_allclose(h_det[:8], h_def[:8], rtol=1e-5)
    assert h_det[-1] < h_det[0] and rel <= 0.02
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    X2, h2, _ = solve(True)
    assert torch.equal(X_det.view(torch.int32), X2.view(torch.int32)) and h_det == h2
