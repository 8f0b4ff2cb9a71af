"""The device spectral initialisation (quadratic.spectral_device) against fp64: its Laplacian operator on every edge
layout and width, its block LOBPCG against shift-invert Lanczos, the dispatch between device and host, and
laplacian_embedding against the closed-form optimum of its quadratic problem.

Operator tolerance, per entry i and column c: |(L V)_ic - op(V)_ic| <= (deg_i + 2) 2^-24 sum_j w_ij (|v_ic| + |v_jc|)
(+ deg_i 2^-40 in the fixed-point mode).  deg_i counts the listed edges at i.  Each term w (v_i - v_j) carries two
fp32 roundings (difference, product); a sum of deg_i terms in any order adds at most deg_i - 1 more of sum |terms|
(Higham, Accuracy and Stability, eq. 4.4), and the row's final store one (the fixed-point mode: its conversion back
to fp32, after it rounded each term to 2^-40).  The weights are fp32 numbers, exact in both computations.

LOBPCG checks: tests/spectral_graphs.py (eigenvalues, Davis-Kahan subspace, objective, constraint, convergence)."""
import functools
import logging

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

from tests import spectral_graphs as SG

pytestmark = pytest.mark.gpu

_ENV = ("MDE_B200_LAYOUT", "MDE_B200_TILE_RB", "MDE_B200_STILE_MB", "MDE_B200_TILE_MIN", "MDE_B200_PULL_EPL",
        "MDE_B200_PULL_REP", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC", "MDE_B200_ELL_BUILD", "PYMDE_B200_SPECTRAL")


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


# ------------------------------------------------------------------------------------------------------------------
# the operator V -> L V
# ------------------------------------------------------------------------------------------------------------------
def _trim(e, w, rem=3):
    """keep p = 32 q + rem edges: not a multiple of 4, of a warp or of any tile group"""
    p = (len(e) - rem) // 32 * 32 + rem
    return e[:p], w[:p]


def _family(name):
    """(n, edges, fp32 weights) of one graph family; n is not a multiple of 4, 32 or a tile"""
    n = 5003
    rng = np.random.default_rng(11)
    pts, _ = SG.mixture(n, 10, 10, 1.0, 3)
    e, w = SG.knn_edges(pts, 10)
    e, w = e[rng.permutation(len(e))], w  # edges in no particular order; weights stay 1 / 2 by position
    if name == "knn12":
        return (n,) + _trim(e, w)
    if name == "spread":  # positive weights over six decades
        return (n,) + _trim(e, (10.0 ** rng.uniform(-3, 3, len(e))).astype(np.float32))
    if name == "dup":  # a third listed again reversed, a fifth listed twice
        r = rng.choice(len(e), len(e) // 3, replace=False)
        d = rng.choice(len(e), len(e) // 5, replace=False)
        e2 = np.concatenate([e, e[r][:, ::-1], e[d]])
        w2 = np.concatenate([w, w[r] * 0.5, w[d] * 3.0]).astype(np.float32)
        o = rng.permutation(len(e2))
        return (n,) + _trim(e2[o], w2[o], 7)
    if name == "isolated":  # 41 nodes without an edge, the first and the last among them
        iso = np.concatenate([[0, n - 1], rng.choice(np.arange(1, n - 1), 39, replace=False)])
        keep = ~np.isin(e, iso).any(1)
        return (n,) + _trim(e[keep], w[keep], 29)
    if name == "dense":  # more than 64 edges per node: the default layout of the fused evaluation is ELL
        n = 1501
        pts, _ = SG.mixture(n, 4, 10, 1.0, 4)
        e, w = SG.knn_edges(pts, 160)
        return (n,) + _trim(e, w, 1)
    raise KeyError(name)


FAMILIES = ("knn12", "spread", "dup", "isolated", "dense")
_T0 = {"MDE_B200_TILE_MIN": "0"}
# config -> (environment, kind it must build on a sparse graph, kind on the dense one)
LAYOUTS = {
    "default": ({}, 0, 3),
    "soa": ({"MDE_B200_LAYOUT": "soa"}, 0, 0),
    "tiles": (dict(_T0, MDE_B200_LAYOUT="tiles"), 1, 1),
    "tiles_rb8": (dict(_T0, MDE_B200_LAYOUT="tiles", MDE_B200_TILE_RB="8"), 1, 1),
    "pull": (dict(_T0, MDE_B200_LAYOUT="pull"), 2, 2),
    "pull_rb8_epl4": (dict(_T0, MDE_B200_LAYOUT="pull", MDE_B200_TILE_RB="8", MDE_B200_PULL_EPL="4"), 2, 2),
    "ell": ({"MDE_B200_LAYOUT": "ell"}, 3, 3),
    "det": ({"MDE_B200_DETERMINISTIC": "1"}, 0, 0),
}
WIDE = (5, 8, 32, 128, 512)


def _operator_case(monkeypatch, family, kb, env):
    from pymde_b200 import _lib, quadratic
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n, e, w = _family(family)
    op = quadratic._LaplacianOperator(n, kb, torch.tensor(e), torch.tensor(w), "cuda")
    kind = int(_lib.load().mde_edges_kind(op.layout.handle))
    det = int(_lib.load().mde_edges_deterministic(op.layout.handle))
    rng = np.random.default_rng(kb)
    V = rng.standard_normal((n, kb)).astype(np.float32)
    V[:, 0] += 40.0  # an offset column: v_i - v_j cancels
    Vd = torch.tensor(V, device="cuda")
    got = op(Vd).cpu().numpy().astype(np.float64)
    L = SG.laplacian(n, e, w)
    want = L @ V.astype(np.float64)
    A = abs(L - sp.diags(L.diagonal())).tocsr()
    scale = L.diagonal()[:, None] * np.abs(V) + A @ np.abs(V)  # sum_j w_ij (|v_i| + |v_j|)
    cnt = np.bincount(e.ravel(), minlength=n)[:, None].astype(np.float64)
    tol = (cnt + 2) * 2.0 ** -24 * scale + (cnt * 2.0 ** -40 if det else 0.0)
    bad = np.abs(got - want) > tol
    assert not bad.any(), (family, kb, env, int(bad.sum()), np.argwhere(bad)[:5],
                           got[bad][:5], want[bad][:5], tol[bad][:5])
    np.testing.assert_allclose(op.degree.cpu().numpy(), L.diagonal(), rtol=2e-6)
    return op, Vd, got, kind, det


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kb", [1, 2, 3, 4])
def test_operator_narrow(monkeypatch, family, layout, kb):
    env, kind_sparse, kind_dense = LAYOUTS[layout]
    op, V, got, kind, det = _operator_case(monkeypatch, family, kb, env)
    assert kind == (kind_dense if family == "dense" else kind_sparse), (layout, family, kind)
    if layout == "det":
        assert det == 1
        assert torch.equal(op(V), op(V)), "the fixed-point mode must give the same bits on every call"


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("kb", WIDE)
def test_operator_wide(monkeypatch, family, det, kb):
    env = {"MDE_B200_DETERMINISTIC": "1"} if det else {}
    op, V, got, kind, d = _operator_case(monkeypatch, family, kb, env)
    assert kind == 0 and d == int(det)
    if det:
        assert torch.equal(op(V), op(V)), "the wide owner kernel must give the same bits on every call"


# ------------------------------------------------------------------------------------------------------------------
# LOBPCG against shift-invert Lanczos
# ------------------------------------------------------------------------------------------------------------------
ITERATIONS = {}  # case -> LOBPCG iterations, printed at the end of the module (pytest -s)


@pytest.fixture(scope="module", autouse=True)
def _report_iterations():
    yield
    for k, v in sorted(ITERATIONS.items()):
        print("LOBPCG iterations %-28s %d" % (k, v))


@functools.lru_cache(maxsize=None)
def _graph(name):
    if name == "mixture":  # connected: a k = 15 neighbour graph of a 10-component mixture in 30 dimensions
        n = 10000
        pts, _ = SG.mixture(n, 10, 30, 1.0, 0)
        return n, SG.knn_edges(pts, 15)
    if name == "square":  # lambda_2 ~ lambda_3
        n = 10000
        return n, SG.knn_edges(SG.square(n, 1), 10)
    if name.startswith("disconnected"):  # c well-separated components: c zero eigenvalues
        n, c = 6000, int(name[len("disconnected"):])
        pts, _ = SG.mixture(n, c, 10, 30.0, 2)
        return n, SG.knn_edges(pts, 10)
    if name.startswith("isolated"):
        n, k = 6000, int(name[len("isolated"):])
        pts, _ = SG.mixture(n, 10, 10, 1.0, 5)
        e, w = SG.knn_edges(pts, 10)
        keep = ~np.isin(e, np.arange(k) * 997 + 13).any(1)
        return n, (e[keep], w[keep])
    raise KeyError(name)


@functools.lru_cache(maxsize=None)
def _reference(name):
    """L, its number of components and its smallest eigenpairs: enough for m <= 30 and the whole null space"""
    n, (e, w) = _graph(name)
    L = SG.laplacian(n, e, w)
    c = csgraph.connected_components(L)[0]
    return L, c, SG.smallest_pairs(L, max(39 if name == "mixture" else 17, c + 6))


def _device_case(name, m):
    from pymde_b200 import quadratic
    n, (e, w) = _graph(name)
    X = quadratic.spectral_device(n, m, torch.tensor(e), torch.tensor(w), "cuda")
    info = X._lobpcg_info
    ITERATIONS["%s m=%d" % (name, m)] = info["iterations"]
    L, c, (vals, vecs) = _reference(name)
    assert info["converged"], info
    out = SG.check(L, X.double().cpu().numpy(), info["eigenvalues"], info["residuals"], vals, vecs, m)
    return L, c, vals, out


@pytest.mark.parametrize("m", [1, 2, 3, 8, 12, 16, 30])
def test_lobpcg_connected_mixture(m):
    _, c, _, _ = _device_case("mixture", m)
    assert c == 1


@pytest.mark.parametrize("m", [1, 2])
def test_lobpcg_near_double_eigenvalue(m):
    _, _, vals, _ = _device_case("square", m)
    assert vals[2] - vals[1] < 0.1 * vals[1]


@pytest.mark.parametrize("name,m", [("disconnected3", 3), ("disconnected12", 3), ("disconnected12", 8)])
def test_lobpcg_disconnected(name, m):
    """fewer components than m + 1: the null space and the lowest modes; more: any standardised basis of the null
    space is right, so only ||L X|| (the objective, ~0) and the rank (the Gram check) are asserted"""
    L, c, vals, out = _device_case(name, m)
    assert c == int(name[len("disconnected"):])
    if c > m + 1:
        assert out["objective"][0] <= 4 * m * SG.FLOOR * SG.a_norm(L)


@pytest.mark.parametrize("name,m", [("isolated1", 2), ("isolated1", 3), ("isolated3", 5), ("isolated3", 2)])
def test_lobpcg_isolated_nodes(name, m):
    L, _, _, _ = _device_case(name, m)
    assert (L.diagonal() == 0).sum() == int(name[len("isolated"):])


def test_anchored_recipe(monkeypatch):
    """anchored preserve_neighbors: anchor-anchor edges removed, the interior of an anchored cluster left isolated"""
    import pymde_b200 as pm
    from pymde_b200 import quadratic
    seen = {}
    real = quadratic.spectral

    def spy(n_items, embedding_dim, edges, weights, **kw):
        X = real(n_items, embedding_dim, edges, weights, **kw)
        seen.update(n=int(n_items), m=int(embedding_dim), e=edges.cpu().numpy(), w=weights.cpu().numpy(), X=X.clone(),
                    info=getattr(X, "_lobpcg_info", None))
        return X

    monkeypatch.setattr(quadratic, "spectral", spy)
    n, m = 6000, 2
    pts, _ = SG.mixture(n - 20, 6, 10, 3.0, 7)
    far = 1000.0 + 0.1 * np.random.default_rng(8).standard_normal((20, 10)).astype(np.float32)
    pts = np.concatenate([pts, far])
    anchors = np.arange(n - 20, n)  # every neighbour of these is another of them: all 20 end up isolated
    c = pm.Anchored(torch.tensor(anchors, device="cuda"), torch.zeros(len(anchors), m, device="cuda"))
    pm.seed(0)
    pm.preserve_neighbors(torch.tensor(pts, device="cuda"), embedding_dim=m, constraint=c, device="cuda")
    assert seen["info"] is not None  # the device path ran
    e, w = seen["e"], seen["w"]
    assert not (np.isin(e[:, 0], anchors) & np.isin(e[:, 1], anchors)).any()
    L = SG.laplacian(n, e, w)
    iso = int((L.diagonal() == 0).sum())
    assert iso == 20
    k = csgraph.connected_components(L)[0]
    vals, vecs = SG.smallest_pairs(L, max(m + 9, k + 6))
    ITERATIONS["anchored m=%d (%d isolated)" % (m, iso)] = seen["info"]["iterations"]
    SG.check(L, seen["X"].double().cpu().numpy(), seen["info"]["eigenvalues"], seen["info"]["residuals"], vals, vecs, m)


# ------------------------------------------------------------------------------------------------------------------
# dispatch and the unconverged fallback
# ------------------------------------------------------------------------------------------------------------------
def _host_reference_objective(L, m):
    vals = SG.smallest_pairs(L, m + 1)[0]
    return float(vals[1:m + 1].sum())


@pytest.mark.parametrize("n,device_path", [(2000, False), (2001, True)])
def test_dispatch_item_count(n, device_path):
    from pymde_b200 import quadratic
    pts, _ = SG.mixture(n, 10, 10, 1.0, 8)
    e, w = SG.knn_edges(pts, 10)
    m = 2
    X = quadratic.spectral(n, m, torch.tensor(e), torch.tensor(w), device="cuda")
    assert hasattr(X, "_lobpcg_info") == device_path
    L = SG.laplacian(n, e, w)
    Xd = X.double().cpu().numpy()
    obj = float(np.sum(Xd * (L @ Xd))) / n
    s = _host_reference_objective(L, m)
    assert s * (1 - 1e-6) <= obj <= s * (1 + 2e-3)
    np.testing.assert_allclose(Xd.T @ Xd / n, np.eye(m), atol=1e-3)


@pytest.mark.parametrize("m", [1998, 1999])
def test_dispatch_wide_blocks_stay_on_host(m):
    """m = n - 3 and n - 2 just above the item threshold: a block of m + 2 vectors is wider than the external
    scatter's kernels (512 columns), so both run on the host"""
    from pymde_b200 import quadratic
    n = 2001
    pts, _ = SG.mixture(n, 10, 10, 1.0, 9)
    e, w = SG.knn_edges(pts, 10)
    X = quadratic.spectral(n, m, torch.tensor(e), torch.tensor(w), device="cuda")
    assert not hasattr(X, "_lobpcg_info")
    assert tuple(X.shape) == (n, m) and X.is_cuda
    Xd = X.double().cpu().numpy()
    assert np.abs(Xd.mean(0)).max() < 1e-3
    np.testing.assert_allclose(Xd.T @ Xd / n, np.eye(m), atol=1e-3)


def test_unconverged_device_result_is_recomputed_on_host(monkeypatch, caplog):
    from pymde_b200 import problem, quadratic
    n, m = 6000, 3
    pts, _ = SG.mixture(n, 10, 10, 1.0, 12)
    e, w = SG.knn_edges(pts, 10)
    X = quadratic.spectral_device(n, m, torch.tensor(e), torch.tensor(w), "cuda", max_iter=2)
    info = X._lobpcg_info
    assert info["iterations"] == 2 and not info["converged"]

    real = quadratic.spectral_device
    monkeypatch.setattr(quadratic, "spectral_device", lambda *a, **kw: real(*a, **dict(kw, max_iter=2)))
    monkeypatch.setattr(problem.LOGGER, "propagate", True)
    with caplog.at_level(logging.WARNING, logger=problem.LOGGER.name):
        X = quadratic.spectral(n, m, torch.tensor(e), torch.tensor(w), device="cuda")
    assert not hasattr(X, "_lobpcg_info")  # the host result
    assert any("did not converge" in r.getMessage() for r in caplog.records)
    L = SG.laplacian(n, e, w)
    Xd = X.double().cpu().numpy()
    s = _host_reference_objective(L, m)
    assert float(np.sum(Xd * (L @ Xd))) / n <= s * (1 + 1e-3)


# ------------------------------------------------------------------------------------------------------------------
# end to end: laplacian_embedding against the optimum of min tr(X^T L X) s.t. X^T X = n I
# ------------------------------------------------------------------------------------------------------------------
INIT_RTOL = 1e-3   # the initialisation: residuals <= 1e-4 lambda put the objective within O((1e-4)^2 / gap) of it
EMBED_RTOL = 5e-3  # the solver starts there and stops at its own tolerance, near the optimum it cannot undercut


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("m", [2, 8])
def test_laplacian_embedding_reaches_the_optimum(sparse, m):
    import pymde_b200 as pm
    n = 5000
    pts, _ = SG.mixture(n, 8, 20, 1.0, 13)
    if sparse:
        pts[np.random.default_rng(14).random(pts.shape) < 0.6] = 0.0
        data = sp.csr_matrix(pts)
    else:
        data = torch.tensor(pts, device="cuda")
    pm.seed(0)
    mde = pm.laplacian_embedding(data, embedding_dim=m, device="cuda")
    e = mde.edges.cpu().numpy()
    w = mde.distortion_function.weights.detach().cpu().numpy()
    L = SG.laplacian(n, e, w)
    vals = SG.smallest_pairs(L, m + 1)[0]
    target = n * float(vals[1:m + 1].sum()) / len(e)
    init = mde.average_distortion(mde._X_init).item()
    assert target * (1 - 1e-5) <= init <= target * (1 + INIT_RTOL), (init, target)
    X = mde.embed()
    final = mde.average_distortion(X).item()
    assert target * (1 - 1e-5) <= final <= target * (1 + EMBED_RTOL), (final, target)
