"""The device spectral initialisation's algorithm on the CPU: `quadratic.lobpcg_smallest` with the Jacobi
preconditioner of `spectral_device`, driven by an fp32 scipy L V in place of the edge kernel, against fp64 eigenpairs
(tests/spectral_graphs.py) on small connected, near-degenerate, disconnected and isolated-node graphs."""
import functools

import numpy as np
import pytest
import scipy.sparse.csgraph as csgraph
import torch

from pymde_b200 import quadratic
from tests import spectral_graphs as SG


def _solve(L, m, max_iter=400):
    """what spectral_device does, on the CPU: kb = m + 2 block vectors, m wanted, the first m standardised"""
    n = L.shape[0]
    L32 = L.astype(np.float32)
    deg = torch.tensor(L.diagonal(), dtype=torch.float32)
    kb = min(m + 2, n - 2)
    lam, X, it, res = quadratic.lobpcg_smallest(
        lambda V: torch.from_numpy(np.asarray(L32 @ V.numpy(), np.float32)), n, kb,
        precond=quadratic.jacobi_preconditioner(deg), device="cpu", max_iter=max_iter, a_norm=SG.a_norm(L), n_wanted=m)
    Xs = X[:, :m].double().numpy()
    Xs = Xs - Xs.mean(0)
    U, _, Vt = np.linalg.svd(Xs, full_matrices=False)
    return lam[:m].numpy(), np.sqrt(n) * (U @ Vt), it, res[:m].numpy(), X


def _check(L, m):
    lam, X, it, res, _ = _solve(L, m)
    vals, vecs = SG.smallest_pairs(L, L.shape[0])
    return SG.check(L, X, lam, res, vals, vecs, m), it


def _mixture_graph(n, c, sep, seed, k=10):
    pts, _ = SG.mixture(n, c, 10, sep, seed)
    e, w = SG.knn_edges(pts, k)
    return SG.laplacian(n, e, w)


@pytest.mark.parametrize("m", [1, 2, 3, 8])
def test_connected_mixture(m):
    _check(_mixture_graph(2000, 10, 1.0, 0), m)


@pytest.mark.parametrize("m", [1, 2, 3])
def test_square_near_double_eigenvalue(m):
    L = SG.laplacian(2000, *SG.knn_edges(SG.square(2000, 1), 10))
    vals = SG.smallest_pairs(L, 4)[0]
    assert abs(vals[2] - vals[1]) < 0.1 * vals[1]  # lambda_2 ~ lambda_3: only the cluster's subspace is unique
    _check(L, m)


@pytest.mark.parametrize("c,m", [(3, 1), (3, 3), (12, 3)])
def test_disconnected_mixture(c, m):
    """c components: c zero eigenvalues.  c <= m: the answer spans the null space and the lowest non-trivial modes
    (at c = 3, m = 3 the block converges in the null space long before its fourth pair, which a recurrence for A P
    does not survive); c > m + 1: any standardised basis inside the null space is right (||L X|| ~ 0, full rank)."""
    L = _mixture_graph(2000, c, 30.0, 2)
    assert csgraph.connected_components(L)[0] == c
    out, _ = _check(L, m)
    if c > m + 1:
        assert out["objective"][0] <= 4 * m * SG.FLOOR * SG.a_norm(L)


@functools.lru_cache(maxsize=None)
def _wide_reference():
    """a k = 15 neighbour graph of a 10-component mixture, n = 10 000 in 30 dimensions, and its 40 smallest pairs"""
    pts, _ = SG.mixture(10000, 10, 30, 1.0, 0)
    L = SG.laplacian(10000, *SG.knn_edges(pts, 15))
    return L, SG.smallest_pairs(L, 40)


@pytest.mark.parametrize("m", [12, 16, 30])
def test_wide_blocks_converge(m):
    """embedding dimensions of 12 and more: the blocks whose P shrinks by orders of magnitude before the last pairs
    converge"""
    L, (vals, vecs) = _wide_reference()
    lam, X, it, res, _ = _solve(L, m)
    assert it < 400
    SG.check(L, X, lam, res, vals, vecs, m)


@pytest.mark.parametrize("n_iso,m", [(1, 2), (1, 3), (3, 2), (3, 5)])
def test_isolated_nodes(n_iso, m):
    """degree-0 nodes (anchored recipes remove anchor-anchor edges): one zero eigenvalue each, with fewer and with
    more isolated nodes than block vectors"""
    pts, _ = SG.mixture(2000, 10, 10, 1.0, 0)
    e, w = SG.knn_edges(pts, 10)
    iso = np.arange(n_iso) * 577 + 5
    keep = ~np.isin(e, iso).any(1)
    L = SG.laplacian(2000, e[keep], w[keep])
    assert (L.diagonal()[iso] == 0).all()
    _check(L, m)


def test_jacobi_preconditioner_is_one_on_isolated_rows():
    deg = torch.tensor([0.0, 2.0, 0.5, 0.0])
    assert torch.equal(quadratic.jacobi_preconditioner(deg), torch.tensor([1.0, 0.5, 2.0, 1.0]))


def test_unconverged_result_reports_its_own_residuals():
    """stopped at max_iter: the residuals returned are those of the pairs returned, and they miss the stopping rule"""
    L = _mixture_graph(2000, 10, 1.0, 0)
    L32 = L.astype(np.float32)
    deg = torch.tensor(L.diagonal(), dtype=torch.float32)
    lam, X, it, res = quadratic.lobpcg_smallest(
        lambda V: torch.from_numpy(np.asarray(L32 @ V.numpy(), np.float32)), L.shape[0], 5,
        precond=quadratic.jacobi_preconditioner(deg), device="cpu", max_iter=3, a_norm=SG.a_norm(L), n_wanted=3)
    assert it == 3
    Xd = X.double().numpy()
    R = L @ Xd - Xd * lam.numpy()[None, :]
    np.testing.assert_allclose(res.numpy(), np.linalg.norm(R, axis=0), rtol=1e-3)
    assert not bool(quadratic.converged(lam, res, 1e-4, SG.a_norm(L))[:3].all())
