"""Graphs and fp64 arbiters of the spectral-initialisation tests (test_spectral_cpu.py, test_gpu_spectral.py).

The checks are written so that they hold when eigenvalues repeat or nearly repeat, where the eigenvectors are not
unique: the eigenvalues themselves, the principal angles between the returned block and a whole invariant subspace
(Davis-Kahan), the quadratic objective tr(X^T L X) / n, and the standardisation constraint."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import scipy.sparse.linalg as sla
from scipy.spatial import cKDTree

# the solver's stopping rule (quadratic.lobpcg_smallest): ||L x - lambda x|| <= max(TOL * lambda, FLOOR * a_norm),
# a_norm = 2 max degree >= ||L||_2 (Gershgorin); FLOOR is the fp32 resolution of L V
TOL = 1e-4
FLOOR = 2e-6


def knn_edges(pts, k):
    """k-nearest-neighbour graph with the recipes' weights: 2 for mutual neighbours, 1 for one-sided ones"""
    n = len(pts)
    _, idx = cKDTree(pts).query(pts, k=k + 1)
    i, j = np.repeat(np.arange(n), k), idx[:, 1:].ravel()
    keep = i != j  # exact duplicate points can put i itself among its neighbours
    lo, hi = np.minimum(i, j)[keep], np.maximum(i, j)[keep]
    key, cnt = np.unique(lo.astype(np.int64) * n + hi, return_counts=True)
    e = np.stack([key // n, key % n], 1).astype(np.int64)
    return e, cnt.astype(np.float32)


def mixture(n, c, d, sep, seed):
    """n points of a c-component Gaussian mixture in d dimensions; centres sep apart on average"""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((c, d)) * sep
    lab = np.arange(n) % c
    return (centres[lab] + rng.standard_normal((n, d))).astype(np.float32), lab


def square(n, seed):
    """uniform points in the unit square: the two lowest non-trivial modes (cos(pi x), cos(pi y)) nearly coincide"""
    return np.random.default_rng(seed).random((n, 2)).astype(np.float32)


def laplacian(n, e, w):
    """fp64 L = D - W, each listed edge contributing w to both (i, j) and (j, i)"""
    e = np.asarray(e, np.int64)
    A = sp.coo_matrix((np.asarray(w, np.float64), (e[:, 0], e[:, 1])), shape=(n, n))
    A = (A + A.T).tocsr()
    return (sp.diags(np.asarray(A.sum(1)).ravel()) - A).tocsr()


def a_norm(L):
    return 2.0 * float(L.diagonal().max())


def _smallest_pairs_connected(L, k):
    n = L.shape[0]
    if n <= 3000:
        vals, vecs = np.linalg.eigh(L.toarray())
        return vals[:k], vecs[:, :k]
    sigma = -1e-3 * max(1.0, float(L.diagonal().mean()))
    v0 = np.random.default_rng(0).standard_normal(n)
    vals, vecs = sla.eigsh(L, k=k, sigma=sigma, which="LM", tol=1e-12, v0=v0)
    o = np.argsort(vals)
    return vals[o], vecs[:, o]


def smallest_pairs(L, k):
    """the k smallest eigenpairs of L in fp64, ascending, component by component (Lanczos can miss copies of a
    repeated eigenvalue, and each component contributes one zero): dense below 3 000 rows, else shift-invert
    Lanczos, whose zero eigenvalue is then simple"""
    n = L.shape[0]
    nc, lab = csgraph.connected_components(L, directed=False)
    vals, cols = [], []
    for c in range(nc):
        idx = np.flatnonzero(lab == c)
        v, V = _smallest_pairs_connected(L[idx][:, idx].tocsr(), min(k, len(idx)))
        vals.append(v)
        cols.extend((idx, V[:, i]) for i in range(V.shape[1]))
    vals = np.concatenate(vals)
    o = np.argsort(vals, kind="stable")[:k]
    vecs = np.zeros((n, len(o)))
    for t, i in enumerate(o):
        vecs[cols[i][0], t] = cols[i][1]
    return vals[o], vecs


def check(L, X, lam, res, ref_vals, ref_vecs, m, objective_rtol=2e-3):
    """Assert that (lam, X, res) from LOBPCG is a right answer for eigenpairs 2..m+1 of L; return what was measured.

    ref_vals / ref_vecs: the smallest eigenpairs of L in fp64, at least m + 3 of them (index 0 is the constant).
    X: n x m, centred and standardised (X^T X = n I)."""
    n = L.shape[0]
    An = a_norm(L)
    X = np.asarray(X, np.float64)
    want = ref_vals[1:m + 1]
    out = {}
    # eigenvalues: the residual criterion bounds each Ritz value's distance from the spectrum by tol * lambda +
    # floor * ||L||; twice that leaves room for the fp32 rounding of the block and of L V
    lam = np.asarray(lam, np.float64)[:m]
    err = np.abs(lam - want)
    lim = 2.0 * (TOL * np.abs(want) + FLOOR * An)
    assert (err <= lim).all(), ("eigenvalues", lam, want, err / lim)
    # convergence: the reported residuals meet the solver's own criterion (and, below, the fp64 residuals of X)
    res = np.asarray(res, np.float64)[:m]
    assert (res <= np.maximum(TOL * np.abs(lam), FLOOR * An) * (1 + 1e-6)).all(), ("residuals", res, lam)
    # constraint: centred, standardised (quadratic.py:178-179)
    out["mean"] = float(np.abs(X.mean(0)).max() / np.sqrt(np.mean(X * X)))
    assert out["mean"] < 1e-4, out
    G = X.T @ X / n
    out["gram"] = float(np.abs(G - np.eye(m)).max())
    assert out["gram"] < 1e-3, out
    # objective: tr(X^T L X) / n against its minimum over standardised X, sum lambda_2..lambda_{m+1}; independent of
    # the basis, so it means the same thing when eigenvalues repeat
    LX = L @ X
    obj = float(np.sum(X * LX)) / n
    s = float(want.sum())
    out["objective"] = (obj, s)
    assert obj >= s - 1e-9 * An * m - 1e-6 * s, ("objective below the minimum", obj, s)
    assert obj <= s * (1 + objective_rtol) + 4 * m * FLOOR * An, ("objective", obj, s)
    # subspace: Davis-Kahan sin-theta.  Q orthonormal basis of X, Theta its Ritz values, R = L Q - Q Theta.  For every
    # cut j >= m (the invariant subspace of ref_vals[0..j], a whole cluster when the cut lies in a gap), the largest
    # principal-angle sine between X and that subspace is at most ||R||_2 / (lambda_{j+1} - max Theta).  A cut between
    # two fp64 values of one repeated eigenvalue (the null space of a disconnected graph) separates nothing.
    Q, _ = np.linalg.qr(X)
    T = Q.T @ (L @ Q)
    th, C = np.linalg.eigh(0.5 * (T + T.T))
    Q = Q @ C
    R = L @ Q - Q * th[None, :]
    Rn = float(np.linalg.norm(R, 2))
    out["resid"] = Rn
    # convergence, recomputed: the Ritz pairs of X meet the stopping rule with L applied in fp64 (1.5x for the
    # rounding of X to fp32 and of the solver's fp32 L V, both far below the floor)
    r64 = np.linalg.norm(R, axis=0)
    lim = np.maximum(TOL * np.abs(th), FLOOR * An)
    assert (r64 <= 1.5 * lim).all(), ("fp64 residuals", r64 / lim, th)
    bounds = []
    for j in range(m, len(ref_vals) - 1):
        gap = ref_vals[j + 1] - th.max()
        if gap <= 0 or ref_vals[j + 1] - ref_vals[j] <= 1e-9 * An:  # no gap inside a (numerically) repeated eigenvalue
            continue
        V = ref_vecs[:, :j + 1]
        sines = np.linalg.svd(Q - V @ (V.T @ Q), compute_uv=False)
        bound = Rn / gap
        bounds.append((j, float(sines.max()), bound))
        assert sines.max() <= 1.05 * bound + 1e-6, ("Davis-Kahan", j, sines.max(), bound)
    out["davis_kahan"] = bounds
    # the check means something only where some cut has a small bound
    assert bounds and min(b for _, _, b in bounds) < 0.1, ("no separated cut among the reference pairs", bounds)
    return out
