"""Quadratic (spectral) initialisation (interface of pymde/quadratic.py:16-179): the bottom eigenvectors
of the graph Laplacian, standardised.  Runs once before `embed`.

On a CUDA device the eigenvectors come from `spectral_device`: a block LOBPCG iteration whose only n-sized
sparse operation, V -> L V, IS the gradient scatter of the edge kernels (`mde_scatter_external` with the edge
weights as per-edge coefficients: sum_k w_k (v_i - v_j)(e_i - e_j) = L V), so the initialisation reuses the
layout machinery of the hot path and never leaves the device.  The host path (scipy Lanczos, what the
reference does at quadratic.py:84-96) remains for tiny problems and as the parity arbiter of the tests."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg
import torch

from . import util


def pca(Y, embedding_dim):
    """Top principal directions, scaled to a standardized embedding (quadratic.py:16-44)."""
    Y = Y if isinstance(Y, torch.Tensor) else torch.as_tensor(np.asarray(Y))
    Y = Y.float()
    n = Y.shape[0]
    Yc = Y - Y.mean(0)
    U, _, _ = torch.linalg.svd(Yc, full_matrices=False)
    return (n ** 0.5) * U[:, :embedding_dim]


def _laplacian(n, edges, weights):
    e = edges.detach().cpu().numpy() if isinstance(edges, torch.Tensor) else np.asarray(edges)
    w = weights.detach().cpu().numpy() if isinstance(weights, torch.Tensor) else np.asarray(weights)
    A = sp.coo_matrix((w, (e[:, 0], e[:, 1])), shape=(n, n), dtype=np.float64)
    A = (A + A.T).tocsr()
    return sp.diags(np.asarray(A.sum(1)).ravel()) - A


class _LaplacianOperator(object):
    """V (n, k) -> L V on the device through the edge layout (k <= 4: quad / tile kernels, else the wide kernel)."""

    def __init__(self, n, k, edges, weights, device):
        from . import _lib
        from .problem import EdgeLayout
        table = _lib.mde_fn_t()
        table.fn_att = table.fn_rep = 100  # MDE_FN_EXTERNAL: the layout only carries the index structure
        self.w = util.as_f32_cuda(weights, device).reshape(-1).contiguous()
        zeros = torch.zeros(int(edges.shape[0]), device=device)
        self.layout = EdgeLayout(edges, int(n), table, zeros, None, device, embedding_dim=int(k))
        e = edges.to(device)
        deg = torch.zeros(int(n), device=device)
        deg.index_add_(0, e[:, 0], self.w)
        deg.index_add_(0, e[:, 1], self.w)
        self.degree = deg

    def __call__(self, V):
        return self.layout.scatter_external(V.contiguous(), self.w)


def converged(lam, res, tol, a_norm):
    """LOBPCG's stopping rule, per pair: ||A x - lambda x|| <= tol * lambda (eigsh's relative criterion,
    quadratic.py:91), floored at the fp32 resolution of the operator, 2e-6 * ||A||.  A Ritz value below -2e-6 ||A||
    is not one of a positive semi-definite operator: the Rayleigh-Ritz step broke down, and no residual makes up
    for that."""
    floor = 2e-6 * a_norm
    return (res <= torch.maximum(tol * lam.abs().float(), torch.full_like(res, floor))) & (lam.float() >= -floor)


def lobpcg_smallest(apply_A, n, k, precond=None, device=None, max_iter=300, tol=1e-4, seed=0, deflate_constant=True,
                    a_norm=1.0, n_wanted=None):
    """k smallest eigenpairs of a symmetric positive semi-definite operator by block LOBPCG (Knyazev 2001), fp32
    vectors, fp64 Rayleigh-Ritz.  `deflate_constant`: iterate in the orthogonal complement of the all-ones vector (the
    Laplacian's known null vector).  `apply_A` is only called on blocks of exactly k columns.  Returns (eigenvalues
    (k,), eigenvectors (n, k), iterations, residual norms ||A x - lambda x|| with A applied to the returned x); the
    first `n_wanted` pairs meet `converged` unless the iteration stopped at `max_iter`.

    Each step searches span[X, W, P] (Ritz vectors, preconditioned residuals, previous update) with an orthonormal
    basis: W and P are orthonormalised against X and each other in fp64, numerically dependent directions are
    dropped, and the operator is applied to that basis afresh.  A recurrence for A P instead (one operator
    application per step) loses its accuracy as P shrinks near convergence, and the Rayleigh-Ritz step on the nearly
    dependent basis then returns Ritz values far below 0."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    nw = k if n_wanted is None else int(n_wanted)

    def clean(V):
        return V - V.mean(0, keepdim=True) if deflate_constant else V

    def apply(V):
        if V.shape[1] == k:
            return apply_A(V.contiguous())
        out = []
        for i in range(0, V.shape[1], k):
            blk = V[:, i:i + k]
            w = blk.shape[1]
            if w < k:
                blk = torch.cat([blk, blk.new_zeros(n, k - w)], 1)
            out.append(apply_A(blk.contiguous())[:, :w])
        return torch.cat(out, 1)

    def basis(Z, X):
        """orthonormal basis of the part of Z orthogonal to X (and to the constant); twice, as in CGS2.  Directions
        below 1e-5 of a unit column are dropped: fp32 data carries nothing there."""
        Zd, Xd = Z.double(), X.double()
        for _ in range(2):
            Zd = clean(Zd)
            Zd = Zd - Xd @ (Xd.T @ Zd)
            Zd = Zd / Zd.norm(dim=0).clamp_min(1e-300)
            mu, V = torch.linalg.eigh(Zd.T @ Zd)
            keep = mu > 1e-10 * max(float(mu[-1]), 1e-300)
            Zd = Zd @ (V[:, keep] / mu[keep].sqrt())
        return Zd.float()

    def rayleigh_ritz(X):
        """X orthonormalised, A X applied afresh, rotated onto its Ritz vectors"""
        Xd, _ = torch.linalg.qr(clean(X.double()))
        X = Xd.float()
        AXd = apply(X).double()
        T = X.double().T @ AXd
        lam, C = torch.linalg.eigh(0.5 * (T + T.T))
        return lam, (X.double() @ C).float(), (AXd @ C).float()

    lam, X, AX = rayleigh_ritz(torch.randn(n, k, device=device, generator=gen))
    P = None
    fresh = True  # AX is the operator applied to X, not the recurrence's update
    res = None
    it = 0
    for it in range(1, max_iter + 1):
        res = (AX - X * lam.float()[None, :]).norm(dim=0)
        if bool(converged(lam, res, tol, a_norm)[:nw].all()):
            if fresh:
                break
            # the recurrence's A X drifts in fp32: confirm with the operator itself
            lam, X, AX = rayleigh_ritz(X)
            fresh = True
            res = (AX - X * lam.float()[None, :]).norm(dim=0)
            if bool(converged(lam, res, tol, a_norm)[:nw].all()):
                break
        R = AX - X * lam.float()[None, :]
        W = R if precond is None else R * precond[:, None]
        Q = basis(torch.cat([W] + ([P] if P is not None else []), 1), X)
        AQ = apply(Q)
        S = torch.cat([X, Q], 1).double()
        AS = torch.cat([AX, AQ], 1).double()
        B = S.T @ S
        G = S.T @ AS
        G = 0.5 * (G + G.T)
        # generalized symmetric eigenproblem through the Cholesky factor of the Gram matrix (the identity up to fp32
        # rounding)
        Lc = torch.linalg.cholesky(B)
        Gt = torch.linalg.solve_triangular(Lc, torch.linalg.solve_triangular(Lc, G, upper=False).T, upper=False).T
        ev, Y = torch.linalg.eigh(0.5 * (Gt + Gt.T))
        Cc = torch.linalg.solve_triangular(Lc.T, Y[:, :k], upper=True)
        lam = ev[:k]
        Cx, Cq = Cc[:k], Cc[k:]
        Pd = S[:, k:] @ Cq
        X = (S[:, :k] @ Cx + Pd).float()
        AX = (AS[:, :k] @ Cx + AS[:, k:] @ Cq).float()
        P = Pd.float()
        fresh = False
    else:  # max_iter reached: the residuals of the pairs returned
        lam, X, AX = rayleigh_ritz(X)
        res = (AX - X * lam.float()[None, :]).norm(dim=0)
    return lam, X, it, res


def jacobi_preconditioner(degree):
    """1 / degree, and 1 on the rows of degree-0 nodes.  Their residual is -lambda x_i: a huge factor there turns every
    search direction into an isolated node's indicator, and with fewer isolated nodes than block vectors the
    iteration diverges."""
    return torch.where(degree > 0, 1.0 / degree, torch.ones_like(degree))


def spectral_device(n_items, embedding_dim, edges, weights, device, max_iter=300, tol=1e-4):
    """Device path of `spectral`: eigenvectors 2..m+1 of L = D - W by LOBPCG with the Jacobi (degree) preconditioner,
    the constant vector deflated exactly (quadratic.py:71-120 asks eigsh / torch.lobpcg for m + 1 vectors and drops
    the first)."""
    n, m = int(n_items), int(embedding_dim)
    dev = util.cuda_device(device)
    edges = edges if isinstance(edges, torch.Tensor) else torch.as_tensor(np.asarray(edges))
    kb = min(m + 2, n - 2)  # two guard vectors: 10-100x fewer iterations on poorly separated spectra
    op = _LaplacianOperator(n, kb, edges.to(dev), weights, dev)
    precond = jacobi_preconditioner(op.degree)
    a_norm = 2.0 * float(op.degree.max())
    lam, X, iters, res = lobpcg_smallest(op, n, kb, precond=precond, device=dev, max_iter=max_iter, tol=tol,
                                         a_norm=a_norm, n_wanted=m)
    lam, res = lam[:m], res[:m]
    ok = bool(converged(lam, res, tol, a_norm).all())
    X = X[:, :m].contiguous()
    out = util.proj_standardized(X, demean=True, inplace=True)
    out._lobpcg_info = {"iterations": iters, "eigenvalues": lam.cpu().numpy(), "residuals": res.cpu().numpy(),
                        "converged": ok}
    return out


def spectral(n_items, embedding_dim, edges, weights, cg=False, max_iter=1000, device=None):
    """Standardized spectral embedding: eigenvectors 2..m+1 of L = D - W (quadratic.py:122-179).  CUDA problems with
    more than 2 000 items use the device LOBPCG (`spectral_device`); PYMDE_B200_SPECTRAL=host forces the host path.
    A device result whose wanted pairs miss the stopping rule at the iteration cap is logged and recomputed on the
    host.  Blocks wider than the edge kernels' external scatter (m + 2 > 512) stay on the host."""
    import os
    if (torch.cuda.is_available() and int(n_items) > 2000 and os.environ.get("PYMDE_B200_SPECTRAL", "device") != "host"
            and int(embedding_dim) + 2 <= 512):
        X = spectral_device(n_items, embedding_dim, edges, weights, device, max_iter=min(int(max_iter), 400))
        info = X._lobpcg_info
        if info["converged"]:
            return X
        from . import problem
        problem.LOGGER.warning("spectral initialisation: LOBPCG did not converge in %d iterations (largest residual "
                               "%.3g); recomputing on the host" % (info["iterations"], float(info["residuals"].max())))
    L = _laplacian(int(n_items), edges, weights)
    k = int(embedding_dim) + 1
    rng = np.random.default_rng(0)
    if int(n_items) <= max(k + 1, 32):  # Lanczos needs k < n; tiny problems go through a dense eigensolver
        vals, vecs = np.linalg.eigh(L.toarray())
        vals, vecs = vals[:k], vecs[:, :k]
        if vecs.shape[1] < k:  # fewer items than requested directions: pad with random columns
            vecs = np.concatenate([vecs, rng.standard_normal((int(n_items), k - vecs.shape[1]))], 1)
            vals = np.concatenate([vals, np.full(k - vals.shape[0], np.inf)])
        return _finish(vals, vecs, k, n_items, device)
    try:
        vals, vecs = scipy.sparse.linalg.eigsh(L, k=k, sigma=-1e-3 * max(1.0, L.diagonal().mean()), which="LM",
                                               maxiter=max_iter, v0=rng.standard_normal(int(n_items)))
    except Exception:
        vals, vecs = scipy.sparse.linalg.eigsh(L, k=k, which="SA", maxiter=max_iter * 10,
                                               v0=rng.standard_normal(int(n_items)))
    return _finish(vals, vecs, k, n_items, device)


def _finish(vals, vecs, k, n_items, device):
    order = np.argsort(vals)
    X = torch.tensor(vecs[:, order[1:k]].astype(np.float32))
    if torch.cuda.is_available():
        X = X.to(util.cuda_device(device)).contiguous()
        return util.proj_standardized(X, demean=True, inplace=True)
    X = X - X.mean(0)
    U, _, Vh = torch.linalg.svd(X, full_matrices=False)
    return (float(n_items) ** 0.5) * (U @ Vh)
