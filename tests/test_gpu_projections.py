"""The Standardized constraint's device projections (csrc/mde_project.cu, csrc/mde_project_wide.cu) against an fp64
polar factor, on input that is off-centre, badly scaled, ill conditioned or rank deficient.

Reference (oracle/mde_oracle.py, Standardized): de-mean in fp64, thin SVD, sqrt(n) U V^T; tangent Z - X (Z^T X) / n
in fp64.  The thin SVD is a QR factorisation of the de-meaned matrix followed by the SVD of its m x m factor, in
fp64 on the device, so that n = 4.4 M rows stay cheap.

Widths reach every path: m <= 4 (a thread per row), 5 <= m <= 32 (a warp per row), 32 < m <= 256 (tiled Gram,
Newton-Schulz) on both sides of the 64-wide Gram tile and of the 32-column padding of the row kernel, and m = 257
(fp64 eigendecomposition through torch).  Row counts straddle the grid caps of the row kernels (264 blocks x 256
rows, 264 x 8 rows, 528 x 32 rows), and one case passes 64 x 264 x 256 rows so that every thread of the m <= 4
moments kernel flushes its fp32 partial sums.

Bounds.  The Gram is accumulated in fp32, so its rounding, seen from the smallest singular direction of the de-meaned
matrix X_c, grows like cond(X_c)^2:
- ||Y^T Y / n - I||_max <= 2e-5 for cond(X_c) <= 200, and 1e-2 (cond(X_c) / 1000)^2 above (the long fp32 runs of
  the tiled Gram of m > 32 reach the 1e-3 range at cond(X_c) = 1e3);
- max |Y - Y_ref| <= 1e-4 * cond(X_c) + a;
- |column mean of Y| <= 1e-5 + a.
Here a = ulp(mu) |W_ref| is what storing the column mean mu in fp32 costs: one ulp of the offset, carried through the
whitening W_ref = sqrt(n) (X_c^T X_c)^(-1/2).  The fp32 SVD of the de-meaned input pays the same.
Rank-deficient input (a constant or duplicated column, n <= m) raises SolverError, and so does a conditioning the
Newton-Schulz chain cannot reach in its 24 iterations.

The test without the gpu mark shows that these inputs separate the two Gram formulas: products of the uncentred
rows minus n mu mu^T miss the constraint bound, products of the rows shifted as the kernels shift them meet it."""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O

gpu = pytest.mark.gpu

NARROW_SMALL = [1, 2, 3, 4]
NARROW_WARP = [5, 7, 16, 31, 32]
WIDE = [33, 63, 64, 65, 128, 129, 255, 256]
WIDTHS = NARROW_SMALL + NARROW_WARP + WIDE + [257]
# (offset in column standard deviations, column scales)
KINDS = {
    "off0": (0.0, "unit"), "off10": (10.0, "unit"), "off1000": (1000.0, "unit"),
    "scaled0": (0.0, "log"), "scaled10": (10.0, "log"), "scaled1000": (1000.0, "log"),
    "cond1e3": (10.0, "cond"), "near": (0.0, "near"),
}
# row counts on both sides of each grid cap: 264 x 256 (m <= 4), 264 x 8 (warp path), 528 x 32 (wide row kernel)
CAPS = [(m, c + d) for m, c in ((2, 67584), (4, 67584), (5, 2112), (32, 2112), (33, 16896), (256, 16896))
        for d in (-1, 0, 1)]


def _pm():
    import pymde_b200 as pm
    return pm


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _polar64(X):
    """(sqrt(n) U V^T of the fp64 de-meaned X, singular values, fp64 column means, W = sqrt(n) V S^-1 V^T)."""
    n = X.shape[0]
    mu = X.double().mean(0)
    Q, R = torch.linalg.qr(X.double() - mu)
    Ur, S, Vh = torch.linalg.svd(R)
    return (n ** 0.5) * (Q @ Ur) @ Vh, S, mu, (n ** 0.5) * (Vh.T / S) @ Vh


def _input(n, m, kind, seed):
    g = _gen(seed)
    G = torch.randn((n, m), generator=g, device="cuda", dtype=torch.float64)
    off, scale = KINDS[kind]
    if scale == "near":  # a standardized matrix plus 1e-2 noise: what every solver retraction sees
        P = _polar64(G.float())[0]
        return (P + 1e-2 * torch.randn((n, m), generator=g, device="cuda", dtype=torch.float64)).float()
    if scale == "cond":  # cond(X_c) = 1e3 along random directions
        Qm, _ = torch.linalg.qr(torch.randn((m, m), generator=g, device="cuda", dtype=torch.float64))
        X = (G * torch.logspace(0, -3, m, device="cuda", dtype=torch.float64)) @ Qm
    elif scale == "log":
        X = G * torch.logspace(0, -2, m, device="cuda", dtype=torch.float64)
    else:
        X = G
    return (X + off * X.std(0)).float()


def _ulp32(x):
    a = x.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def _check_retraction(X, label):
    pm = _pm()
    n, m = X.shape
    ref, S, mu, W = _polar64(X)
    kappa = float(S.max() / S.min())
    Y = pm.Standardized().project_onto_constraint(X.clone(), inplace=True)
    assert bool(torch.isfinite(Y).all()), label
    Y64 = Y.double()
    a = float((_ulp32(mu) @ W.abs()).max())
    err_c = float((Y64.T @ Y64 / n - torch.eye(m, device="cuda", dtype=torch.float64)).abs().max())
    err_mu = float(Y64.mean(0).abs().max())
    err_y = float((Y64 - ref).abs().max())
    bound_c = 2e-5 if kappa <= 200.0 else 1e-2 * (kappa / 1000.0) ** 2
    msg = "%s: cond %.3g, constraint %.3g (bound %.3g), mean %.3g (bound %.3g), |Y - Y_ref| %.3g (bound %.3g)" % (
        label, kappa, err_c, bound_c, err_mu, 1e-5 + a, err_y, 1e-4 * kappa + a)
    assert err_c <= bound_c, msg
    assert err_mu <= 1e-5 + a, msg
    assert err_y <= 1e-4 * kappa + a, msg
    return err_c


def _check_tangent(n, m, seed):
    pm = _pm()
    X = _polar64(_input(n, m, "scaled10", seed))[0].float()
    g = _gen(seed + 1)
    R = torch.randn((m, m), generator=g, device="cuda") / m ** 0.5
    Z = (X @ R + 0.5 * torch.randn((n, m), generator=g, device="cuda")).contiguous()
    T = pm.Standardized().project_onto_tangent_space(X, Z, inplace=False)
    X64, Z64, T64 = X.double(), Z.double(), T.double()
    Tref = Z64 - X64 @ (Z64.T @ X64) / n
    zmax = float(Z64.abs().max())
    err = float((T64 - Tref).abs().max())
    assert err <= 2e-5 * zmax, "m %d n %d: |T - T_ref| %.3g, max |Z| %.3g" % (m, n, err, zmax)
    skew = float((X64.T @ T64 + T64.T @ X64).abs().max() / n)
    assert skew <= 1e-5 * zmax, "m %d n %d: |X^T T + T^T X| / n %.3g, max |Z| %.3g" % (m, n, skew, zmax)


@gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("m", WIDTHS)
def test_retraction_matches_fp64_polar_factor(m, kind):
    _check_retraction(_input(20000, m, kind, 1000 * m + len(kind)), "m %d %s" % (m, kind))


@gpu
@pytest.mark.parametrize("kind", ["off1000", "scaled10"])
@pytest.mark.parametrize("m,n", CAPS)
def test_retraction_across_grid_caps(m, n, kind):
    _check_retraction(_input(n, m, kind, n + m), "m %d n %d %s" % (m, n, kind))


@gpu
@pytest.mark.parametrize("kind", ["off1000", "scaled10"])
def test_retraction_flushes_fp32_partials_at_4_4m_rows(kind):
    """n > 64 x 264 x 256: every thread of the m <= 4 moments kernel passes its 64-row fp32 flush."""
    _check_retraction(_input(4_400_000, 2, kind, 7), "m 2 n 4.4M %s" % kind)


@gpu
@pytest.mark.parametrize("m", WIDTHS)
def test_tangent_matches_fp64(m):
    _check_tangent(20000, m, 50 + m)


@gpu
@pytest.mark.parametrize("m,n", CAPS)
def test_tangent_across_grid_caps(m, n):
    _check_tangent(n, m, n + 3 * m)


@gpu
@pytest.mark.parametrize("m", [300, 1000])
@pytest.mark.parametrize("n", [2112, 20000])
def test_centered_wide_removes_a_large_offset(m, n):
    """colsum_wide_kernel's column-block loop (m > 256) on columns 1e4 standard deviations off-centre."""
    pm = _pm()
    g = _gen(m + n)
    X = (torch.randn((n, m), generator=g, device="cuda", dtype=torch.float64) + 1e4).float()
    C = pm.Centered().project_onto_constraint(X.clone(), inplace=True)
    mu = X.double().mean(0)
    ref = X.double() - mu
    a = float(_ulp32(mu).max())  # the mean is subtracted in fp32
    err = float((C.double() - ref).abs().max())
    assert err <= 1e-5 + a, "m %d n %d: |C - C_ref| %.3g, ulp of the mean %.3g" % (m, n, err, a)


def _rank_deficient_cases():
    cases = []
    for m in [1, 2, 4, 5, 32, 33, 64, 65, 256, 257]:
        cases.append((m, 1000, "constant"))
        if m >= 2:
            cases.append((m, 1000, "duplicate"))
        for n in sorted({2, m - 1, m}):
            if 1 <= n <= m:
                cases.append((m, n, "rows"))
    return cases


@gpu
@pytest.mark.parametrize("m,n,what", _rank_deficient_cases())
def test_rank_deficient_input_raises(m, n, what):
    """A constant column, a duplicated column or n <= m rows leave the de-meaned matrix without full column rank: the
    retraction raises SolverError instead of returning a W of a singular Gram."""
    pm = _pm()
    g = _gen(m * 7 + n)
    X = torch.randn((n, m), generator=g, device="cuda") + 10.0
    if what == "constant":
        X[:, m // 2] = 3.7
    elif what == "duplicate":
        X[:, m - 1] = X[:, 0]
    with pytest.raises(pm.util.SolverError):
        pm.Standardized().project_onto_constraint(X.contiguous(), inplace=False)
    # the workspace does not keep the error: a full-rank matrix of the same width projects again
    if n > m:
        _check_retraction(_input(n, m, "off10", n), "m %d after a rank-deficient call" % m)


@gpu
@pytest.mark.parametrize("m", [64, 256])
def test_newton_schulz_limits(m):
    """cond(X_c) = 1e3 (cond of the Gram 1e6) converges within the 24 iterations; at cond(X_c) = 1e4 the chain gives
    up, and the retraction says so instead of returning an unconverged W."""
    pm = _pm()
    _check_retraction(_input(20000, m, "cond1e3", m), "m %d cond 1e3" % m)
    g = _gen(m + 1)
    Qm, _ = torch.linalg.qr(torch.randn((m, m), generator=g, device="cuda", dtype=torch.float64))
    X = (torch.randn((20000, m), generator=g, device="cuda", dtype=torch.float64)
         * torch.logspace(0, -4, m, device="cuda", dtype=torch.float64)) @ Qm
    with pytest.raises(pm.util.SolverError):
        pm.Standardized().project_onto_constraint(X.float().contiguous(), inplace=False)


@gpu
@pytest.mark.parametrize("m", [2, 8, 48])
def test_embed_from_an_off_centre_start_follows_the_oracle(m):
    """mde.embed from X0 = 50 + N(0, 1) diag(logspace(0, -2)): the device solver retracts X0 first, so its losses
    follow the fp32 oracle (fp64 SVD retraction) only when that retraction is accurate."""
    pm = _pm()
    from tests.test_gpu_solver import _knn_problem
    n = 600
    _, edges, w = _knn_problem(pm, n, 6, 2, 5, pm.Centered())
    f = pm.penalties.Quadratic(torch.tensor(np.abs(w), device="cuda"))
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, pm.Standardized())
    rng = np.random.default_rng(m)
    X0 = (50.0 + rng.standard_normal((n, m)) * np.logspace(0, -2, m)).astype(np.float32)
    X = mde.embed(X=torch.tensor(X0, device="cuda"), max_iter=5)
    spec = O.FnSpec(O.P_QUADRATIC, np.abs(w).astype(np.float32), (0, 0, 0))
    _, st = O.embed(X0, edges, spec, O.Standardized(), max_iter=5, dtype=np.float32)
    ours = mde.solve_stats.average_distortions
    k = min(len(ours), len(st.average_distortions))
    assert k >= 2
    np.testing.assert_allclose(ours[:k], st.average_distortions[:k], rtol=1e-4)
    X64 = X.double()
    np.testing.assert_allclose((X64.T @ X64 / n).cpu().numpy(), np.eye(m), atol=2e-5)
    np.testing.assert_allclose(X64.mean(0).cpu().numpy(), 0, atol=1e-5)


def _gram_retraction_error(X, shift):
    """Constraint error of the polar factor from a Gram of fp32 products summed in fp64 (no other rounding).
    shift=False: products of the uncentred rows, G_c = G - n mu mu^T.  shift=True: products of X - s with the
    kernels' shift s = X[0] + mean(X[:32] - X[0]), G_c = G_s - n (mu - s)(mu - s)^T."""
    n, m = X.shape
    s = (X[0] + (X[1:32] - X[0]).sum(0, dtype=np.float32) / np.float32(32)).astype(np.float32)
    Xs = (X - s).astype(np.float32) if shift else X
    G = np.zeros((m, m))
    for r in range(0, n, 2000):
        B = Xs[r:r + 2000]
        G += (B[:, :, None] * B[:, None, :]).sum(0, dtype=np.float64)
    d = Xs.sum(0, dtype=np.float64) / n
    lam, V = np.linalg.eigh(G - n * np.outer(d, d))
    W = np.sqrt(n) * (V / np.sqrt(lam)) @ V.T
    Y = (X.astype(np.float64) - X.mean(0, dtype=np.float64)) @ W
    return np.abs(Y.T @ Y / n - np.eye(m)).max()


@pytest.mark.parametrize("n,m,offset,scales", [
    (1000, 2, 50.0, (1.0, 1e-2)),
    (1000, 3, 1000.0, (1.0, 1.0, 1.0)),
    (20000, 64, 1000.0, (1.0,) * 64),
])
def test_off_centre_inputs_separate_the_gram_formulas(n, m, offset, scales):
    """The off-centre inputs of the retraction tests above defeat a Gram of uncentred rows: n mu mu^T cancels most of
    its fp32 digits, and the constraint error passes the 2e-5 bound.  Shifting the rows first meets it."""
    rng = np.random.default_rng(n + m)
    X = (offset + rng.standard_normal((n, m)) * np.array(scales)).astype(np.float32)
    assert _gram_retraction_error(X, shift=False) > 2e-5
    assert _gram_retraction_error(X, shift=True) <= 2e-5
