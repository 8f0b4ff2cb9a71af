"""The Standardized constraint at 256 < m <= 1024 on the device (csrc/mde_project_wide.cu: 128 x 128 tiles of the Gram
and row products, the Newton-Schulz products on the fp64 tensor cores), against the fp64 polar factor and tangent
projection of tests/test_gpu_projections.py, with that file's inputs and bounds.

Widths straddle the 128-wide tiles of both products (384/385 via 320 and 511-513, 576/577, 704/705, 767, 1000,
1024).  Row counts straddle the caps of the Gram split (256 rows per row block until 264 / tiles^2 blocks, at least
16, are reached: n = 7424 at m = 300, 4096 at m = 512 and 1024), the row product's chunks (14 336 rows at m = 300,
8192 at m = 512, 16 384 at m = 1024) and 16 896 rows, plus n = m + 2, n = 2m, and n = 1 050 000 at m = 512, whose
row blocks sum 65 632 rows each in one fp32 run, the longest run any width reaches for that n."""
import numpy as np
import pytest
import torch

from tests.test_gpu_projections import KINDS, _check_retraction, _check_tangent, _gen, _input, _polar64

from tests import lbfgs_replay as L

pytestmark = pytest.mark.gpu

XWIDE = [257, 300, 320, 511, 512, 513, 576, 577, 704, 705, 767, 1000, 1024]
# (m, n): both sides of each grid cap, then n = m + 2 and n = 2m
CAPS = ([(300, c + d) for c in (7424, 14336, 16896) for d in (-1, 0, 1)]
        + [(m, c + d) for m, cs in ((512, (4096, 8192, 16896)), (1024, (4096, 16384, 16896))) for c in cs
           for d in (-1, 0, 1)]
        + [(m, m + 2) for m in (257, 512, 1024)] + [(m, 2 * m) for m in (257, 512, 1024)])


def _pm():
    import pymde_b200 as pm
    return pm


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("m", XWIDE)
def test_retraction_matches_fp64_polar_factor(m, kind):
    _check_retraction(_input(20000, m, kind, 1000 * m + len(kind)), "m %d %s" % (m, kind))


@pytest.mark.parametrize("m", XWIDE)
def test_tangent_matches_fp64(m):
    _check_tangent(20000, m, 50 + m)


@pytest.mark.parametrize("kind", ["off1000", "scaled10"])
@pytest.mark.parametrize("m,n", CAPS)
def test_retraction_across_grid_caps(m, n, kind):
    """n = m + 2 leaves a nearly square X_c, whose conditioning can pass what the Newton-Schulz chain reaches
    (about 1e3.5): there the retraction must either meet the bounds or raise SolverError, never return a wrong X."""
    X = _input(n, m, kind, n + m)
    label = "m %d n %d %s" % (m, n, kind)
    if n > m + 2:
        _check_retraction(X, label)
        return
    pm = _pm()
    S = _polar64(X)[1]
    kappa = float(S.max() / S.min())
    try:
        pm.Standardized().project_onto_constraint(X.clone(), inplace=False)
    except pm.util.SolverError:
        assert kappa > 1e3, "%s: SolverError at cond %.3g" % (label, kappa)
        return
    _check_retraction(X, label)


@pytest.mark.parametrize("m,n", CAPS)
def test_tangent_across_grid_caps(m, n):
    _check_tangent(n, m, n + 3 * m)


def test_retraction_longest_fp32_run_at_1m_rows():
    """n = 1 050 000 at m = 512: 16 row blocks of 65 632 rows, each summed in one fp32 run per Gram element."""
    _check_retraction(_input(1_050_000, 512, "off1000", 11), "m 512 n 1.05M off1000")


def _rank_deficient_cases():
    cases = []
    for m in [257, 512, 1024]:
        cases += [(m, 4 * m, "constant"), (m, 4 * m, "duplicate")]
        cases += [(m, n, "rows") for n in (2, m - 1, m)]
    return cases


@pytest.mark.parametrize("m,n,what", _rank_deficient_cases())
def test_rank_deficient_input_raises(m, n, what):
    """A constant column, a duplicated column or n <= m rows: SolverError, and the next full-rank call on the same
    workspace projects correctly."""
    pm = _pm()
    g = _gen(m * 7 + n)
    X = torch.randn((n, m), generator=g, device="cuda") + 10.0
    if what == "constant":
        X[:, m // 2] = 3.7
    elif what == "duplicate":
        X[:, m - 1] = X[:, 0]
    with pytest.raises(pm.util.SolverError):
        pm.Standardized().project_onto_constraint(X.contiguous(), inplace=False)
    _check_retraction(_input(4 * m, m, "off10", n), "m %d after a rank-deficient call" % m)


@pytest.mark.parametrize("m", [512, 1024])
def test_newton_schulz_limits(m):
    """cond(X_c) = 1e3 converges within the 24 iterations (c = ||A||_inf: 23 of them in fp64 at these widths, as at
    m = 256); cond(X_c) = 1e4 raises SolverError."""
    pm = _pm()
    _check_retraction(_input(20000, m, "cond1e3", m), "m %d cond 1e3" % m)
    g = _gen(m + 1)
    Qm, _ = torch.linalg.qr(torch.randn((m, m), generator=g, device="cuda", dtype=torch.float64))
    X = (torch.randn((20000, m), generator=g, device="cuda", dtype=torch.float64)
         * torch.logspace(0, -4, m, device="cuda", dtype=torch.float64)) @ Qm
    with pytest.raises(pm.util.SolverError):
        pm.Standardized().project_onto_constraint(X.float().contiguous(), inplace=False)


def _tiny_mde(m):
    pm = _pm()
    n = 64
    i = torch.arange(n, device="cuda")
    edges = torch.stack([i, (i + 1) % n], 1)
    f = pm.penalties.Quadratic(torch.ones(n, device="cuda"))
    return pm.MDE(n, m, edges, f, pm.Standardized())


def test_solver_takes_the_new_widths():
    """Standardized no longer decides: the evaluation kernels' caps do (m % 4 == 0 up to 1024, else up to 512)."""
    pm = _pm()
    for m in (260, 300, 512, 1024):
        assert _tiny_mde(m)._fused_ok(pm.Standardized(), 10), m
    assert not _tiny_mde(514)._fused_ok(pm.Standardized(), 10)


# The replay's tolerances (lbfgs_replay.TOL) come from cases of m <= 40.  Distances, gradient rows and the
# projections' products here are fp32 sums over m terms, whose rounding grows like sqrt(m): the tolerances of the
# quantities built from them are widened by sqrt(512 / 32) = 4.  The bitwise and rule checks stay exact.
WIDE_TOL = {k: 4.0 * v for k, v in L.TOL.items() if k in ("direction", "move", "average", "residual", "gradient",
                                                          "percent")}


@pytest.mark.parametrize("m", [300, 512])
def test_embed_replays_against_fp64(m):
    """The device solver, paused after every iteration, against the fp64 replay (tests/lbfgs_replay.py):
    Standardized, PushAndPull(Log1p, Log) with weights +-10, n = 3000, memory 10, 32 iterations.  At weights +-1 every
    candidate pair fails the curvature test (y.s <= 1e-10) at these widths; at +-10 the pairs are accepted and the
    history wraps, so the two-loop recursion runs on a full history."""
    from tests.test_gpu_lbfgs_replay import _case, paused_solve
    mde, X0, prob = _case("standardized", m, 10.0)
    assert mde._fused_ok(mde.constraint, 10)
    pauses, stats = paused_solve(mde, X0, 10, 32)
    R = L.replay(pauses, stats, prob, 10, tol=WIDE_TOL)
    assert R.evicted >= 1, (R.accepted, R.rejected, R.evicted, R.resets)


def test_laplacian_embedding_300_ends_on_the_device_solver():
    pm = _pm()
    rng = np.random.default_rng(3)
    data = torch.tensor(rng.standard_normal((1500, 12)).astype(np.float32), device="cuda")
    mde = pm.laplacian_embedding(data, embedding_dim=300, n_neighbors=15)
    assert mde._fused_ok(mde.constraint, 10)
    X = mde.embed(max_iter=40)
    assert mde.__dict__["_device_solver"] is not None
    assert mde.solve_stats.iterations >= 1
    n = X.shape[0]
    X64 = X.double()
    err_c = float((X64.T @ X64 / n - torch.eye(300, device="cuda", dtype=torch.float64)).abs().max())
    assert err_c <= 2e-5, err_c
    assert float(X64.mean(0).abs().max()) <= 1e-5
