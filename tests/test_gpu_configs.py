"""Driver-visible parity at the sizes BASELINE.json names (VERDICT r01 row N1 / item 3):

  C2 slice  n = 20 000, 444 024 edges, PushAndPull(Log1p, Log): reference-generated fixture (tests/golden/c2slice.npz:
            runs of the unmodified reference to convergence with 1 / 4 / 8 threads, and 300 non-converged iterations)
  C3 shape  n = 44 682, 2e7 sampled pairs, losses.Huber, Standardized          -- value + gradient vs the C oracle
  C4 slice  n = 200 000, m = 128, 3e6 edges, PushAndPull (wide kernel)          -- value + gradient vs the C oracle
  C5 shape  n = 1e7, 5e7 SBM edges, PushAndPull (tile layouts, super-tiles)     -- value + gradient vs the C oracle
Tolerances: value 1e-5 relative (north_star), gradient 3e-5 of its largest entry (fp32 sums of up to 1e3 terms)."""
import hashlib
import os

import numpy as np
import pytest
import torch

import bench
from oracle import c_oracle, mde_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check_against_oracle(mde, X, edges_np, spec, value_rtol=1e-5, grad_tol=3e-5):
    Xg = X.clone().requires_grad_(True)
    v = mde.average_distortion(Xg)
    v.backward()
    v_ref, g_ref = c_oracle.average_distortion(X.cpu().numpy(), edges_np, spec, True)
    np.testing.assert_allclose(v.item(), v_ref, rtol=value_rtol)
    err = np.abs(Xg.grad.cpu().numpy().astype(np.float64) - g_ref).max()
    assert err <= grad_tol * np.abs(g_ref).max(), (err, np.abs(g_ref).max())
    return v.item(), v_ref


# --------------------------------------------------------------------------------------- C2 slice
@pytest.fixture(scope="module")
def c2slice(golden):
    g = golden["c2slice"]
    edges, w = bench.c2_edges(0, n=20000, k=15)
    sha = np.frombuffer(hashlib.sha1(edges.tobytes() + w.tobytes()).digest(), dtype=np.uint8)
    if len(edges) != int(g["n_edges"]) or not np.array_equal(sha, g["edges_sha1"]):
        pytest.fail("bench.c2_edges no longer reproduces the edge list the fixture was generated on")
    return g, edges, w


def _inside_reference_envelope(ours, runs, k):
    """First k iterations: ours must lie inside the band spanned by the reference's own runs (different thread
    counts => different fp32 summation order), widened by the band's width and 1e-5 relative.  On this problem the
    reference's 1- and 8-thread runs already differ by 2e-4 at iteration 1 and by 11 % at iteration 4."""
    runs = np.stack([np.asarray(r[:k], dtype=np.float64) for r in runs])
    lo, hi = runs.min(0), runs.max(0)
    width = (hi - lo) + 1e-5 * np.abs(hi)
    a = np.asarray(ours[:k], dtype=np.float64)
    assert np.all(a >= lo - width) and np.all(a <= hi + width), (a, lo, hi)


def _c2_mde(pm, edges, w, constraint):
    wt = torch.tensor(w, device=DEV)
    return pm.MDE(20000, 2, torch.tensor(edges, device=DEV), pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log),
                  constraint, device=DEV)


def test_c2slice_value_and_stationarity_at_the_reference_optimum(c2slice):
    """At the embedding the REFERENCE converged to: same objective value to 1e-5, and our projected gradient is as
    small as the reference's stopping residual -- the two implementations agree on what a solution is."""
    import pymde_b200 as pm
    g, edges, w = c2slice
    mde = _c2_mde(pm, edges, w, pm.Standardized())
    Xr = torch.tensor(g["std/t8/X"], device=DEV)
    np.testing.assert_allclose(mde.average_distortion(Xr).item(), float(g["std/t8/final_value"]), rtol=1e-5)
    Xg = Xr.clone().requires_grad_(True)
    mde.average_distortion(Xg).backward()
    proj = pm.Standardized().project_onto_tangent_space(Xr, Xg.grad, inplace=False)
    assert float(proj.norm()) < 5e-5  # the reference stopped at <= 1e-5 with ITS fp32 gradient


def test_c2slice_converged_value_within_the_references_own_spread(c2slice):
    import pymde_b200 as pm
    g, edges, w = c2slice
    mde = _c2_mde(pm, edges, w, pm.Standardized())
    X0 = torch.tensor(g["std/X0"], device=DEV)
    X = mde.embed(X=X0, eps=1e-5, max_iter=1500)
    st = mde.solve_stats
    assert st.iterations < 1500 and st.residual_norms[-1] <= 1e-5  # converged like the reference (578-882 iterations)
    # iteration 0 is a plain evaluation: 1e-5; the first iterations follow the reference
    ref8 = g["std/t8/average_distortions"]
    np.testing.assert_allclose(st.average_distortions[0], ref8[0], rtol=1e-5)
    _inside_reference_envelope(st.average_distortions, [g["std/t%d/average_distortions" % t] for t in (1, 4, 8)], 6)
    # the objective is non-convex: the reference itself lands on different stationary points with 1 / 4 / 8 threads
    refs = np.array([float(g["std/t%d/final_value" % t]) for t in (1, 4, 8)])
    spread = refs.max() - refs.min()
    assert spread > 1e-5 * refs.mean()  # (documents why a 1e-5 comparison of end points is not defined here)
    final = mde.average_distortion(X).item()
    # not worse than the reference's own worst run (it may be better), and the
    # same basin: within 2 % of the reference's best
    assert final <= refs.max() + 2 * spread, (final, refs)
    assert final >= 0.98 * refs.min(), (final, refs)


def test_c2slice_300_iterations_centered(c2slice):
    import pymde_b200 as pm
    g, edges, w = c2slice
    mde = _c2_mde(pm, edges, w, pm.Centered())
    mde.embed(X=torch.tensor(g["cen/X0"], device=DEV), eps=1e-5, max_iter=300)
    a = np.array(mde.solve_stats.average_distortions)
    r8, r1 = g["cen/t8/average_distortions"], g["cen/t1/average_distortions"]
    assert len(a) == 300
    np.testing.assert_allclose(a[0], r8[0], rtol=1e-5)
    np.testing.assert_allclose(mde.solve_stats.residual_norms[0], g["cen/t8/residual_norms"][0], rtol=1e-4)
    _inside_reference_envelope(a, [r8, r1], 4)  # (from iteration 4 on the two reference runs cross each other)
    # after 300 iterations the reference's two runs differ by several percent; ours must be as good a descent
    lo, hi = min(r8[-1], r1[-1]), max(r8[-1], r1[-1])
    assert a[-1] <= hi + 2 * (hi - lo), (a[-1], lo, hi)
    assert a[-1] >= lo - 2 * (hi - lo), (a[-1], lo, hi)


# --------------------------------------------------------------------------------------- C3 / C4 / C5 shapes
def test_c3_shape_huber_standardized_2e7_edges():
    import pymde_b200 as pm
    n, m, p = 44682, 2, 20_000_000
    gen = torch.Generator(device=DEV)
    gen.manual_seed(0)
    e = torch.randint(0, n, (p, 2), device=DEV, generator=gen)
    e = e[e[:, 0] != e[:, 1]]
    delta = torch.randint(1, 9, (e.shape[0],), device=DEV, generator=gen).float()
    delta = pm.preprocess.scale(delta, pm.Standardized().natural_length(n, m))
    mde = pm.MDE(n, m, e, pm.losses.Huber(delta, 0.5), pm.Standardized(), device=DEV)
    X = torch.randn(n, m, device=DEV, generator=gen)
    X = pm.Standardized().project_onto_constraint(X, inplace=True)
    spec = O.FnSpec(O.L_HUBER, delta.cpu().numpy(), (0.5, 0, 0))
    _check_against_oracle(mde, X, e.cpu().numpy(), spec)
    from pymde_b200 import _lib
    assert _lib.load().mde_edges_kind(mde._layout().handle) == 3  # dense graph: sorted SoA + ELL pull records
    mde.embed(X=X, max_iter=6, eps=0.0)  # the device solver runs at this size (Gram + Jacobi retraction)
    st = mde.solve_stats
    assert st.iterations == 6 and st.average_distortions[-1] < st.average_distortions[0]
    Xe = mde.X
    np.testing.assert_allclose((Xe.T @ Xe / n).cpu().numpy(), np.eye(m), atol=5e-4)


def test_c4_slice_m128_wide_kernel():
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
    X = torch.randn(n, m, device=DEV, generator=gen)
    X -= X.mean(0)
    spec = O.FnSpec(O.P_LOG1P, w.cpu().numpy(), (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    _check_against_oracle(mde, X, e.cpu().numpy(), spec)


@pytest.mark.parametrize("layout", [None, "soa"])
def test_c5_shape_1e7_nodes(layout, monkeypatch):
    import pymde_b200 as pm
    if layout:
        monkeypatch.setenv("MDE_B200_LAYOUT", layout)
    n, m = 10_000_000, 2
    edges, w = bench.c5_shard(0, n=n, p=50_000_000)
    e = torch.tensor(edges, device=DEV)
    wt = torch.tensor(w, device=DEV)
    mde = pm.MDE(n, m, e, pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log), pm.Centered(), device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(2)
    X = torch.randn(n, m, device=DEV, generator=gen)
    X -= X.mean(0)
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    _check_against_oracle(mde, X, edges, spec)
    # size-independent properties: the gradient of a translation-invariant objective sums to zero per column
    Xg = X.clone().requires_grad_(True)
    mde.average_distortion(Xg).backward()
    assert float(Xg.grad.double().sum(0).abs().max()) < 1e-6
