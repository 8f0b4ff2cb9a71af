"""Why deterministic mode's fixed-point gradient at m <= 4 picks its scale per evaluation, on the CPU.

The emulation in tests/det_fx.py follows the kernel term by term (fp32 contributions added at both ends, round to
nearest at the row's scale, int64 sums, one final conversion); `old_accumulate` applies the fixed scale 2^40 the kernel
used before to the same terms.  It reproduces what that fixed scale did wrong:

- resolution: the quantum 2^-40 is absolute while the contributions scale like f'/p, so the gradient's error grew
  with the edge count and passed the fp32 sum's at about 10^6 edges;
- range: an int64 at 2^40 holds +-2^23; a term beyond it was clamped and a row sum beyond it wrapped, both into a
  wrong finite gradient;
- non-finite input: the conversion maps NaN to 0, so a NaN contribution vanished.

With a scale per row, S_r = 61 - ceil(log2(deg_r)) - eM_r (the row's largest finite |v| below 2^eM_r), the row's
deg_r terms sum in magnitude to at most 2^61 (plus half a quantum each) after scaling, so nothing clamps or wraps, and the quantum is at most
2^(ceil(log2 deg_r) - 61) M_r.  The per-entry bound of det_fx.bound (contribution rounding + half a quantum per term +
the final rounding) is checked below on every entry without a safety factor, and shown not to be vacuous."""
import numpy as np
import pytest

from oracle import mde_oracle as O
from tests import det_fx as D
from tests import lbfgs_replay as L

U = D.U


def _pushpull_problem(n, k, m, seed, scale=1.0):
    """A knn_graph problem's external coefficients: g = fl32(f'/(p d)) of PushAndPull(Log1p, Log), in fp64 first."""
    edges, w = L.knn_graph(n, k, seed)
    rng = np.random.default_rng(seed)
    X = (scale * rng.standard_normal((n, m))).astype(np.float32)
    X -= X.mean(0)
    d, _ = O.edge_distances(X.astype(np.float64), edges)
    _, fp = O.eval_function(L.push_pull_spec(w), d)
    with np.errstate(all="ignore"):
        g = fp / (len(edges) * d)
    g[~np.isfinite(g)] = 1.0
    return edges, X, g.astype(np.float32)


def _fp32_sum(X, edges, g):
    """The default mode's kind of gradient: fp32 contributions added in fp32 (edge order)."""
    X = np.asarray(X, np.float32)
    v = g[:, None] * (X[edges[:, 0]] - X[edges[:, 1]])
    G = np.zeros(X.shape, np.float32)
    np.add.at(G, edges[:, 0], v)
    np.add.at(G, edges[:, 1], -v)
    return G


def _run(X, edges, g):
    """(new gradient, old gradient, exact gradient, per-entry bound, S)"""
    n = len(X)
    order, src, dst = D.sort_edges(edges)
    v = D.external_contributions(X, src, dst, g[order])
    rows, vals = D.terms(src, dst, v)
    S = D.scale_exponent(src, dst, v, D.lg_degree(src, dst, n))
    F, nan = D.accumulate(n, rows, vals, S)
    new = D.finish(F, nan, S)
    assert np.all(np.abs(F) < 2 ** 62)
    old = D.old_accumulate(n, rows, vals)
    G, A = D.exact_scatter(X, edges, g)
    deg = np.bincount(np.asarray(edges).ravel(), minlength=n)
    B = D.bound(n, rows, A, deg, 2 * U + U * U, S, new)
    return new, old, G, B, S


def _rel(a, G):
    return float(np.linalg.norm(a.astype(np.float64) - G) / np.linalg.norm(G))


# --------------------------------------------------------------------------------------- resolution
def test_fixed_scale_loses_to_fp32_as_edges_grow():
    """The issue's table at 6e4 and 1.55e6 edges (m = 2, PushAndPull(Log1p, Log), random centred X): the 2^40
    accumulator's relative Frobenius error grows with p and passes the fp32 sum's; the per-evaluation scale stays
    below the fp32 sum's at both sizes (the 1e7 and 5e7 rows are measured on the device, tests/test_gpu_det_fx.py)."""
    errs = []
    for n in (3000, 78_000):
        edges, X, g = _pushpull_problem(n, 10, 2, seed=n)
        new, old, G, _, _ = _run(X, edges, g)
        e_old, e_new, e_32 = _rel(old, G), _rel(new, G), _rel(_fp32_sum(X, edges, g), G)
        assert e_new < e_32 < 2e-7, (len(edges), e_new, e_32)
        errs.append((len(edges), e_old, e_32))
    (p0, old0, f0), (p1, old1, f1) = errs
    assert 5e4 < p0 < 7e4 and 1.4e6 < p1 < 1.7e6
    assert old0 < f0 and old1 > 2 * f1 and old1 > 4 * old0, errs


# --------------------------------------------------------------------------------------- the bound
def _hub_problem(seed, m):
    """Random edges plus a hub of degree 3 000, magnitudes over 12 decades, duplicates and zero-length edges."""
    rng = np.random.default_rng(seed)
    n = 4000
    e = rng.integers(0, n, (30_000, 2))
    e = e[e[:, 0] != e[:, 1]]
    hub = np.stack([np.zeros(3000, np.int64), rng.integers(1, n, 3000)], 1)
    e = np.concatenate([e, hub, e[:50]]).astype(np.int64)
    X = rng.standard_normal((n, m)).astype(np.float32)
    X[e[:20, 1]] = X[e[:20, 0]]
    g = (rng.standard_normal(len(e)) * 10.0 ** rng.uniform(-8, 4, len(e))).astype(np.float32)
    return e, X, g


@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("case", ["pushpull", "hub", "far"])
def test_bound_holds_on_every_entry_and_is_not_vacuous(m, case):
    if case == "pushpull":
        edges, X, g = _pushpull_problem(3000, 8, m, seed=m)
    elif case == "hub":
        edges, X, g = _hub_problem(m, m)
    else:  # coordinates around 1e6, the guard's g = 1: contributions of 1e6..1e7, row sums far beyond 2^23
        edges, X, _ = _pushpull_problem(3000, 8, m, seed=m, scale=3e6)
        g = np.ones(len(edges), np.float32)
    new, old, G, B, S = _run(X, edges, g)
    err = np.abs(new.astype(np.float64) - G)
    assert np.all(err <= B), float(np.max(err / B))
    # not vacuous: the worst entry uses a good part of its bound, and the bound is far below the gradient's scale
    assert np.max(err / B) > 0.2
    assert np.median(B) < 1e-5 * np.abs(G).max()
    if case == "far":
        assert np.abs(G).max() > 2.0 ** 23
        assert not np.all(np.abs(old.astype(np.float64) - G) <= B)  # the 2^40 accumulator wrapped or clamped


def test_quantum_is_relative_to_the_largest_contribution():
    """Scaling every coefficient by 2^k shifts every S_r by -k and leaves the bits of the gradient scaled by 2^k: the
    quantum tracks the contributions, from far below 1 to far above (while every contribution stays a normal float)."""
    edges, X, g = _hub_problem(5, 2)
    base, S0 = D.gradient(X, edges, g)
    for k in (-80, -40, -20, 20, 60, 90):
        got, S = D.gradient(X, edges, (g.astype(np.float64) * 2.0 ** k).astype(np.float32))
        assert np.array_equal(S, S0 - k)
        assert np.array_equal(got.astype(np.float64), base.astype(np.float64) * 2.0 ** k)


# --------------------------------------------------------------------------------------- range and NaN
def _one_row(vals_per_edge, m=1):
    """A star: nodes 0..k-1 joined to the hub k with x_j = 0, x_k = 1 and coefficients vals.  The hub is every
    edge's dst: the hub's terms are the coefficients themselves."""
    k = len(vals_per_edge)
    edges = np.stack([np.arange(k), np.full(k, k)], 1).astype(np.int64)
    X = np.zeros((k + 1, m), np.float32)
    X[k] = 1.0
    return edges, X, np.asarray(vals_per_edge, np.float32)


@pytest.mark.parametrize("kind", ["single_above", "single_below", "sum_above", "sum_below", "hub_wraps"])
def test_range_of_the_fixed_scale(kind):
    """A term and a row sum at 2^23 (1 +- 2^-10), and a hub whose sum crosses the old range with every term inside
    it: the old accumulator clamps or wraps into a wrong finite number; the new one is within the bound."""
    t = 2.0 ** 23
    vals = {"single_above": [t * (1 + 2 ** -10)], "single_below": [t * (1 - 2 ** -10)],
            "sum_above": [t * (1 + 2 ** -10) / 4] * 4, "sum_below": [t * (1 - 2 ** -10) / 4] * 4,
            "hub_wraps": [t / 3] * 7}[kind]
    edges, X, g = _one_row(vals)
    new, old, G, B, _ = _run(X, edges, g)
    assert np.all(np.abs(new - G) <= B)
    old_ok = bool(np.all(np.abs(old.astype(np.float64) - G) <= B))
    assert old_ok == kind.endswith("below"), (kind, old[0], G[0])


def test_non_finite_contributions_turn_their_entries_nan():
    edges, X, g = _one_row([1.0, 2.0, 3.0], m=2)
    g[1] = np.nan
    new, _ = D.gradient(X, edges, g)
    order, src, dst = D.sort_edges(edges)
    v = D.external_contributions(X, src, dst, g[order])
    rows, vals = D.terms(src, dst, v)
    old = D.old_accumulate(len(X), rows, vals)
    assert np.isnan(new[3]).all() and np.isnan(new[1]).all()  # the hub row and the NaN edge's other end
    assert np.all(new[[0, 2]] == [[-1.0, -1.0], [-3.0, -3.0]])
    assert np.isfinite(old).all()  # the 2^40 accumulator dropped the NaN: a wrong finite gradient
    G32 = _fp32_sum(X, edges, g)
    assert np.array_equal(np.isfinite(G32), np.isfinite(new))  # the default mode's outcome
