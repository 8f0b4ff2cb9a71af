"""A numpy emulation of deterministic mode's fixed-point gradient at m <= 4 (csrc/mde_edges.cu: distortion_quad_kernel
with `fx` set, red_row_fx, fx_apply_kernel), and the per-entry error bound it obeys.

The kernel walks the layout's sorted edges (canonical (min, max) endpoints sorted by (class, src, dst)) four at a time.
Every edge's fp32 contribution v is added at src and subtracted at dst, one term at each end.  A scan pass finds every
row's largest finite |v| over its edges, M_r < 2^eM_r, and the row's power-of-two scale is 2^S_r,
S_r = 61 - ceil(log2(deg_r)) - eM_r.  Every term t is rounded to the integer round(t 2^S_r) (to nearest, ties to even,
in double: t 2^S_r is exact there) and added into an int64 per entry.  The result is fl32(fl64(F) 2^-S_r); a
non-finite term makes its entry NaN.

`old_accumulate` is the accumulator this replaced: a fixed scale 2^40 applied in fp32, a conversion that clamps to the
int64 range and maps NaN to 0, and int64 sums that wrap."""
import numpy as np

U = 2.0 ** -24
HEADROOM = 61


def sort_edges(edges, cls=None):
    """(order, src, dst): the layout's sorted edges; duplicates keep their input order (a stable radix sort)."""
    e = np.asarray(edges, np.int64)
    lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
    c = np.zeros(len(e), np.int64) if cls is None else np.asarray(cls, np.int64)
    order = np.lexsort((np.arange(len(e)), hi, lo, c))
    return order, lo[order], hi[order]


def external_contributions(X, src, dst, g):
    """v = fl(g fl(x_src - x_dst)) of the sorted edges: the kernel's own floats for external coefficients g."""
    X = np.asarray(X, np.float32)
    return (np.asarray(g, np.float32)[:, None] * (X[src] - X[dst])).astype(np.float32)


def terms(src, dst, v):
    """(rows, values) of every term the kernel adds: v at src, -v at dst"""
    return np.concatenate([src, dst]), np.concatenate([v, -v])


def lg_degree(src, dst, n):
    """ceil(log2(deg)) of every row (0 for degrees 0 and 1)"""
    deg = np.bincount(np.r_[src, dst], minlength=n)
    return np.ceil(np.log2(np.maximum(deg, 1))).astype(np.int64)


def scale_exponent(src, dst, v, lgdeg):
    """S_r of every row: the scan's largest finite |v| over the row's edges, as fp32 bits, M_r < 2^eM_r"""
    a = np.where(np.isfinite(v), np.abs(v), 0).astype(np.float32).max(axis=1).view(np.uint32).astype(np.int64)
    bits = np.zeros(len(lgdeg), np.int64)
    np.maximum.at(bits, src, a)
    np.maximum.at(bits, dst, a)
    em = np.maximum(bits >> 23, 1) - 126
    return HEADROOM - lgdeg - em


def accumulate(n, rows, vals, S):
    """(F, nan): the int64 sums (exact: the scale keeps every partial sum below 2^62) and the entries a non-finite term
    turned into NaN."""
    m = vals.shape[1]
    fin = np.isfinite(vals)
    q = np.rint(np.where(fin, vals, 0).astype(np.float64) * 2.0 ** S[rows][:, None]).astype(np.int64)
    F = np.zeros((n, m), np.int64)
    np.add.at(F, rows, q)
    nan = np.zeros((n, m), bool)
    np.logical_or.at(nan, rows, ~fin)
    return F, nan


def finish(F, nan, S):
    g = (F.astype(np.float64) * 2.0 ** -S[:, None]).astype(np.float32)
    g[nan] = np.nan
    return g


def gradient(X, edges, g, cls=None):
    """The deterministic kernel's gradient of the external coefficients g (original edge order), bit for bit, and
    the rows' S."""
    X = np.asarray(X, np.float32)
    order, src, dst = sort_edges(edges, cls)
    v = external_contributions(X, src, dst, np.asarray(g, np.float32)[order])
    rows, vals = terms(src, dst, v)
    S = scale_exponent(src, dst, v, lg_degree(src, dst, len(X)))
    F, nan = accumulate(len(X), rows, vals, S)
    return finish(F, nan, S), S


def old_accumulate(n, rows, vals):
    """The fixed 2^40 accumulator: fp32 scaling, clamped conversion (NaN -> 0), wrapping int64 sums."""
    x = (vals * np.float32(2.0 ** 40)).astype(np.float64)
    big = 2.0 ** 63
    q = np.rint(np.where(np.isfinite(x) & (np.abs(x) < big), x, 0.0)).astype(np.int64)
    q = np.where(x >= big, np.iinfo(np.int64).max, q)
    q = np.where(x < -big, np.iinfo(np.int64).min, q)
    F = np.zeros((n, vals.shape[1]), np.int64)
    with np.errstate(over="ignore"):
        np.add.at(F, rows, q)
    return (F.astype(np.float64) * 2.0 ** -40).astype(np.float32)


def bound(n, rows, exact_abs, deg, v_rel, S, result):
    """Per-entry bound on |kernel - exact| from the terms the kernel adds:

      contributions   v_rel |v*| per edge, v* the exact contribution (`exact_abs` holds sum |v*| per entry, every edge
                      at both of its ends): for external coefficients fl(g fl(x_s - x_d)) is 2 u + u^2;
      rounding        every term is rounded to its row's quantum 2^-S_r: half a quantum per term;
      final           fl64(F) and fl32(.) round once each: (u + 2^-53) |F 2^-S|;
      reference       the fp64 scatter of v* (deg additions at each end): (deg + 2) 2^-53 sum |v*|."""
    nterms = np.bincount(rows, minlength=n).astype(np.float64)
    B = (v_rel + (np.asarray(deg, np.float64)[:, None] + 2) * 2.0 ** -53) * exact_abs
    B += (nterms * 2.0 ** -(S + 1.0))[:, None]
    B += (U + 2.0 ** -53) * np.abs(result.astype(np.float64))
    return B


def exact_scatter(X, edges, g):
    """(gradient, sum |v*| per entry) of the exact contributions g (x_i - x_j), in fp64."""
    X = np.asarray(X, np.float64)
    e = np.asarray(edges, np.int64)
    v = np.asarray(g, np.float64)[:, None] * (X[e[:, 0]] - X[e[:, 1]])
    n, m = X.shape
    G = np.zeros((n, m))
    A = np.zeros((n, m))
    for c in range(m):
        G[:, c] = np.bincount(e[:, 0], weights=v[:, c], minlength=n) - np.bincount(e[:, 1], weights=v[:, c], minlength=n)
        A[:, c] = np.bincount(e.ravel(), weights=np.abs(np.repeat(v[:, c], 2)), minlength=n)
    return G, A
