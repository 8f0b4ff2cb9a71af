"""The fused value-and-gradient kernels row by row: every gradient row against an fp64 sum of the kernel's own edge terms.

The edge-by-edge suite (test_gpu_function_matrix.py) runs on matchings, so it never sees how a row's terms are gathered
and summed; the graph suites (test_gpu_layout_geometry.py) check the gradient with one global tolerance, 3e-5 max|g|,
which the hubs set.  Here every row and column is checked on its own.

A  Terms.  The exploded matching M of a graph G has one edge per edge k = (i, j) of G, joining rows 2k and 2k + 1 with
   X_M[2k] = X[i], X_M[2k + 1] = X[j].  Evaluated on the same layout kind, at the same m, with the same function and
   kernel switch and p_total = p (the same bits of 1/p), d^2, f and g of edge k are the same floats in G and in M, so
   t_k = grad_M[2k] is the kernel's own fp32 term of edge k.  Checked: both ends of M agree bit for bit, every term is
   within the fp64 oracle's range over d (1 +- e) (e = the layout's distance error: (m + 2) u from the fp32 sum of
   squares, 2^-20 on ELL) widened by the per-point tolerances of test_gpu_function_matrix.py (TOL), every row satisfies
       |grad_ic - sum_k s_ik t_kc| <= gamma_(deg_i + 1) sum_k |t_kc|,   gamma_n = n u / (1 - n u),  u = 2^-24
   in fp64 (deg_i - 1 additions and one rounding of each product, which may be fused into the sum), and isolated rows
   are exactly 0.  The MUFU ELL kernel scales a lane-slot's sum by the class constant 1.5 / p or 1 / p after the sum,
   which is one more rounding in the row and one more in each term: gamma_(deg_i + 3) there.
B  Stars.  A hub at small-integer coordinates with neighbours at X[h] +- e_c (d = 1, d^2 = 1) and p a power of two:
   every term at the hub is +-t with a t of at most 3 significant bits (Log1p at d = 1: f' = 0.75 w; the losses and
   the quadratic penalty: dyadic f'), so every partial sum is exact in fp32 whatever the order, and the hub row must be
   t (n- - n+) bit for bit, 0 for balanced stars.  Degrees 1, 2^k - 1, 2^k, 2^k + 1 up to k = 16.  Identical terms of
   24 significant bits do not sum exactly (3 t needs 25), so the repulsive class of PushAndPull (Log: f' = w /
   expm1(d)) is not exact at any d: on those columns the stars get check A's bound only.
C  External coefficients.  Dyadic per-edge g and small-integer X (test_gpu_owner_pass._exact_graph): the scatter is
   exact on every layout kind, on the wide kernel, and at an m other than the layout's own.
D  Exact fused sums.  PushAndPull(Quadratic, Quadratic) with weights +-2^-k, p a power of two and small-integer X:
   g = ((2 w d) (1/p)) / d = 2 w / p exactly, so the fused gradient is the fp64 sum bit for bit on the owner, quad,
   wide, tile and pull kernels.  The ELL kernel forms g with rsqrt.approx: not exact, and not claimed (A and B cover it).
E  The loss.  The same fp32 f enter the loss of G and of M.  The layouts add them in fp64, except the MUFU kernels,
   which add at most 8 consecutive terms of one lane in fp32 first (quad and tile kernels: 4, pull: EPL <= 8, ELL: the
   lane's K W <= 8 entries of a record, in log2 units, each edge once from each end): |S_G - S_M| <= 2 gamma_8 sum |f|,
   else 2 gamma64_p sum |f|.  Value-only evaluations (MODE 1, IEEE math on every layout) are held to the fp64 bound
   against M's; fused, value-only and distortions() to the per-edge function tolerances.

Every case asserts the layout kind and the deterministic flag it built and prints them with the largest
|grad - sum t| / (gamma sum |t|) it saw.  The CPU self-checks at the end run without a GPU."""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O
from tests import test_gpu_layout_geometry as LG
from tests.test_gpu_function_matrix import TOL
from tests.test_gpu_owner_pass import _exact_expected, _exact_graph



def gpu(test):
    """marked gpu, and skipped where no CUDA device is present"""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")(test))


U = 2.0 ** -24
_G1 = dict(LG.GEOMETRIES["G1"][1])


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in LG._ENV:
        monkeypatch.delenv(k, raising=False)


def _setenv(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def gamma(n, u=U):
    n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def _ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


# ------------------------------------------------------------------------------------------------ paths
# path -> (environment, m the layout is built for, m evaluated, kind, deterministic flag)
PATHS = {}
for _m in (1, 2, 3, 4):
    PATHS["owner_m%d" % _m] = ({"MDE_B200_LAYOUT": "soa"}, _m, _m, 0, 0)
    PATHS["tiles_m%d" % _m] = (dict(_G1, MDE_B200_LAYOUT="tiles"), _m, _m, 1, 0)
    PATHS["pull4_m%d" % _m] = (dict(_G1, MDE_B200_LAYOUT="pull", MDE_B200_PULL_EPL="4"), _m, _m, 2, 0)
    PATHS["pull8_m%d" % _m] = (dict(_G1, MDE_B200_LAYOUT="pull", MDE_B200_PULL_EPL="8"), _m, _m, 2, 0)
    PATHS["pullpush_m%d" % _m] = (dict(_G1, MDE_B200_LAYOUT="pull", MDE_B200_PULL_REP="push"), _m, _m, 2, 0)
    PATHS["ell_m%d" % _m] = ({"MDE_B200_LAYOUT": "ell"}, _m, _m, 3, 0)
    PATHS["ellrb8_m%d" % _m] = (dict(_G1, MDE_B200_LAYOUT="ell"), _m, _m, 3, 0)
for _m in (1, 2, 3):  # the quad kernel: a layout built for m = 4 evaluated at another m
    PATHS["quad_m%d" % _m] = ({"MDE_B200_LAYOUT": "soa"}, 4, _m, 0, 0)
    PATHS["quadell_m%d" % _m] = ({"MDE_B200_LAYOUT": "ell"}, 4, _m, 3, 0)
WIDE_M = (5, 8, 13, 27, 36, 61, 100, 125, 200, 255, 400, 511, 512, 1024)  # every launch_wide<G, CPL, VW>
for _m in WIDE_M:
    PATHS["wide_m%d" % _m] = ({"MDE_B200_LAYOUT": "soa"}, _m, _m, 0, 0)
for _m in (5, 16, 33, 257, 512):
    PATHS["wideowner_m%d" % _m] = ({"MDE_B200_DETERMINISTIC": "1"}, _m, _m, 0, 1)


def _graph_of(path):
    """G1 (8155 rows, 32 tiles of 256 under the G1 switches) for every path; G3 (100 000 rows) for kinds 0 and 3 at
    m <= 4; a 3000-row graph for the wide kernels."""
    return "W" if PATHS[path][1] >= 5 else "G1"


# ------------------------------------------------------------------------------------------------ graphs
_GRAPHS = {}


def _problem(geom, m):
    """(n, edges, coincident pairs, isolated rows, X) of G1 / G3 (test_gpu_layout_geometry._graph) or W, plus close
    pairs: ordinary rows moved to 2^-4 .. 2^-16 from a partner they are joined to, so |grad_i| spans many decades."""
    key = (geom, m)
    if key not in _GRAPHS:
        if geom == "W":
            n, bounds, sizes, seed = 3000, (256,), (12000, 1500), 31
            e, co, isolated, hubs = LG._graph(n, bounds, sizes[0], sizes[1], seed=seed, hub_deg=2000)
        else:
            n, _, bounds = LG.GEOMETRIES[geom]
            e, co, isolated, hubs = LG._problem(geom, 1)[1:5]
        rng = np.random.default_rng(1000 + m)
        X = rng.standard_normal((n, m)).astype(np.float32)
        X -= X.mean(0)
        X[co[:, 1]] = X[co[:, 0]]
        used = set(np.concatenate([co.ravel(), hubs, isolated]).tolist())
        cand = np.array([r for r in rng.permutation(n) if r not in used][:26], dtype=np.int64).reshape(13, 2)
        u = rng.standard_normal((13, m))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        X[cand[:, 1]] = (X[cand[:, 0]] + (2.0 ** -np.arange(4, 17))[:, None] * u).astype(np.float32)
        e = np.concatenate([e, cand])
        _GRAPHS[key] = (n, e, co, isolated, X)
    return _GRAPHS[key]


# ------------------------------------------------------------------------------------------------ functions
FNS = ("pp_fast", "pp_precise", "pp_logratio", "huber", "quadratic", "wquad")
_LOSS = ("huber", "quadratic", "wquad")


def _fn_env(name):
    return {"MDE_B200_KERNEL": "precise"} if name == "pp_precise" else {}


def _function(pm, name, p, seed):
    rng = np.random.default_rng(seed)
    w = torch.tensor(rng.choice([1.0, 2.0, -1.0], p).astype(np.float32), device="cuda")
    dev = torch.tensor(rng.uniform(0.5, 2.0, p).astype(np.float32), device="cuda")
    pen, los = pm.penalties, pm.losses
    return {
        "pp_fast": lambda: pen.PushAndPull(w, pen.Log1p, pen.Log),
        "pp_precise": lambda: pen.PushAndPull(w, pen.Log1p, pen.Log),
        "pp_logratio": lambda: pen.PushAndPull(w, pen.Log1p, pen.LogRatio),
        "huber": lambda: los.Huber(dev, 0.5),
        "quadratic": lambda: los.Quadratic(dev),
        "wquad": lambda: los.WeightedQuadratic(dev),
    }[name]()


def _edges_for(name, e, co):
    """coincident rows only for the functions whose f' is finite at d = 0"""
    return np.concatenate([e, co]) if name in _LOSS else e


def _mufu(name, m, kind, m_eval):
    """the MUFU kernels: the recipe default, fused, at m = 2, 3 (owner, quad, tile, pull) or any m <= 4 (ELL)"""
    if name != "pp_fast" or m_eval >= 5:
        return False
    return kind == 3 and m_eval == m or m_eval in (2, 3)


# ------------------------------------------------------------------------------------------------ layouts
def _flags(lay):
    from pymde_b200 import _lib
    lib = _lib.load()
    return int(lib.mde_edges_kind(lay.handle)), int(lib.mde_edges_deterministic(lay.handle))


def _layout(f, edges, n, p_total, m_hint, sl=slice(None)):
    from pymde_b200.problem import EdgeLayout
    table, par0, par1 = f._table()
    par0 = par0.reshape(-1)[sl].contiguous()
    par1 = None if par1 is None else par1.reshape(-1)[sl].contiguous()
    return EdgeLayout(torch.tensor(edges, device="cuda"), n, table, par0, par1, torch.device("cuda", 0),
                      p_total=p_total, embedding_dim=m_hint)


def _chunk_edges(kind, m_hint):
    """ELL pull records address at most 32 neighbour tiles of R rows: M is built 16 R edges at a time"""
    if kind != 3:
        return 1 << 40
    import os
    rb = int(os.environ.get("MDE_B200_TILE_RB", "0"))
    rb = rb if 8 <= rb <= 15 else (13 if m_hint <= 2 else 12)
    return 16 << rb


def _evaluate(lay, X, want_grad=True):
    """(fp64 loss sum S = sum f before the division by p, gradient or None)"""
    _, g = lay.value_and_grad(X, want_grad=want_grad)
    torch.cuda.synchronize()
    return float(lay.loss.item()), (None if g is None else g.cpu().numpy())


def _exploded(f, edges, X, m_hint, m_eval, kind, det, want_grad=True):
    """(S_M, terms t (p, m_eval) = grad_M[2k], grad_M[2k + 1]) of the exploded matching on the layout kind"""
    p = len(edges)
    step = _chunk_edges(kind, m_hint)
    S, t0, t1 = 0.0, [], []
    for a in range(0, p, step):
        b = min(p, a + step)
        q = b - a
        em = np.stack([2 * np.arange(q), 2 * np.arange(q) + 1], 1).astype(np.int64)
        xm = np.empty((2 * q, m_eval), np.float32)
        xm[0::2] = X[edges[a:b, 0]]
        xm[1::2] = X[edges[a:b, 1]]
        lay = _layout(f, em, 2 * q, p, m_hint, slice(a, b))
        assert _flags(lay) == (kind, det), ("exploded matching", _flags(lay), kind, det)
        s, g = _evaluate(lay, torch.tensor(xm, device="cuda"), want_grad)
        lay.close()
        S += s
        if want_grad:
            t0.append(g[0::2])
            t1.append(g[1::2])
    if not want_grad:
        return S, None, None
    return S, np.concatenate(t0), np.concatenate(t1)


# ------------------------------------------------------------------------------------------------ checks
def check_rows(grad, t, edges, n, extra=1):
    """check A: |grad_ic - sum_k s_ik t_kc| <= gamma_(deg_i + extra) sum_k |t_kc| for every row and column; returns the
    largest ratio.  extra = 1: the product rounding; 3: MUFU ELL's class constant as well."""
    t = np.asarray(t, np.float64)
    g = np.asarray(grad, np.float64)
    deg = np.bincount(edges.ravel(), minlength=n)
    bound_k = gamma(deg + extra)
    worst = 0.0
    for c in range(t.shape[1]):
        s = np.bincount(edges[:, 0], t[:, c], n) - np.bincount(edges[:, 1], t[:, c], n)
        a = np.bincount(edges[:, 0], np.abs(t[:, c]), n) + np.bincount(edges[:, 1], np.abs(t[:, c]), n)
        err = np.abs(g[:, c] - s)
        bound = bound_k * a
        bad = np.flatnonzero(~(err <= bound))
        assert not len(bad), ("row sum", c, [(int(i), int(deg[i]), g[i, c], s[i], bound[i]) for i in bad[:5]])
        with np.errstate(all="ignore"):
            r = np.where(bound > 0, err / bound, 0.0)
        worst = max(worst, float(r.max()))
    return worst


def check_terms(t, edges, X, spec, p, mufu, ell, loss):
    """check A's second part: t_kc against the fp64 oracle's g (x_i - x_j) over d (1 +- e), widened by TOL"""
    X64 = X.astype(np.float64)
    diff = X64[edges[:, 0]] - X64[edges[:, 1]]
    m = X.shape[1]
    d = np.sqrt((diff * diff).sum(1))
    pos = d > 0
    assert np.all(t[~pos] == 0.0), "terms of coincident rows must be exactly 0"
    d, diff, t = d[pos], diff[pos], np.asarray(t, np.float64)[pos]
    sub = O.FnSpec(spec.fn_att, spec.par0[pos], spec.att, fn_rep=spec.fn_rep if spec.push_pull else None,
                   rep=spec.rep if spec.push_pull else None, par1=None if spec.par1 is None else spec.par1[pos])
    eps = max((m + 2) * U, TOL["ell_d_rel"] if ell else 0.0)
    with np.errstate(all="ignore"):
        fp64 = O.eval_function(sub, d)[1]
        o32 = O.eval_function(sub, d.astype(np.float32), np.float32)[1].astype(np.float64)
        gs = [O.eval_function(sub, d * s)[1] / (p * d * s) for s in (1.0 - eps, 1.0, 1.0 + eps)]
    tol = TOL["ieee_k"] * np.abs(o32 - fp64) + TOL["ieee_ulp"] * _ulp32(fp64) + 2.0 ** -126
    if loss:
        w = np.abs(sub.par0.astype(np.float64))
        tol = tol + TOL["ieee_ulp"] * _ulp32(w + 1.0 / w)
    if mufu:
        tol = tol + TOL["mufu_fp_rel"] * np.abs(fp64)
    glo, ghi = np.minimum.reduce(gs), np.maximum.reduce(gs)
    gtol = tol / (p * d) + 8 * _ulp32(ghi) + 8 * _ulp32(glo) + (2.0 ** -20 if ell else 0.0) * np.abs(ghi)
    for c in range(m):
        lo = np.minimum(glo * diff[:, c], ghi * diff[:, c]) - gtol * np.abs(diff[:, c]) - 2.0 ** -126
        hi = np.maximum(glo * diff[:, c], ghi * diff[:, c]) + gtol * np.abs(diff[:, c]) + 2.0 ** -126
        bad = np.flatnonzero(~((t[:, c] >= lo) & (t[:, c] <= hi)))
        assert not len(bad), ("term", c, [(d[k], t[k, c], glo[k] * diff[k, c], gtol[k] * abs(diff[k, c]))
                                          for k in bad[:5]])


def loss_bound(f32_terms_abs_sum, p, mufu_or_ell):
    """check E: |S_G - S_M| for two sums of the same fp32 terms"""
    if mufu_or_ell:
        return 2 * gamma(8) * f32_terms_abs_sum
    return 2 * gamma(p, 2.0 ** -53) * f32_terms_abs_sum + 1e-300


def _f_tol(spec, d, f_out, mufu, ell, loss):
    """per-edge tolerance between two of the kernels' f values (fused, value-only, distortions())"""
    w = np.abs(spec.par0.astype(np.float64))
    tol = 2 * TOL["ieee_ulp"] * _ulp32(f_out)
    if loss:
        tol = tol + TOL["ieee_ulp"] * _ulp32(w + 1.0 / w)
    if mufu or ell:
        tol = tol + TOL["mufu_f_abs"] * w + TOL["mufu_f_rel"] * np.abs(f_out)
    if ell:
        with np.errstate(all="ignore"):
            tol = tol + np.abs(O.eval_function(spec, d)[1]) * d * TOL["ell_d_rel"]
    return tol


# ------------------------------------------------------------------------------------------------ A and E
_SEEN = {}


def _run_a(pm, path, name, geom=None):
    env, m_hint, m_eval, kind, det = PATHS[path]
    geom = geom or _graph_of(path)
    n, e, co, isolated, X0 = _problem(geom, m_eval)
    edges = _edges_for(name, e, co)
    p = len(edges)
    if name == "wquad" and kind != 0:
        kind = 0  # WeightedQuadratic's second parameter array keeps every graph on the sorted-SoA layout
    f = _function(pm, name, p, seed=p + m_eval)
    spec = O.spec_from_function(f)
    lay = _layout(f, edges, n, p, m_hint)
    assert _flags(lay) == (kind, det), (path, name, _flags(lay))
    X = torch.tensor(X0, device="cuda")
    SG, gG = _evaluate(lay, X)
    SG1, _ = _evaluate(lay, X, want_grad=False)
    _, fo = lay.outputs(X, distances=False, distortions=True)
    fo = fo.cpu().numpy().astype(np.float64)
    lay.close()
    SM, t, t1 = _exploded(f, edges, X0, m_hint, m_eval, kind, det)
    SM1, _, _ = _exploded(f, edges, X0, m_hint, m_eval, kind, det, want_grad=False)
    mufu = _mufu(name, m_hint, kind, m_eval)
    ell = kind == 3 and m_eval == m_hint
    # A
    assert np.array_equal(t1, -t), (path, name, "the two ends of an edge of M")
    check_terms(t, edges, X0, spec, p, mufu, ell, name in _LOSS)
    worst = check_rows(gG, t, edges, n, extra=3 if (ell and mufu) else 1)
    assert not np.any(gG[isolated]), "isolated rows must get an exact zero gradient"
    rows = np.abs(gG).max(1)
    span = rows.max() / rows[rows > 0].min()
    # E
    d = np.sqrt(((X0[edges[:, 0]].astype(np.float64) - X0[edges[:, 1]]) ** 2).sum(1))
    fabs = np.abs(fo).sum()
    assert abs(SG - SM) <= loss_bound(fabs * 1.01, p, mufu or ell), (path, name, "fused loss", SG, SM)
    assert abs(SG1 - SM1) <= loss_bound(fabs * 1.01, p, False), (path, name, "value-only loss", SG1, SM1)
    ftol = _f_tol(spec, d, fo, mufu, ell, name in _LOSS).sum()
    assert abs(SG - fo.sum()) <= ftol, (path, name, "fused loss vs distortions()", SG, fo.sum(), ftol)
    assert abs(SG1 - fo.sum()) <= ftol, (path, name, "value-only loss vs distortions()", SG1, fo.sum(), ftol)
    key = path.rsplit("_m", 1)[0]
    _SEEN[key] = max(_SEEN.get(key, 0.0), worst)
    print("A %s %s %s: kind %d det %d, max |g - sum t| / (gamma sum |t|) = %.3g (path max %.3g), |g_i| spans %.1e, "
          "loss bound / mean |f| = %.2g" % (path, geom, name, kind, det, worst, _SEEN[key], span,
                                             loss_bound(fabs, p, mufu or ell) / (fabs / p)))


_A_SMALL = [(path, name) for path in PATHS if not path.startswith("wide")
            for name in FNS if not (name == "wquad" and PATHS[path][3] != 0)]
_A_WIDE = [(path, name) for path in PATHS if path.startswith("wide")
           for name in ("pp_fast", "pp_logratio", "huber", "wquad")]


@gpu
@pytest.mark.parametrize("path,name", _A_SMALL)
def test_rows_are_sums_of_their_terms(path, name, monkeypatch):
    import pymde_b200 as pm
    _setenv(monkeypatch, PATHS[path][0])
    _setenv(monkeypatch, _fn_env(name))
    _run_a(pm, path, name)


@gpu
@pytest.mark.parametrize("path,name", _A_WIDE)
def test_wide_rows_are_sums_of_their_terms(path, name, monkeypatch):
    import pymde_b200 as pm
    _setenv(monkeypatch, PATHS[path][0])
    _run_a(pm, path, name)


@gpu
@pytest.mark.parametrize("name", ["pp_fast", "pp_precise", "huber", "wquad"])
@pytest.mark.parametrize("path", ["owner_m%d" % m for m in (1, 2, 3, 4)] + ["ell_m%d" % m for m in (1, 2, 3, 4)])
def test_g3_rows_are_sums_of_their_terms(path, name, monkeypatch):
    """100 000 rows, about 10^6 edges: several super-tiles and, at the default tile size, 13 or 25 ELL tiles"""
    if name == "wquad" and PATHS[path][3] != 0:
        pytest.skip("WeightedQuadratic builds the sorted-SoA layout")
    import pymde_b200 as pm
    _setenv(monkeypatch, PATHS[path][0])
    _setenv(monkeypatch, LG.GEOMETRIES["G3"][1])
    _setenv(monkeypatch, _fn_env(name))
    _run_a(pm, path, name, geom="G3")


# ------------------------------------------------------------------------------------------------ B
STAR_DEGREES = sorted({1} | {2 ** k + o for k in range(1, 17) for o in (-1, 0, 1)})
BALANCED = (1, 4, 64, 255, 4096, 32768)  # n+ = n- on column 0 (and column 1)
_STAR_P = 1 << 20
_STAR_N = 8155
_POOL = 8  # neighbour rows per star and side; edges to them repeat (duplicate edges)


def star_graph(m, seed=5):
    """(edges, X, stars): stars = [(hub, {column: (n_plus, n_minus)})].  Column 0 holds the hub's attractive
    neighbours (weight +1) at X[h] - e_0 (n_plus) and X[h] + e_0 (n_minus); column 1 (m >= 2) the second class
    (weight -1, or a second deviation) the same way.  Filler edges between the other rows bring p to 2^20, so 1/p is a
    power of two."""
    rng = np.random.default_rng(seed)
    rows = list(rng.permutation(_STAR_N))
    X = np.zeros((_STAR_N, m), np.float32)
    edges, cls, stars = [], [], []
    shapes = [(d, 0) for d in STAR_DEGREES] + [(b, b) for b in BALANCED]
    for si, (npl, nmi) in enumerate(shapes):
        h = rows.pop()
        X[h] = rng.integers(-6, 7, m)
        X[h, 0] = 20 * (si % 40) - 400  # hubs far apart
        cols = {0: (npl, nmi)}
        if m >= 2:
            cols[1] = (nmi + 1, npl) if si % 2 else (npl, nmi)
        for c, (a, b) in cols.items():
            for sgn, cnt in ((-1.0, a), (1.0, b)):
                if not cnt:
                    continue
                pool = [rows.pop() for _ in range(min(_POOL, cnt))]
                for r in pool:
                    X[r] = X[h]
                    X[r, c] += sgn  # x_h - x_r = -sgn e_c: a term -sgn t on the hub's column c
                nb = np.array(pool)[np.arange(cnt) % len(pool)]
                e = np.stack([np.full(cnt, h), nb], 1)
                flip = rng.random(cnt) < 0.5
                e[flip] = e[flip][:, ::-1]
                edges.append(e)
                cls.append(np.full(cnt, c))
        stars.append((h, cols))
    fill_rows = np.array(rows)
    X[fill_rows] = rng.integers(-30, 31, (len(fill_rows), m))
    e = np.concatenate(edges)
    k = _STAR_P - len(e)
    assert k > 0
    a = rng.choice(fill_rows, k)
    b = rng.choice(fill_rows, k)
    b = np.where(a == b, fill_rows[(np.searchsorted(fill_rows, b) + 1) % len(fill_rows)], b)
    fill = np.stack([a, b], 1)
    fill = fill[fill[:, 0] != fill[:, 1]]
    fill = np.concatenate([fill, fill[: k - len(fill)]]) if len(fill) < k else fill
    edges = np.concatenate([e, fill]).astype(np.int64)
    cls = np.concatenate(cls + [np.full(k, 2)])
    assert len(edges) == _STAR_P
    return edges, cls, X, stars


# function -> (column-0 class parameter, column-1 class parameter, filler parameter), f'(1) of a column's class,
# whether column 1 is exact
STAR_FNS = {
    "pp_fast": (1.0, -1.0, -1.0, 0.75, False),
    "pp_precise": (1.0, -1.0, -1.0, 0.75, False),
    "huber": (0.75, 0.25, 1.5, (0.5, 1.0), True),  # threshold 0.5: r = 0.25 quadratic (2 r), r = 0.75 linear (2 * 0.5)
    "quadratic": (0.75, 0.25, 1.5, (0.5, 1.5), True),
    "wquad": (0.5, 0.25, 1.5, (4.0, 24.0), True),  # w = 1 / dev^2: 2 * 4 * 0.5, 2 * 16 * 0.75
}


def star_expected(stars, fp1, m, p, exact_cols):
    """{hub: {column: exact fp64 value}}: sum over the hub's neighbours of g (x_h - x_r), g = f'(1) / p"""
    out = {}
    for h, cols in stars:
        out[h] = {}
        for c, (npl, nmi) in cols.items():
            if c in exact_cols:
                out[h][c] = fp1[c] / p * (npl - nmi)  # x_h - x_r = +e_c at the n_plus neighbours, -e_c at the others
    return out


def _star_function(pm, name, cls):
    a, b, fill, _, _ = STAR_FNS[name]
    par = np.where(cls == 0, a, np.where(cls == 1, b, fill)).astype(np.float32)
    t = torch.tensor(par, device="cuda")
    pen, los = pm.penalties, pm.losses
    if name.startswith("pp"):
        return pen.PushAndPull(t, pen.Log1p, pen.Log)
    return {"huber": lambda: los.Huber(t, 0.5), "quadratic": lambda: los.Quadratic(t),
            "wquad": lambda: los.WeightedQuadratic(t)}[name]()


_B_PATHS = (["owner_m%d" % m for m in (1, 2, 3, 4)] + ["tiles_m1", "tiles_m2", "tiles_m3", "tiles_m4"] +
            ["pull4_m2", "pull8_m3", "pullpush_m2", "pullpush_m4", "pull4_m1"] +
            ["ell_m%d" % m for m in (1, 2, 3, 4)] + ["ellrb8_m2", "ellrb8_m3"] + ["quad_m2", "quad_m3"] +
            ["wide_m%d" % m for m in (5, 8, 13, 36, 100, 512)] + ["wideowner_m%d" % m for m in (5, 33, 257, 512)])


@gpu
@pytest.mark.parametrize("name", sorted(STAR_FNS))
@pytest.mark.parametrize("path", _B_PATHS)
def test_star_rows_are_exact(path, name, monkeypatch):
    import pymde_b200 as pm
    env, m_hint, m_eval, kind, det = PATHS[path]
    if name == "wquad":
        if kind != 0:
            pytest.skip("WeightedQuadratic builds the sorted-SoA layout")
    _setenv(monkeypatch, env)
    _setenv(monkeypatch, _fn_env(name))
    edges, cls, X, stars = star_graph(m_eval)
    f = _star_function(pm, name, cls)
    lay = _layout(f, edges, _STAR_N, _STAR_P, m_hint)
    assert _flags(lay) == (kind, det), (path, name, _flags(lay))
    _, g = _evaluate(lay, torch.tensor(X, device="cuda"))
    lay.close()
    fp1 = STAR_FNS[name][3]
    fp1 = (fp1, fp1) if not isinstance(fp1, tuple) else fp1
    exact = (0, 1) if STAR_FNS[name][4] else (0,)
    want = star_expected(stars, fp1, m_eval, _STAR_P, exact)
    bad = [(h, c, g[h, c], v) for h, cols in want.items() for c, v in cols.items() if g[h, c] != v]
    assert not bad, (path, name, bad[:6])
    for h, cols in stars:  # columns without neighbours of the hub are exactly 0
        assert not np.any(g[h, 2:])
    print("B %s %s: kind %d det %d, %d hubs exact on columns %s" % (path, name, kind, det, len(stars), exact))


# ------------------------------------------------------------------------------------------------ C
_C_PATHS = (["tiles_m%d" % m for m in (1, 2, 3, 4)] + ["pull4_m%d" % m for m in (1, 2, 3, 4)] +
            ["pullpush_m2", "pull8_m3"] + ["ellrb8_m%d" % m for m in (1, 2, 3, 4)] + ["ell_m2"] +
            ["quad_m%d" % m for m in (1, 2, 3)] + ["quadell_m%d" % m for m in (1, 2, 3)] +
            ["wide_m%d" % m for m in (5, 8, 13, 36, 100, 255, 512, 1024)])


@gpu
@pytest.mark.parametrize("path", _C_PATHS)
def test_external_scatter_is_exact_on_every_kind(path, monkeypatch):
    import pymde_b200 as pm
    env, m_hint, m_eval, kind, det = PATHS[path]
    _setenv(monkeypatch, env)
    n = 6000
    e, g, w, X4, isolated = _exact_graph(300 + m_eval, n)
    X = (X4[:, :m_eval] if m_eval <= 4 else
         np.random.default_rng(m_eval).integers(-8, 9, (n, m_eval)).astype(np.float32))
    X = np.ascontiguousarray(X)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    lay = _layout(f, e, n, len(e), m_hint)
    assert _flags(lay) == (kind, det), (path, _flags(lay))
    got = lay.scatter_external(torch.tensor(X, device="cuda"), torch.tensor(g, device="cuda")).cpu().numpy()
    lay.close()
    want = _exact_expected(e, g, X, n)
    assert np.array_equal(got.astype(np.float64), want), (path, np.abs(got - want).max())
    assert not np.any(got[isolated])
    print("C %s: kind %d det %d, exact" % (path, kind, det))


@gpu
@pytest.mark.parametrize("layout", ["tiles", "pull4"])
def test_external_scatter_at_another_m_on_tile_layouts(layout, monkeypatch):
    """Tile and pull records are cut for the layout's m: an evaluation at another m is refused, not miscomputed."""
    import pymde_b200 as pm
    from pymde_b200 import _lib
    env = PATHS["%s_m4" % layout][0]
    _setenv(monkeypatch, env)
    n = 6000
    e, g, w, X4, isolated = _exact_graph(400, n)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    lay = _layout(f, e, n, len(e), 4)
    assert _flags(lay)[0] in (1, 2)
    for m in (1, 2, 3):
        X = np.ascontiguousarray(X4[:, :m])
        Xt = torch.tensor(X, device="cuda")
        try:
            got = lay.scatter_external(Xt, torch.tensor(g, device="cuda")).cpu().numpy()
        except _lib.MdeError as err:
            print("C %s m=%d on a layout for m=4: refused (%s)" % (layout, m, err))
            continue
        assert np.array_equal(got.astype(np.float64), _exact_expected(e, g, X, n)), (layout, m)
        print("C %s m=%d on a layout for m=4: exact" % (layout, m))
    lay.close()


# ------------------------------------------------------------------------------------------------ D
D_PATHS = (["owner_m%d" % m for m in (1, 2, 3, 4)] + ["quad_m%d" % m for m in (1, 2, 3)] +
           ["tiles_m%d" % m for m in (1, 2, 3, 4)] + ["pull4_m%d" % m for m in (1, 2, 3, 4)] +
           ["pull8_m2", "pullpush_m2", "pullpush_m3"] + ["wide_m%d" % m for m in (5, 13, 36, 100, 512, 1024)] +
           ["wideowner_m%d" % m for m in (5, 33, 257, 512)])
_D_P = 1 << 16


def quadratic_graph(m, seed=9, n=6000):
    """(edges (2^16, 2) with a hub of degree 5200, duplicates, coincident rows; weights +-2^-k; X small integers)"""
    e, g, w, X4, isolated = _exact_graph(seed, n)
    rng = np.random.default_rng(seed + m)
    e = np.concatenate([e, e[: _D_P - len(e)]]) if len(e) < _D_P else e[:_D_P]
    w = (rng.choice([1.0, -1.0], len(e)) * 2.0 ** -rng.integers(0, 4, len(e))).astype(np.float32)
    X = rng.integers(-8, 9, (n, m)).astype(np.float32)
    co = e[-10:]
    X[co[:, 1]] = X[co[:, 0]]
    return e, w, X, isolated


def quadratic_expected(e, w, X, p):
    """fp64: g = 2 w / p, grad = sum_k g_k (x_i - x_j) at i, minus at j"""
    return _exact_expected(e, (2.0 * w.astype(np.float64) / p), X, X.shape[0])


@gpu
@pytest.mark.parametrize("path", D_PATHS)
def test_quadratic_pushpull_is_exact(path, monkeypatch):
    import pymde_b200 as pm
    env, m_hint, m_eval, kind, det = PATHS[path]
    assert kind != 3
    _setenv(monkeypatch, env)
    e, w, X, isolated = quadratic_graph(m_eval)
    n = X.shape[0]
    pen = pm.penalties
    f = pen.PushAndPull(torch.tensor(w, device="cuda"), pen.Quadratic, pen.Quadratic)
    lay = _layout(f, e, n, len(e), m_hint)
    assert _flags(lay) == (kind, det), (path, _flags(lay))
    _, g = _evaluate(lay, torch.tensor(X, device="cuda"))
    lay.close()
    want = quadratic_expected(e, w, X, len(e))
    assert np.array_equal(g.astype(np.float64), want), (path, np.abs(g - want).max())
    assert not np.any(g[isolated])
    print("D %s: kind %d det %d, exact" % (path, kind, det))


# ------------------------------------------------------------------------------------------------ CPU self-checks
def _emulated_terms(edges, X, w, p):
    """fp32 terms g (x_i - x_j) of PushAndPull(Log1p, Log) from the fp64 oracle, rounded to fp32"""
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    X64 = X.astype(np.float64)
    diff = X64[edges[:, 0]] - X64[edges[:, 1]]
    d = np.sqrt((diff * diff).sum(1))
    fp = O.eval_function(spec, d)[1]
    return ((fp / (p * d))[:, None] * diff).astype(np.float32)


def _fp32_rows(edges, t, n):
    """fp32 sums of the terms, in edge order (one summation order a kernel might take)"""
    g = np.zeros((n, t.shape[1]), np.float32)
    for k in range(len(edges)):
        g[edges[k, 0]] += t[k]
        g[edges[k, 1]] -= t[k]
    return g


def test_row_check_catches_a_dropped_duplicated_or_flipped_entry():
    rng = np.random.default_rng(3)
    n, m = 400, 2
    e = rng.integers(0, n, (3000, 2))
    e = e[e[:, 0] != e[:, 1]]
    hub = np.stack([np.zeros(300, np.int64), rng.integers(1, n, 300)], 1)
    e = np.concatenate([e, hub]).astype(np.int64)
    X = rng.standard_normal((n, m)).astype(np.float32)
    w = rng.choice([1.0, 2.0, -1.0], len(e)).astype(np.float32)
    t = _emulated_terms(e, X, w, len(e))
    g = _fp32_rows(e, t, n)
    check_rows(g, t, e, n)  # an fp32 summation passes
    deg = np.bincount(e.ravel(), minlength=n)
    k = int(np.flatnonzero((deg[e[:, 0]] < 30) & (np.abs(t[:, 0]) > 1e-3 * np.abs(t[:, 0]).max()))[0])
    i = e[k, 0]
    for how in ("drop", "dup", "flip"):
        bad = g.copy()
        bad[i] += {"drop": -1, "dup": 1, "flip": -2}[how] * t[k]
        with pytest.raises(AssertionError):
            check_rows(bad, t, e, n)


def test_row_check_catches_a_term_perturbed_by_2_to_the_minus_18():
    """a degree-13 row whose largest term carries most of its mass (twelve edges of weight 2^-8, one of weight 1): that
    term off by 2^-18 of itself exceeds gamma_14 sum |t| ~ 2^-20 |t|"""
    rng = np.random.default_rng(4)
    n, m = 14, 2
    e = np.stack([np.zeros(13, np.int64), np.arange(1, 14)], 1)
    X = np.zeros((n, m), np.float32)
    X[1:] = rng.uniform(0.8, 1.2, (13, m)).astype(np.float32)
    t = _emulated_terms(e, X, np.array([2.0 ** -8] * 12 + [1.0], np.float32), 13)
    g = _fp32_rows(e, t, n)
    check_rows(g, t, e, n)
    bad = g.astype(np.float64)
    bad[0] += t[12].astype(np.float64) * 2.0 ** -18
    with pytest.raises(AssertionError):
        check_rows(bad, t, e, n)


def test_star_check_catches_one_lost_entry():
    """at k = 16 (degree 2^16 + 1) an fp32 sum of the exact terms equals the expected value, and one entry less does
    not; the star's neighbours all have the same fp32 d^2"""
    m = 2
    edges, cls, X, stars = star_graph(m)
    p = _STAR_P
    fp1 = (0.75, 0.75)
    want = star_expected(stars, fp1, m, p, (0,))
    h, cols = next(s for s in stars if s[1][0] == (2 ** 16 + 1, 0))
    sel = np.flatnonzero(((edges[:, 0] == h) | (edges[:, 1] == h)) & (cls == 0))
    assert len(sel) == 2 ** 16 + 1
    nb = np.where(edges[sel, 0] == h, edges[sel, 1], edges[sel, 0])
    diff = X[h][None, :] - X[nb]  # fp32
    d2 = (diff * diff).sum(1, dtype=np.float32)
    assert np.all(d2 == np.float32(1.0)), "every neighbour of the star at the same fp32 d^2"
    t = np.float32(fp1[0] / p) * diff[:, 0]
    acc = np.float32(0.0)
    for v in t:  # fp32, one order
        acc = np.float32(acc + v)
    assert acc == want[h][0]
    acc2 = np.float32(0.0)
    for v in t[1:]:
        acc2 = np.float32(acc2 + v)
    assert acc2 != want[h][0]
    assert np.float32(np.sum(t[::-1], dtype=np.float32)) == want[h][0]  # another order, the same bits


def test_star_terms_that_are_not_dyadic_do_not_sum_exactly():
    """why the repulsive class of the stars is held to check A only: three copies of 1 + 2^-23 need 25 bits"""
    t = np.float32(1.0 + 2.0 ** -23)
    assert np.float32(np.float32(t + t) + t) != 3.0 * np.float64(t)


def test_quadratic_graph_has_exact_fp32_partial_sums():
    """check D's graph: every term 2 w (x_i - x_j) / p and every fp32 partial sum in edge order is exact"""
    for m in (1, 3):
        e, w, X, isolated = quadratic_graph(m)
        p = len(e)
        assert p == _D_P and p & (p - 1) == 0
        X64 = X.astype(np.float64)
        t64 = (2.0 * w.astype(np.float64) / p)[:, None] * (X64[e[:, 0]] - X64[e[:, 1]])
        assert np.array_equal(t64.astype(np.float32).astype(np.float64), t64)
        g32 = _fp32_rows(e, t64.astype(np.float32), X.shape[0])
        assert np.array_equal(g32.astype(np.float64), quadratic_expected(e, w, X, p))
        deg = np.bincount(e.ravel(), minlength=X.shape[0])
        assert deg.max() >= 5000
