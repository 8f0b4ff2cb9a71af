"""Every table distortion function, edge by edge, on every kernel path, against the reference's fp32 and fp64 values.

The points of tests/golden/function_matrix.npz (tests/function_matrix_cases.py) become one MDE problem per case, on a
matching graph that makes every edge observable:

  edge k = (2k, 2k+1), given as (2k+1, 2k) for odd k;  X[2k] = 0,  X[2k+1] = d_k e_c,  c = k mod m.

The fp32 distance is then exactly d_k (sqrt(fl(d^2)) = d in IEEE arithmetic while d^2 is normal), grad[2k+1, c] =
g_k d_k = f'_k / p (or d_k where the guard set g_k = 1), grad[2k, c] is its negative, every other gradient entry is
exactly 0, and distortions() returns f_k.  Points where d^2 is not a normal fp32 number (and, in the fixed-point
deterministic mode, gradients beyond its +-8e6 range) leave the MDE paths; the function API takes every point.

Tolerances (r64 / r32: the reference in fp64 / fp32, o32: the fp32 oracle, w: weight or deviation, all per point):

  TOL["ieee"]   |k - r64| <= 10 |o32 - r64| + 16 ulp32(r64) + 2^-126
                ten times the fp32 oracle's own error at that point, floored at 16 ulp (the kernels use other but
                equivalent fp32 sequences: d sqrt(d) for d^1.5, a branch-free Huber, 1 / (d^e d) for InvPower).
  TOL["mufu"]   the recipe default on its MUFU kernels (m = 2, 3, fused): rsqrt / sqrt / rcp / lg2 / ex2.approx are
                within 2 ulp each (lg2 within 2^-22 absolute near 1); with the roundings around them f is within
                |w| 2^-18 + 2^-18 |f| and f' within 2^-17 |f'| (relative 2^-19 for 1 - e^-d above the series
                threshold, where it cancels, doubled).  The 4-term series below d = 0.0625 adds < 2^-23.
  TOL["ell"]    the ELL kernel forms d and 1/d from one rsqrt.approx: d carries a relative error below 2^-21.  The
                kernel value must lie in the range of the fp64 oracle over d (1 +- 2^-20), widened by TOL["ieee"]
                (and TOL["mufu"] for the recipe default) -- this holds across kinks as well.
  Losses add 16 ulp32 of gamma (delta + 1/delta) (gamma: SoftFractional's, else 1): near d = delta their closed forms
                subtract terms of that size (SoftFractional's f' = pu (-delta / d^2) + pv / delta, Fractional's tie).
                On the ELL paths the gradient is not checked within 2^-20 d of a loss's kink at d = delta: an
                approximate d lands on either side of it, where f' of loss Power(delta, e < 1) is unbounded.
  TOL["det"]    the fixed-point mode rounds every term to its row's quantum 2^-S, S = 61 - ceil(log2(deg)) - eM with
                the row's largest |contribution| below 2^eM: + 2^(eM - 62) absolute on the gradient here (every row
                of the matching holds one term).  A contribution that is not a finite fp32 number turns its entry NaN.
  TOL["g_abs"]  g = f' / (p d) is an fp32 number: where it falls below 2^-126 (tiny f' at large d) it is subnormal or
                flushed to 0, in the reference too; + 2^-126 d absolute on the gradient entry g d.
  Non-finite reference values must be matched exactly: f in the same class as r32; where the reference's fp32
  g = f' / p / d is non-finite the kernel's g is exactly 1 (its gradient entry is exactly d_k).
The mean is checked against the fp64 mean with the sum of the per-point f tolerances over p, plus 2 ulp32.
"""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O
from tests import function_matrix_cases as FM
from tests.test_function_matrix_cpu import GOLD, nonfinite_class, spec_of

gpu = pytest.mark.gpu

_ENV = ("MDE_B200_LAYOUT", "MDE_B200_TILE_RB", "MDE_B200_STILE_MB", "MDE_B200_TILE_MIN", "MDE_B200_PULL_EPL",
        "MDE_B200_PULL_REP", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC", "MDE_B200_ELL_BUILD")

TOL = {"mufu_f_abs": 2.0 ** -18, "mufu_f_rel": 2.0 ** -18, "mufu_fp_rel": 2.0 ** -17, "ell_d_rel": 2.0 ** -20,
       "det_headroom": 62, "g_abs": 2.0 ** -126, "ieee_ulp": 16, "ieee_k": 10.0}

_TILES = {"MDE_B200_TILE_MIN": "0"}
# path -> (environment, m, layout kind it must build)
PATHS = {
    "owner_m1": ({}, 1, 0), "owner_m2": ({}, 2, 0), "owner_m3": ({}, 3, 0), "owner_m4": ({}, 4, 0),
    "precise_owner_m2": ({"MDE_B200_KERNEL": "precise"}, 2, 0),
    "tiles_m2": (dict(_TILES, MDE_B200_LAYOUT="tiles"), 2, 1), "tiles_m3": (dict(_TILES, MDE_B200_LAYOUT="tiles"), 3, 1),
    "precise_tiles_m2": (dict(_TILES, MDE_B200_LAYOUT="tiles", MDE_B200_KERNEL="precise"), 2, 1),
    "pull_m2": (dict(_TILES, MDE_B200_LAYOUT="pull"), 2, 2), "pull_m3": (dict(_TILES, MDE_B200_LAYOUT="pull"), 3, 2),
    "precise_pull_m3": (dict(_TILES, MDE_B200_LAYOUT="pull", MDE_B200_KERNEL="precise"), 3, 2),
    "ell_m1": ({"MDE_B200_LAYOUT": "ell"}, 1, 3), "ell_m2": ({"MDE_B200_LAYOUT": "ell"}, 2, 3),
    "ell_m3": ({"MDE_B200_LAYOUT": "ell"}, 3, 3), "ell_m4": ({"MDE_B200_LAYOUT": "ell"}, 4, 3),
    "precise_ell_m2": ({"MDE_B200_LAYOUT": "ell", "MDE_B200_KERNEL": "precise"}, 2, 3),
    "det_m1": ({"MDE_B200_DETERMINISTIC": "1"}, 1, 0), "det_m2": ({"MDE_B200_DETERMINISTIC": "1"}, 2, 0),
    "det_m3": ({"MDE_B200_DETERMINISTIC": "1"}, 3, 0), "det_m4": ({"MDE_B200_DETERMINISTIC": "1"}, 4, 0),
}
for _m in (5, 13, 16, 33, 128, 257, 1024):  # wide push <8,1,1> <16,1,1> <8,1,4> <32,2,1> <32,1,4> <32,16,1> <32,8,4>
    PATHS["wide_m%d" % _m] = ({}, _m, 0)
for _m in (5, 16, 33, 257, 512):  # wide owner (deterministic, 5 <= m <= 512)
    PATHS["wide_owner_m%d" % _m] = ({"MDE_B200_DETERMINISTIC": "1"}, _m, 0)


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


def _ulp32(x):
    x = np.abs(np.where(np.isfinite(x), x, 0.0)).astype(np.float32)
    return np.spacing(x).astype(np.float64)


class Expected(object):
    """reference columns and per-point tolerances of one case on a subset `idx` of its points"""

    def __init__(self, name, idx, mufu, approx_d):
        spec = spec_of(name)
        case = FM.BY_NAME[name]
        gamma = max(1.0, spec.att[0]) if spec.fn_att == O.L_SOFT_FRACTIONAL else 1.0
        self.d = GOLD[name + "/d"][idx].astype(np.float64)
        self.w = GOLD[name + "/par0"][idx].astype(np.float64)
        self.r32 = {c: GOLD["%s/f32/%s" % (name, c)][idx] for c in ("f", "fp")}
        self.r64 = {c: GOLD["%s/f64/%s" % (name, c)][idx].astype(np.float64) for c in ("f", "fp")}
        with np.errstate(all="ignore"):
            o32 = O.eval_function(spec, GOLD[name + "/d"], np.float32)
        self.tol = {}
        for i, c in enumerate(("f", "fp")):
            r64 = self.r64[c]
            err = np.abs(o32[i][idx].astype(np.float64) - r64)
            t = TOL["ieee_k"] * np.where(np.isfinite(err), err, 0.0) + TOL["ieee_ulp"] * _ulp32(r64) + 2.0 ** -126
            if case.family == "loss":  # terms of size gamma (delta + 1 / delta) cancel near d = delta
                t = t + TOL["ieee_ulp"] * _ulp32(gamma * (np.abs(self.w) + 1.0 / np.abs(self.w)))
            if mufu:
                t = t + (TOL["mufu_f_abs"] * np.abs(self.w) + TOL["mufu_f_rel"] * np.abs(r64) if c == "f"
                         else TOL["mufu_fp_rel"] * np.abs(r64))
            self.tol[c] = t
        self.lo, self.hi = dict(self.r64), dict(self.r64)
        if approx_d:  # the fp64 oracle's range over d (1 +- 2^-20)
            for s in (1.0 - TOL["ell_d_rel"], 1.0 + TOL["ell_d_rel"]):
                sub = O.FnSpec(spec.fn_att, spec.par0[idx], spec.att,
                               fn_rep=spec.fn_rep if spec.push_pull else None, rep=spec.rep if spec.push_pull else None,
                               par1=None if spec.par1 is None else spec.par1[idx])
                with np.errstate(all="ignore"):
                    v = O.eval_function(sub, self.d * s, np.float64)
                for i, c in enumerate(("f", "fp")):
                    self.lo[c] = np.fmin(self.lo[c], v[i])
                    self.hi[c] = np.fmax(self.hi[c], v[i])

    def check(self, what, c, k, scale=1.0, extra_abs=0.0, mask=None):
        """k (fp32 kernel values) against column c, scaled by `scale` (1 / p for gradient entries)"""
        k = np.asarray(k, np.float64)
        r32 = self.r32[c]
        bad_cls = nonfinite_class(k) != nonfinite_class(r32 * scale)
        if c == "fp":  # the derivative's non-finite class is only seen through the guard
            bad_cls = np.isfinite(k) != np.isfinite(r32)
        if mask is not None:
            bad_cls &= mask
        i = np.flatnonzero(bad_cls)
        assert not len(i), (what, c, [(self.d[j], self.w[j], k[j], r32[j]) for j in i[:6]])
        fin = np.isfinite(r32) & np.isfinite(self.r64[c]) & (mask if mask is not None else True)
        t = self.tol[c] * scale + extra_abs
        with np.errstate(invalid="ignore"):
            ok = (k >= self.lo[c] * scale - t) & (k <= self.hi[c] * scale + t)
        i = np.flatnonzero(fin & ~ok)
        assert not len(i), (what, c, [(self.d[j], self.w[j], k[j], self.r64[c][j] * scale, t[j]) for j in i[:6]])


def _mufu(name, env):
    return name == "pp_log1p_log" and env.get("MDE_B200_KERNEL") != "precise"


def _problem(name, m, det):
    """(idx of the points used, edges, X) of the matching graph of case `name`"""
    d = GOLD[name + "/d"]
    ok = (d == 0) | ((d >= 2.0 ** -60) & (d <= 2.0 ** 60))
    if det:  # a contribution f'/p that is not a finite fp32 number is NaN in the fixed-point mode, inf in the others
        with np.errstate(all="ignore"):
            fp = np.abs(GOLD[name + "/f64/fp"].astype(np.float64)) / max(1, int(ok.sum()))
        ok &= ~(fp >= 2.0 ** 128)
    idx = np.flatnonzero(ok)
    p = len(idx)
    e = np.stack([2 * np.arange(p), 2 * np.arange(p) + 1], 1)
    e[1::2] = e[1::2, ::-1]
    X = np.zeros((2 * p, m), np.float32)
    X[2 * np.arange(p) + 1, np.arange(p) % m] = d[idx]
    return idx, e, X


def _function(pm, name, idx):
    case = FM.BY_NAME[name]
    _, par0, par1 = FM.points(case)
    par0 = torch.tensor(par0[idx], device="cuda")
    par1 = None if par1 is None else torch.tensor(par1[idx], device="cuda")
    return FM.build(pm, case, par0, par1)


def _kind(mde):
    from pymde_b200 import _lib
    return int(_lib.load().mde_edges_kind(mde._layout().handle))


def _run_case(pm, name, path):
    env, m, want = PATHS[path]
    det = env.get("MDE_B200_DETERMINISTIC") == "1"
    idx, e, X0 = _problem(name, m, det)
    p = len(idx)
    f = _function(pm, name, idx)
    mde = pm.MDE(2 * p, m, torch.tensor(e, device="cuda"), f, pm.Centered())
    X = torch.tensor(X0, device="cuda")
    Xg = X.clone().requires_grad_(True)
    v = mde.average_distortion(Xg)
    v.backward()
    kind = _kind(mde)
    has_par1 = name + "/par1" in GOLD.files
    assert kind == (0 if has_par1 and want in (1, 2, 3) else want), (path, name, kind)
    fused_mufu = _mufu(name, env) and m in (2, 3)
    ex = Expected(name, idx, mufu=fused_mufu, approx_d=(kind == 3))
    # gradient: row 2k+1 column c holds f'_k / p, or d_k where the reference's g was not finite
    G = Xg.grad.cpu().numpy().astype(np.float64)
    rows, cols = 2 * np.arange(p) + 1, np.arange(p) % m
    gk = G[rows, cols]
    assert np.array_equal(G[rows - 1, cols], -gk), (path, name, "the two ends of an edge")
    rest = G.copy()
    rest[rows, cols] = 0.0
    rest[rows - 1, cols] = 0.0
    assert not np.any(rest), (path, name, "entries off the edge direction must be exactly 0")
    with np.errstate(all="ignore"):
        inv_p = np.float32(1.0) / np.float32(p)
        g32 = (ex.r32["fp"] * inv_p) / GOLD[name + "/d"][idx]
    guard = ~np.isfinite(g32)
    at0 = ex.d == 0
    if kind == 3:  # an approximate d does not resolve a loss's kink at d = delta: points within 2^-20 d of it are
        # not checked (among them the guard's points at d > 0, loss Power(delta, e < 1) at d = delta)
        ex_mask = ~((FM.BY_NAME[name].family == "loss") & (np.abs(ex.d - ex.w) <= TOL["ell_d_rel"] * ex.d))
        guard = guard & ex_mask
    else:
        ex_mask = np.ones(p, bool)
    assert np.all(gk[at0] == 0.0), (path, name, "d = 0")
    det_abs = np.zeros(p)
    if det:  # half the quantum of the row's one term, |gk| <= 2^eM
        with np.errstate(all="ignore"):
            det_abs = np.where(np.isfinite(gk) & (gk != 0),
                               2.0 ** (np.floor(np.log2(np.abs(gk))) + 1 - TOL["det_headroom"]), 0.0)
    hit = guard & ~at0
    j = np.flatnonzero(np.abs(gk[hit] - ex.d[hit]) > det_abs[hit])
    assert not len(j), (path, name, "guard: g = 1", [(ex.d[hit][i], ex.w[hit][i], gk[hit][i]) for i in j[:6]])
    # g = f' / (p d) is an fp32 intermediate: below 2^-126 it is subnormal or flushed, which the entry g d carries as an
    # absolute error up to 2^-126 d (the reference's own g underflows there as well)
    ex.check(path + " grad", "fp", gk, scale=1.0 / p, extra_abs=TOL["g_abs"] * ex.d + det_abs,
             mask=~guard & ~at0 & ex_mask)
    # the mean, fused and value-only
    f64 = ex.r64["f"]
    for val, what in ((v.item(), "fused"), (mde.average_distortion(X).item(), "value")):
        if np.all(np.isfinite(ex.r32["f"])):
            t = ex.tol["f"].sum() / p + np.abs(np.fmax(ex.hi["f"] - f64, f64 - ex.lo["f"])).sum() / p
            assert abs(val - f64.mean()) <= t + 2 * _ulp32(np.array([f64.mean()]))[0], (path, name, what, val, f64.mean())
        else:
            assert not np.isfinite(val), (path, name, what, val)
    # per-edge outputs (kinds 0, 1, 2; ELL layouts answer from their sorted-SoA arrays)
    dist = mde.distances(X).cpu().numpy()
    np.testing.assert_array_equal(dist, GOLD[name + "/d"][idx])
    fo = mde.distortions(X).cpu().numpy()
    ex_out = Expected(name, idx, mufu=_mufu(name, env), approx_d=False)
    ex_out.check(path + " distortions", "f", fo)


@gpu
@pytest.mark.parametrize("path", sorted(PATHS))
def test_every_function_on_every_path(path, monkeypatch):
    import pymde_b200 as pm
    for k, v in PATHS[path][0].items():
        monkeypatch.setenv(k, v)
    for case in FM.CASES:
        _run_case(pm, case.name, path)


@gpu
@pytest.mark.parametrize("name", [c.name for c in FM.CASES])
def test_function_api(name):
    """f(d) with autograd (function_eval_kernel) at every point, overflow and underflow included."""
    import pymde_b200 as pm
    d = GOLD[name + "/d"]
    idx = np.arange(len(d))
    f = _function(pm, name, idx)
    dt = torch.tensor(d, device="cuda", requires_grad=True)
    val = f(dt)
    val.sum().backward()
    ex = Expected(name, idx, mufu=False, approx_d=False)
    ex.check("api f", "f", val.detach().cpu().numpy())
    ex.check("api fp", "fp", dt.grad.cpu().numpy())
