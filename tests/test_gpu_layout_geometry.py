"""Edge layouts across neighbour-tile and super-tile boundaries, against the fp64 oracle.

The tile records (kind 1, mde_tiled.cu), pull records (kind 2, mde_pull.cu) and ELL pull records (kind 3,
mde_ell.cu) cut the rows into neighbour tiles of R = 2^rb rows; kinds 1 and 2 also group owners into super-tiles of
S = 2^ss rows.  At their default sizes (R = 8192 / 4096 rows) every small test problem fits in one tile.  The
library's geometry switches, read when a layout is created, make a few thousand rows span tens of tiles:

  G1  MDE_B200_TILE_RB=8, MDE_B200_STILE_MB=0 (super-tile = tile), MDE_B200_TILE_MIN=0, n = 8155: 32 tiles of
      256 rows, the last one partial
  G2  MDE_B200_TILE_RB=8, n = 4096: 16 whole tiles
  G3  default tile size, MDE_B200_STILE_MB=1 (2^16 / 2^15 / 2^14 / 2^14 owner rows per super-tile at m = 1 / 2 / 3 /
      4), n = 100 000, p ~ 10^6
  G4  MDE_B200_TILE_RB=8 with ELL requested: n = 8192 is 32 tiles (ELL's limit), n = 8193 must fall back to SoA
  G5  pull records where one warp-tile would span more than 65 536 owner rows (a u16 owner offset)

Every graph has edges at rows 0, R - 1, R, S - 1, S and n - 1, hubs of degree >= 5000 reaching every tile (runs and
lane-slots split across records), isolated rows (gradient exactly 0), edges inside a tile and across tiles, and, for
functions with a finite f'(0), edges between coincident rows.  Every case asserts the layout kind it built
(mde_edges_kind: 0 sorted SoA, 1 tiles, 2 pull, 3 ELL), so a quiet fallback to SoA fails the test.

Tolerances are the suite's: value rtol 1e-5, gradient atol 3e-5 max|g_ref|, distances rtol 1e-6.  The GPU tests are
marked one by one: the oracle self-check at the end runs without a GPU."""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O

gpu = pytest.mark.gpu

# every switch that changes which layout or kernel the library picks; cleared before each test
_ENV = ("MDE_B200_LAYOUT", "MDE_B200_TILE_RB", "MDE_B200_STILE_MB", "MDE_B200_TILE_MIN", "MDE_B200_PULL_EPL",
        "MDE_B200_PULL_REP", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC", "MDE_B200_ELL_BUILD")

# layout variant -> (environment, kind it must build)
LAYOUTS = {
    "soa": ({"MDE_B200_LAYOUT": "soa"}, 0),
    "tiles": ({"MDE_B200_LAYOUT": "tiles"}, 1),
    "pull4": ({"MDE_B200_LAYOUT": "pull", "MDE_B200_PULL_EPL": "4"}, 2),
    "pull8": ({"MDE_B200_LAYOUT": "pull", "MDE_B200_PULL_EPL": "8"}, 2),
    "pull_push": ({"MDE_B200_LAYOUT": "pull", "MDE_B200_PULL_REP": "push"}, 2),
    "ell": ({"MDE_B200_LAYOUT": "ell"}, 3),
}

# geometry -> (n, environment, tile / super-tile boundaries the edges must touch)
_G3_BOUNDS = (4096, 8192, 16384, 32768, 65536)
GEOMETRIES = {
    "G1": (8155, {"MDE_B200_TILE_RB": "8", "MDE_B200_STILE_MB": "0", "MDE_B200_TILE_MIN": "0"}, (256,)),
    "G2": (4096, {"MDE_B200_TILE_RB": "8", "MDE_B200_TILE_MIN": "0"}, (256,)),
    "G3": (100_000, {"MDE_B200_STILE_MB": "1"}, _G3_BOUNDS),
    "G4a": (8192, {"MDE_B200_TILE_RB": "8"}, (256,)),
    "G4b": (8193, {"MDE_B200_TILE_RB": "8"}, (256,)),
}
_SIZES = {"G1": (40_000, 4000), "G2": (20_000, 2000), "G3": (1_000_000, 50_000), "G4a": (40_000, 4000),
          "G4b": (40_000, 4000)}

# functions: every compile-time function pair of the kernel families (select_fn in mde_edges.cuh and the pair lists)
FNS = ("pp_fast_mixed", "pp_fast_att", "pp_fast_rep", "pp_precise_mixed", "pp_logratio", "pen_quadratic",
       "loss_absolute", "loss_quadratic", "loss_huber", "pen_cubic", "loss_logistic", "pp_quad_invpower")
_COINCIDENT_OK = ("pen_quadratic", "loss_absolute", "loss_quadratic", "loss_huber", "pen_cubic", "loss_logistic")


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


def _setenv(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ------------------------------------------------------------------------------------------------ problems
def _graph(n, bounds, p_rand, p_local, seed, hub_deg=5000):
    """(edges (p, 2) int64 in random order and orientation, coincident pairs (k, 2), isolated rows, hubs)."""
    rng = np.random.default_rng(seed)
    special = sorted({r for b in bounds for r in (b - 1, b) if 0 <= r < n} | {0, n - 1})
    hubs = np.array([1, n // 3 + 7, (2 * n) // 3 + 11], dtype=np.int64)
    protected = set(special) | set(hubs.tolist())
    cand = np.setdiff1d(np.arange(2, n - 2), np.array(sorted(protected)))
    isolated = np.union1d(rng.choice(cand, max(8, n // 400), replace=False), [n - 2])
    active = np.setdiff1d(np.arange(n), isolated)
    parts = []
    # boundary rows: to their neighbour, to each other, to far rows
    sp = np.array(special, dtype=np.int64)
    for r in sp:
        nb = r + 1 if r + 1 < n and r + 1 not in isolated else r - 1
        parts.append([[r, nb]])
        parts.append(np.stack([np.full(4, r), rng.choice(active, 4)], 1))
    parts.append(np.array([(a, b) for a in sp for b in sp if a < b]))
    # hubs: degree >= hub_deg (or every active row), neighbours spread over every tile
    for h in hubs:
        deg = min(hub_deg, len(active) - 8)
        parts.append(np.stack([np.full(deg, h), rng.choice(active, deg, replace=False)], 1))
    # inside a tile (small offsets) and across tiles (uniform pairs)
    i = rng.choice(active, p_local)
    parts.append(np.stack([i, np.clip(i + rng.integers(1, 40, p_local), 0, n - 1)], 1))
    parts.append(np.stack([rng.choice(active, p_rand), rng.choice(active, p_rand)], 1))
    e = np.concatenate([np.asarray(x, dtype=np.int64).reshape(-1, 2) for x in parts])
    e = e[(e[:, 0] != e[:, 1]) & ~np.isin(e[:, 0], isolated) & ~np.isin(e[:, 1], isolated)]
    e = np.unique(np.sort(e, axis=1), axis=0)
    # coincident rows (X[b] = X[a]): pairs of ordinary rows in different tiles, not otherwise joined
    ordinary = np.setdiff1d(active, np.concatenate([sp, hubs]))
    co = rng.choice(ordinary, 16, replace=False).reshape(8, 2)
    co = np.sort(co, axis=1)
    key = e[:, 0] * n + e[:, 1]
    e = e[~np.isin(key, co[:, 0] * n + co[:, 1])]
    rng.shuffle(e)
    flip = rng.random(len(e)) < 0.5
    e[flip] = e[flip][:, ::-1]
    return e, co, isolated, hubs


_PROBLEMS = {}
_ORACLE = {}


def _problem(geom, m):
    key = (geom, m)
    if key not in _PROBLEMS:
        n, _, bounds = GEOMETRIES[geom]
        if (geom, 0) not in _PROBLEMS:
            p_rand, p_local = _SIZES[geom]
            _PROBLEMS[(geom, 0)] = _graph(n, bounds, p_rand, p_local, seed=len(geom) * 1000 + n)
        e, co, isolated, hubs = _PROBLEMS[(geom, 0)]
        rng = np.random.default_rng(7 * n + m)
        X = rng.standard_normal((n, m)).astype(np.float32)
        X -= X.mean(0)
        X[co[:, 1]] = X[co[:, 0]]
        _PROBLEMS[key] = (n, e, co, isolated, hubs, X)
    return _PROBLEMS[key]


def _fn_env(name):
    return {"MDE_B200_KERNEL": "precise"} if name.startswith("pp_precise") else {}


def _function(pm, name, p, seed):
    """Distortion function `name` on cuda for p edges, parameters drawn from `seed`."""
    rng = np.random.default_rng(seed)
    mix = name.rsplit("_", 1)[-1]
    if mix == "att":
        w = rng.uniform(0.5, 2.0, p)
    elif mix == "rep":
        w = -rng.uniform(0.5, 1.5, p)
    else:
        w = rng.choice([1.0, 2.0, -1.0], p)
    w = torch.tensor(w.astype(np.float32), device="cuda")
    dev = torch.tensor(rng.uniform(0.5, 2.0, p).astype(np.float32), device="cuda")
    pen, los = pm.penalties, pm.losses
    if name.startswith("pp_fast") or name.startswith("pp_precise"):
        return pen.PushAndPull(w, pen.Log1p, pen.Log)
    table = {
        "pp_logratio": lambda: pen.PushAndPull(w, pen.Log1p, pen.LogRatio),
        "pp_quad_invpower": lambda: pen.PushAndPull(w, pen.Quadratic, pen.InvPower),
        "pen_quadratic": lambda: pen.Quadratic(w.abs()),
        "pen_cubic": lambda: pen.Cubic(w.abs()),
        "loss_absolute": lambda: los.Absolute(dev),
        "loss_quadratic": lambda: los.Quadratic(dev),
        "loss_huber": lambda: los.Huber(dev, 0.5),
        "loss_logistic": lambda: los.Logistic(dev),
    }
    return table[name]()


def _edges_for(name, e, co):
    return np.concatenate([e, co]) if name in _COINCIDENT_OK else e


def _reference(geom, m, name, f, edges, X):
    key = (geom, m, name)
    if key not in _ORACLE:
        spec = O.spec_from_function(f)
        v, g = O.average_distortion(X.astype(np.float64), edges, spec, True)
        d, _ = O.edge_distances(X.astype(np.float64), edges)
        _ORACLE[key] = (v, g, d, O.eval_function(spec, d)[0])
    return _ORACLE[key]


def _assert_value(v, v_ref):
    np.testing.assert_allclose(v, v_ref, rtol=1e-5)


def _assert_grad(g, g_ref):
    err = np.abs(np.asarray(g, dtype=np.float64) - g_ref).max()
    assert err <= 3e-5 * np.abs(g_ref).max(), (err, np.abs(g_ref).max())


def _kind(mde):
    from pymde_b200 import _lib
    return int(_lib.load().mde_edges_kind(mde._layout().handle))


def _check_case(pm, geom, m, name, want_kind, X=None, record=None):
    """Fused value + gradient, value only and per-edge outputs of one (geometry, layout, m, function) case."""
    n, e, co, isolated, hubs, X0 = _problem(geom, m)
    edges = _edges_for(name, e, co)
    f = _function(pm, name, len(edges), seed=len(edges) + m)
    v_ref, g_ref, d_ref, f_ref = _reference(geom, m, name, f, edges, X0)
    mde = pm.MDE(n, m, torch.tensor(edges, device="cuda"), f, pm.Centered())
    if X is None:
        X = torch.tensor(X0, device="cuda")
    Xg = X.detach().requires_grad_(True)
    v = mde.average_distortion(Xg)
    v.backward()
    kind = _kind(mde)
    if record is not None:
        record("kind", kind)
    print("%s m=%d %s: kind %d" % (geom, m, name, kind))
    if want_kind is not None:
        assert kind == want_kind, (geom, m, name, kind, want_kind)
    _assert_value(v.item(), v_ref)
    g = Xg.grad.cpu().numpy()
    _assert_grad(g, g_ref)
    assert not np.any(g[isolated]), "isolated rows must get an exact zero gradient"
    v2 = mde.average_distortion(X.detach())
    np.testing.assert_allclose(v2.item(), v.item(), rtol=1e-6)
    d = mde.distances(X).cpu().numpy()
    np.testing.assert_allclose(d, d_ref, rtol=1e-6, atol=0)
    fo = mde.distortions(X).cpu().numpy()
    np.testing.assert_allclose(fo, f_ref, rtol=2e-5, atol=2e-6)
    return mde, kind


# ------------------------------------------------------------------------------------------------ G1
@gpu
@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_g1_many_tiles_every_function(layout, m, name, monkeypatch, record_property):
    import pymde_b200 as pm
    env, want = LAYOUTS[layout]
    _setenv(monkeypatch, GEOMETRIES["G1"][1])
    _setenv(monkeypatch, env)
    _setenv(monkeypatch, _fn_env(name))
    _check_case(pm, "G1", m, name, want, record=record_property)


@gpu
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_g1_embed_keeps_layout_and_starts_at_the_oracle(layout, m, monkeypatch):
    """embed(): iteration 0 is a plain evaluation of the layout's fused kernel, and the solver keeps the layout."""
    import pymde_b200 as pm
    env, want = LAYOUTS[layout]
    _setenv(monkeypatch, GEOMETRIES["G1"][1])
    _setenv(monkeypatch, env)
    n, e, co, isolated, hubs, X0 = _problem("G1", m)
    f = _function(pm, "pp_fast_mixed", len(e), seed=len(e) + m)
    v_ref = _reference("G1", m, "pp_fast_mixed", f, e, X0)[0]
    mde = pm.MDE(n, m, torch.tensor(e, device="cuda"), f, pm.Centered())
    mde.embed(X=torch.tensor(X0, device="cuda"), max_iter=5)
    assert _kind(mde) == want
    np.testing.assert_allclose(mde.solve_stats.average_distortions[0], v_ref, rtol=1e-5)
    assert mde.solve_stats.average_distortions[-1] < mde.solve_stats.average_distortions[0]


@gpu
@pytest.mark.parametrize("geom", ["G1", "G3"])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", ["soa", "tiles", "pull4", "ell"])
def test_external_callable_against_autograd(geom, layout, m, monkeypatch):
    """A Python callable as distortion function: distances and the scatter of per-edge coefficients
    (mde_scatter_external, also used by spectral initialisation) run on the layout's kernels."""
    import pymde_b200 as pm
    env, want = LAYOUTS[layout]
    _setenv(monkeypatch, GEOMETRIES[geom][1])
    _setenv(monkeypatch, env)
    n, e, co, isolated, hubs, X0 = _problem(geom, m)
    edges = np.concatenate([e, co])
    wts = torch.tensor(np.random.default_rng(m).uniform(0.5, 2.0, len(edges)).astype(np.float32), device="cuda")

    def f(d):
        return wts * d.pow(2)

    et = torch.tensor(edges, device="cuda")
    mde = pm.MDE(n, m, et, f, pm.Centered())
    Xd = torch.tensor(X0, device="cuda", requires_grad=True)
    v = mde.average_distortion(Xd)
    v.backward()
    assert _kind(mde) == want
    Xr = torch.tensor(X0, device="cuda", dtype=torch.float64, requires_grad=True)
    ref = (wts.double() * (Xr[et[:, 0]] - Xr[et[:, 1]]).pow(2).sum(1)).mean()
    ref.backward()
    _assert_value(v.item(), ref.item())
    _assert_grad(Xd.grad.cpu().numpy(), Xr.grad.cpu().numpy())
    assert not Xd.grad[torch.tensor(isolated, device="cuda")].any()


@gpu
@pytest.mark.parametrize("m", [1, 2, 3])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_g1_unaligned_rows_take_the_plain_load_path(layout, m, monkeypatch):
    """X = Xbig[1:] is a contiguous row slice whose data pointer is m * 4 bytes past a 16-byte boundary: the tile
    kernels then load the X tile with plain loads instead of cp.async.bulk.  Every X load in the kernels is at most one
    row wide (float2 at m = 2), so the pointer is aligned for each of them."""
    import pymde_b200 as pm
    env, want = LAYOUTS[layout]
    _setenv(monkeypatch, GEOMETRIES["G1"][1])
    _setenv(monkeypatch, env)
    n, e, co, isolated, hubs, X0 = _problem("G1", m)
    big = torch.zeros((n + 1, m), device="cuda")
    big[1:] = torch.tensor(X0, device="cuda")
    X = big[1:]
    assert X.is_contiguous() and big.data_ptr() % 16 == 0 and X.data_ptr() - big.data_ptr() == 4 * m
    for name in ("pp_fast_mixed", "loss_huber"):
        mde, _ = _check_case(pm, "G1", m, name, want, X=X)
        assert mde._check_X(X).data_ptr() == X.data_ptr()  # handed to the library as it is


@gpu
@pytest.mark.parametrize("m", [2, 4])
def test_flat_views_misaligned_for_row_loads_are_copied(m):
    """buf[1:1 + n m].view(n, m) is contiguous but only 4-byte aligned; the kernels load a row of m = 2 as one float2
    and of m = 4 as one float4, so such a view is copied before it reaches the library."""
    import pymde_b200 as pm
    n, e, co, isolated, hubs, X0 = _problem("G1", m)
    buf = torch.zeros(1 + n * m, device="cuda")
    Xv = buf[1:].view(n, m)
    Xv.copy_(torch.tensor(X0, device="cuda"))
    assert Xv.is_contiguous() and Xv.data_ptr() % (4 * m) != 0
    f = _function(pm, "pp_fast_mixed", len(e), seed=len(e) + m)
    mde = pm.MDE(n, m, torch.tensor(e, device="cuda"), f, pm.Centered())
    Xc = mde._check_X(Xv)
    assert Xc.data_ptr() % 16 == 0 and torch.equal(Xc, Xv)
    Xa = torch.tensor(X0, device="cuda")
    assert mde.average_distortion(Xv).item() == mde.average_distortion(Xa).item()


# ------------------------------------------------------------------------------------------------ G2, G3, G4
_FEW = ("pp_fast_mixed", "loss_huber", "pp_quad_invpower")


@gpu
@pytest.mark.parametrize("name", _FEW)
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", ["tiles", "pull4", "pull8", "ell"])
def test_g2_whole_tiles(layout, m, name, monkeypatch):
    import pymde_b200 as pm
    env, want = LAYOUTS[layout]
    _setenv(monkeypatch, GEOMETRIES["G2"][1])
    _setenv(monkeypatch, env)
    _check_case(pm, "G2", m, name, want)


@gpu
@pytest.mark.parametrize("name", _FEW)
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", ["soa", "tiles", "pull4", "ell"])
def test_g3_default_tiles_several_super_tiles(layout, m, name, monkeypatch, record_property):
    import pymde_b200 as pm
    env, want = LAYOUTS[layout]
    _setenv(monkeypatch, GEOMETRIES["G3"][1])
    _setenv(monkeypatch, env)
    _check_case(pm, "G3", m, name, want, record=record_property)


@gpu
@pytest.mark.parametrize("name", ["pp_fast_mixed", "loss_huber"])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("geom,want", [("G4a", 3), ("G4b", 0)])
def test_g4_ell_at_its_tile_limit(geom, want, m, name, monkeypatch):
    """ELL pull records address at most 32 neighbour tiles: 8192 rows of R = 256 build them, 8193 rows fall back to
    the sorted-SoA layout, which must still match the oracle."""
    import pymde_b200 as pm
    _setenv(monkeypatch, GEOMETRIES[geom][1])
    _setenv(monkeypatch, LAYOUTS["ell"][0])
    _check_case(pm, geom, m, name, want)


# ------------------------------------------------------------------------------------------------ G5
def _g5_graph(far):
    """Sparse graph of 300 000 rows whose edges stay within 40 rows, except (with `far`) two edges into neighbour
    tile 5 from owners 10 and 250 000: that bucket's only warp-tile spans 249 990 owner rows."""
    n = 300_000
    rng = np.random.default_rng(55)
    tile5 = (5 * 8192, 6 * 8192)
    i = rng.integers(0, n, 400_000)
    j = np.clip(i + rng.integers(1, 40, len(i)), 0, n - 1)
    e = np.unique(np.sort(np.stack([i, j], 1), axis=1), axis=0)
    e = e[(e[:, 0] != e[:, 1]) & ~((e >= tile5[0]) & (e < tile5[1])).any(1)]
    w = rng.choice([1.0, 2.0, -1.0], len(e)).astype(np.float32)
    if far:
        e = np.concatenate([e, [[10, tile5[0] + 3], [250_000, tile5[0] + 100]]])
        w = np.concatenate([w, [1.0, 1.0]]).astype(np.float32)
    return n, e.astype(np.int64), w


@gpu
@pytest.mark.parametrize("far", [False, True])
def test_g5_pull_owner_offset_overflow(far, monkeypatch, record_property):
    """Pull records store owners as u16 offsets from the warp-tile's first owner.  Without the two far edges the graph
    builds pull records; with them the builder must refuse them (or store them correctly): whatever it builds must
    match the oracle, and the kind is reported."""
    import pymde_b200 as pm
    monkeypatch.setenv("MDE_B200_LAYOUT", "pull")
    n, e, w = _g5_graph(far)
    rng = np.random.default_rng(5)
    X = rng.standard_normal((n, 2)).astype(np.float32)
    for f in (pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log),
              pm.losses.Huber(torch.tensor(np.abs(w), device="cuda"), 0.5)):
        mde = pm.MDE(n, 2, torch.tensor(e, device="cuda"), f, pm.Centered())
        Xg = torch.tensor(X, device="cuda", requires_grad=True)
        v = mde.average_distortion(Xg)
        v.backward()
        kind = _kind(mde)
        record_property("kind", kind)
        print("G5 far=%s %s: kind %d" % (far, type(f).__name__, kind))
        assert kind in ((0, 2) if far else (2,))
        v_ref, g_ref = O.average_distortion(X.astype(np.float64), e, O.spec_from_function(f), True)
        _assert_value(v.item(), v_ref)
        _assert_grad(Xg.grad.cpu().numpy(), g_ref)
        d_ref, _ = O.edge_distances(X.astype(np.float64), e)
        np.testing.assert_allclose(mde.distances(Xg.detach()).cpu().numpy(), d_ref, rtol=1e-6)


# ------------------------------------------------------------------------------------------------ kernel switches
@gpu
@pytest.mark.parametrize("m", [2, 3])
@pytest.mark.parametrize("layout", ["soa", "tiles", "pull4", "ell"])
def test_precise_and_fast_in_one_process(layout, m, monkeypatch):
    """MDE_B200_KERNEL is resolved when a layout is created: a precise layout and a default one built in the same
    process both match the oracle and differ in at least one bit (the default one runs the MUFU kernel), whichever
    kernel ran first in the process."""
    import pymde_b200 as pm
    _setenv(monkeypatch, GEOMETRIES["G1"][1])
    _setenv(monkeypatch, LAYOUTS[layout][0])
    n, e, co, isolated, hubs, X0 = _problem("G1", m)
    X = torch.tensor(X0, device="cuda")

    def run(precise):
        if precise:
            monkeypatch.setenv("MDE_B200_KERNEL", "precise")
        else:
            monkeypatch.delenv("MDE_B200_KERNEL", raising=False)
        f = _function(pm, "pp_fast_mixed", len(e), seed=len(e) + m)
        mde = pm.MDE(n, m, torch.tensor(e, device="cuda"), f, pm.Centered())
        Xg = X.clone().requires_grad_(True)
        v = mde.average_distortion(Xg)
        v.backward()
        assert _kind(mde) == LAYOUTS[layout][1]
        v_ref, g_ref = _reference("G1", m, "pp_fast_mixed", f, e, X0)[:2]
        _assert_value(v.item(), v_ref)
        _assert_grad(Xg.grad.cpu().numpy(), g_ref)
        # the fp64 sum of the per-edge values the kernel left in the layout: summed in a fixed order (no atomics), so
        # the same kernel gives the same bits; the fp32 value returned to the caller is too coarse to tell them apart
        return mde._layout().loss.item()

    fast, precise, fast2 = run(False), run(True), run(False)
    assert fast == fast2
    assert fast != precise, "MDE_B200_KERNEL=precise did not change the kernel"


# ------------------------------------------------------------------------------------------------ oracle self-check
def test_dropped_edges_fail_the_gradient_check():
    """The gradient tolerance is tight enough to see one missing edge: dropping the edge at row n - 1, or one hub edge
    into the last (partial) tile, from the oracle's input must fail the check the GPU tests apply."""
    m = 2
    n, e, co, isolated, hubs, X0 = _problem("G1", m)
    rng = np.random.default_rng(len(e) + m)
    w = rng.choice([1.0, 2.0, -1.0], len(e)).astype(np.float32)
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    X64 = X0.astype(np.float64)
    v_ref, g_ref = O.average_distortion(X64, e, spec, True)
    _assert_grad(g_ref.astype(np.float32), g_ref)  # an fp32 rounding of the truth passes
    assert not np.any(g_ref[isolated])
    last_tile = (n - 1) // 256 * 256
    at_last_row = np.flatnonzero((e == n - 1).any(1))
    hub_last = np.flatnonzero(np.isin(e, hubs).any(1) & (e >= last_tile).any(1) & ~np.isin(e, [n - 1]).any(1))
    assert len(at_last_row) and len(hub_last)
    for k in (at_last_row[0], hub_last[0]):
        keep = np.ones(len(e), bool)
        keep[k] = False
        sub = O.FnSpec(O.P_LOG1P, w[keep], (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
        _, g_drop = O.average_distortion(X64, e[keep], sub, True, p_total=len(e))
        with pytest.raises(AssertionError):
            _assert_grad(g_drop.astype(np.float32), g_ref)
