"""`embed_new_points` on graphs, and the row-range graph k-NN search under it (`mde_graph_knn_rows`).

The row search must give the rows of the full search (`mde_graph_knn`) bit for bit, on every kind of graph, range and
batch size, and both row searches (device and host) must equal an fp64 scipy Dijkstra oracle with the (length, node
index) tie-break.  The recipe keeps the fitted nodes where they are, repeats bit for bit under
MDE_B200_DETERMINISTIC=1, never runs a full search, and places new nodes of a 10-community stochastic block model as
well as the reference workflow does: `preserve_neighbors` on the union graph with every fitted node anchored
(reference docs, "Embedding new points").  The score is the share of new nodes whose nearest fitted point in the
embedding is in their community.

Measured on an H100 80GB HBM3 (700 W power limit), 20 000 fitted and 2 000 new nodes: unweighted 1.000 for
`embed_new_points` and 1.000 for the reference workflow; weights in [0.5, 1.5]: 0.999 and 0.999.  The floor (0.95) and
the margin (0.02 below the reference workflow) leave room for noise."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

pytestmark = pytest.mark.gpu

N_OLD, N_NEW, COMMUNITIES = 20000, 2000, 10
FLOOR, MARGIN = 0.95, 0.02


def _lib():
    from pymde_b200 import _lib
    return _lib, _lib.load()


def _sym(e, w, n):
    e = np.asarray(e, dtype=np.int64)
    lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
    keep = lo != hi
    key, first = np.unique(lo[keep] * n + hi[keep], return_index=True)
    w = np.asarray(w, dtype=np.float32)[keep][first]
    U = sp.coo_matrix((w, (key // n, key % n)), shape=(n, n)).tocsr()
    return (U + U.T).tocsr()


def _geometric(n, k, seed, weighted=True, isolated=0, components=1):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 2))
    pts[:, 0] += 10.0 * (np.arange(n) % components)
    _, idx = cKDTree(pts).query(pts, k=k + 1)
    e = np.stack([np.repeat(np.arange(n), k), idx[:, 1:].ravel()], 1)
    e = e[(e < n - isolated).all(1)]
    w = np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1) if weighted else np.ones(len(e))
    return _sym(e, w, n)


def _sbm(n, seed, weighted, labels=None, d_in=6, d_out=0.4):
    """Stochastic block model: about d_in edges per node inside its community and d_out to uniform nodes."""
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, COMMUNITIES, n) if labels is None else labels
    members = [np.flatnonzero(lab == c) for c in range(COMMUNITIES)]
    src = np.repeat(np.arange(n), d_in)
    dst = np.empty_like(src)
    for c in range(COMMUNITIES):
        sel = lab[src] == c
        dst[sel] = rng.choice(members[c], sel.sum())
    n_out = int(d_out * n)
    e = np.concatenate([np.stack([src, dst], 1), rng.integers(0, n, (n_out, 2))])
    w = rng.uniform(0.5, 1.5, len(e)) if weighted else np.ones(len(e))
    return _sym(e, w, n), lab


def _path(n, seed):
    rng = np.random.default_rng(seed)
    e = np.stack([np.arange(n - 1), np.arange(1, n)], 1)
    return _sym(e, rng.uniform(0.5, 1.5, n - 1), n)


def _lattice(side):
    """Unit-weight grid: a great many equal lengths."""
    v = np.arange(side * side).reshape(side, side)
    e = np.concatenate([np.stack([v[:, :-1].ravel(), v[:, 1:].ravel()], 1),
                        np.stack([v[:-1].ravel(), v[1:].ravel()], 1)])
    return _sym(e, np.ones(len(e)), side * side)


GRAPHS = {
    "geometric": lambda: _geometric(3000, 8, 0, isolated=5, components=2),
    "geometric_unweighted": lambda: _geometric(3000, 5, 1, weighted=False, isolated=3),
    "sbm": lambda: _sbm(3000, 2, True)[0],
    "sbm_unweighted": lambda: _sbm(3000, 3, False)[0],
    "path": lambda: _path(1200, 4),
    "components": lambda: _geometric(2000, 4, 5, isolated=40, components=7),
    "lattice": lambda: _lattice(50),
}


def _unweighted(A):
    return bool((A.data == 1.0).all())


def _device(A):
    from pymde_b200.preprocess import graph as G
    dev = torch.device("cuda", 0)
    indptr, indices, w = G._device_csr(A, dev)
    return indptr, indices, (None if _unweighted(A) else w)


def _stream():
    from pymde_b200 import util
    return util.stream_ptr(torch.device("cuda", 0))


def _full(csr, n, k, md):
    _l, lib = _lib()
    indptr, indices, w = csr
    ws = torch.empty(int(lib.mde_graph_knn_ws_bytes(n, (n + 31) // 32 * 32)), dtype=torch.uint8, device="cuda")
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    ln = torch.empty((n, k), dtype=torch.float32, device="cuda")
    _l.check(lib.mde_graph_knn(indptr.data_ptr(), indices.data_ptr(), None if w is None else w.data_ptr(), n, k, md,
                               idx.data_ptr(), ln.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
    return idx.cpu().numpy(), ln.cpu().numpy()


def _rows(csr, n, k, md, s0, s1, batch=None):
    """mde_graph_knn_rows; `batch` forces a workspace of exactly that batch (default: all rows in one batch)."""
    _l, lib = _lib()
    indptr, indices, w = csr
    b = batch or max(32, (s1 - s0 + 31) // 32 * 32)
    ws = torch.empty(int(lib.mde_graph_knn_ws_bytes(n, b)), dtype=torch.uint8, device="cuda")
    idx = torch.full((s1 - s0, k), -7, dtype=torch.int32, device="cuda")
    ln = torch.full((s1 - s0, k), -7.0, dtype=torch.float32, device="cuda")
    _l.check(lib.mde_graph_knn_rows(indptr.data_ptr(), indices.data_ptr(), None if w is None else w.data_ptr(), n, s0,
                                    s1, k, md, idx.data_ptr(), ln.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
    return idx.cpu().numpy(), ln.cpu().numpy()


def _radius(A):
    return float(3 * np.quantile(sp.triu(A).data, 0.75))


# 1. the row search gives the full search's rows ----------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_rows_equal_the_full_search(name):
    A = GRAPHS[name]()
    n = A.shape[0]
    csr = _device(A)
    for md in (0.0, _radius(A)):
        for k in (1, 15, 64):
            want_i, want_l = _full(csr, n, k, md)
            for s0, s1, batch in [(0, n, None), (n - 1, n, None), (30, 97, None), (31, 33, None),
                                  (n // 2 - 40, n // 2 + 300, 64), (5, 200, 32), (n - 130, n, 32)]:
                got_i, got_l = _rows(csr, n, k, md, s0, s1, batch)
                assert np.array_equal(got_i, want_i[s0:s1]), (name, md, k, s0, s1, batch)
                assert np.array_equal(got_l.view(np.int32), want_l[s0:s1].view(np.int32)), (name, md, k, s0, s1)


def test_rows_straddle_the_full_searchs_batches():
    """The full search in batches of 64 and a row search in batches of 96 starting off any batch boundary."""
    _l, lib = _lib()
    A = GRAPHS["geometric"]()
    n = A.shape[0]
    csr = _device(A)
    indptr, indices, w = csr
    ws = torch.empty(int(lib.mde_graph_knn_ws_bytes(n, 64)), dtype=torch.uint8, device="cuda")
    idx = torch.empty((n, 15), dtype=torch.int32, device="cuda")
    ln = torch.empty((n, 15), dtype=torch.float32, device="cuda")
    _l.check(lib.mde_graph_knn(indptr.data_ptr(), indices.data_ptr(), w.data_ptr(), n, 15, 0.0, idx.data_ptr(),
                               ln.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
    for s0, s1 in [(63, 65), (100, 1000), (127, 1153)]:
        got_i, got_l = _rows(csr, n, 15, 0.0, s0, s1, batch=96)
        assert np.array_equal(got_i, idx[s0:s1].cpu().numpy()) and np.array_equal(got_l, ln[s0:s1].cpu().numpy())


# 2. both row searches against fp64 Dijkstra ----------------------------------------------------------------------------
def _oracle(A, k, limit, s0, s1):
    D = csgraph.dijkstra(A.astype(np.float64), directed=False, indices=np.arange(s0, s1),
                         limit=np.inf if not limit else limit)
    D[np.arange(s1 - s0), np.arange(s0, s1)] = np.inf
    order = np.argsort(D, axis=1, kind="stable")[:, :k]
    d = np.take_along_axis(D, order, 1)
    return np.where(np.isfinite(d), order, -1).astype(np.int32), d.astype(np.float32)


@pytest.mark.parametrize("name", ["geometric", "sbm_unweighted", "path", "lattice"])
def test_row_searches_match_dijkstra(name):
    from pymde_b200.preprocess import graph as G
    A = GRAPHS[name]()
    n = A.shape[0]
    g = G.Graph(A)
    for md in (None, _radius(A)):
        for k in (1, 15, 64, 100):
            for s0, s1 in [(0, 37), (n - 300, n)]:
                want_i, want_l = _oracle(A, k, md, s0, s1)
                hi, hl = G.knn_rows_host(g, k, s0, s1, max_distance=md)
                assert np.array_equal(hi, want_i) and np.array_equal(hl, want_l), (name, md, k, s0, s1)
                if k <= 64:
                    di, dl = G.knn_rows_device(g, k, s0, s1, max_distance=md, device="cuda")
                    assert di.is_cuda and di.shape == (s1 - s0, k)
                    assert np.array_equal(di.cpu().numpy(), want_i), (name, md, k, s0, s1)
                    assert np.array_equal(dl.cpu().numpy(), want_l), (name, md, k, s0, s1)
    with pytest.raises(ValueError):
        G.knn_rows_device(g, 65, 0, 10, device="cuda")


# 3. the recipe ---------------------------------------------------------------------------------------------------------
def _split(A, n_old):
    from pymde_b200.preprocess import Graph
    U = sp.triu(A, k=1).tocoo()
    old = (U.row < n_old) & (U.col < n_old)
    e = np.stack([U.row, U.col], 1)
    return (Graph.from_edges(e[old], U.data[old], n_items=n_old),
            Graph.from_edges(e[~old], U.data[~old], n_items=A.shape[0]))


def _fit(weighted):
    import pymde_b200 as pm
    A, lab = _sbm(N_OLD + N_NEW, 11 if weighted else 12, weighted)
    data, new = _split(A, N_OLD)
    pm.seed(0)
    emb = pm.preserve_neighbors(data).embed()
    return A, lab, data, new, emb


@pytest.fixture(scope="module")
def fitted():
    return _fit(False)


@pytest.fixture(scope="module")
def fitted_weighted():
    return _fit(True)


def _score(emb, lab, out):
    nearest = torch.cdist(out.double(), emb.double()).argmin(1).cpu().numpy()
    return float((lab[:N_OLD][nearest] == lab[N_OLD:N_OLD + out.shape[0]]).mean())


def test_anchors_stay_and_no_full_search_runs(fitted, monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    from pymde_b200.preprocess import generic
    from pymde_b200.preprocess import graph as G

    def refuse(*a, **kw):
        raise AssertionError("a full graph k-NN search ran")

    for mod, name in ((G, "k_nearest_neighbors_device"), (G, "k_nearest_neighbors"),
                      (generic, "k_nearest_neighbors"), (pm.preprocess, "k_nearest_neighbors")):
        if hasattr(mod, name):
            monkeypatch.setattr(mod, name, refuse)
    A, lab, data, new, emb = fitted
    mde, items = recipes._new_points_mde(data, emb, new)
    assert torch.equal(items[:N_NEW].cpu(), torch.arange(N_OLD, N_OLD + N_NEW))
    X = mde.embed()
    assert torch.equal(X[N_NEW:], emb[items[N_NEW:]])
    assert X.shape[1] == 2 and bool(torch.isfinite(X).all())
    assert mde.n_items < N_OLD + N_NEW
    out = pm.embed_new_points(data, emb, new)
    assert out.shape == (N_NEW, 2) and out.dtype == torch.float32 and out.is_cuda


def test_lists_are_the_full_searchs_rows(fitted):
    """The recipe's lists are rows n_old .. n - 1 of the full device search on the union graph, at the default
    radius, and the host route gives the same lists."""
    from pymde_b200 import recipes
    A, lab, data, new, emb = fitted
    n = N_OLD + N_NEW
    got = recipes._graph_new_lists(data, new, 15, None, torch.device("cuda", 0)).cpu().numpy()
    md = float(3 * torch.quantile(recipes.Graph(A).distances, 0.75))
    want_i, _ = _full(_device(A), n, 15, md)
    assert np.array_equal(got, want_i[N_OLD:])
    host = recipes._graph_new_lists(data, new, 15, md, torch.device("cuda", 0))
    assert np.array_equal(host.cpu().numpy(), got)


def test_host_route_gives_the_same_lists(fitted, monkeypatch):
    from pymde_b200 import recipes
    A, lab, data, new, emb = fitted
    dev = torch.device("cuda", 0)
    want = recipes._graph_new_lists(data, new, 15, None, dev)
    monkeypatch.setenv("PYMDE_B200_SHORTEST_PATHS", "host")
    got = recipes._graph_new_lists(data, new, 15, None, dev)
    assert got.is_cuda and torch.equal(got, want)


def test_deterministic_mode_repeats_bit_for_bit(fitted, monkeypatch):
    import pymde_b200 as pm
    A, lab, data, new, emb = fitted
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    pm.seed(0)
    a = pm.embed_new_points(data, emb, new)
    pm.seed(0)
    b = pm.embed_new_points(data, emb, new)
    assert a.shape == (N_NEW, 2) and torch.equal(a, b)


@pytest.mark.parametrize("weighted", [False, True])
def test_quality_against_the_reference_workflow(weighted, request):
    import pymde_b200 as pm
    A, lab, data, new, emb = request.getfixturevalue("fitted_weighted" if weighted else "fitted")
    pm.seed(0)
    ours = pm.embed_new_points(data, emb, new)
    acc = _score(emb, lab, ours)
    pm.seed(0)
    ref = pm.preserve_neighbors(pm.Graph(A), constraint=pm.Anchored(torch.arange(N_OLD, device="cuda"), emb)).embed()
    acc_ref = _score(emb, lab, ref[N_OLD:])
    print("weighted=%s accuracy: embed_new_points %.4f, reference workflow %.4f" % (weighted, acc, acc_ref))
    assert acc >= FLOOR, (acc, acc_ref)
    assert acc >= acc_ref - MARGIN, (acc, acc_ref)


def test_one_and_zero_new_nodes(fitted):
    import pymde_b200 as pm
    A, lab, data, new, emb = fitted
    one = _split(A[:N_OLD + 1, :N_OLD + 1], N_OLD)[1]
    out = pm.embed_new_points(data, emb, one)
    assert out.shape == (1, 2) and bool(torch.isfinite(out).all())
    none = pm.Graph.from_edges(np.zeros((0, 2), dtype=np.int64), n_items=N_OLD)
    out = pm.embed_new_points(data, emb, none)
    assert out.shape == (0, 2) and out.dtype == torch.float32


def test_isolated_and_indirectly_reached_new_nodes(fitted):
    """New node a touches fitted nodes; b touches only a, c only b; d has no edge at all."""
    import pymde_b200 as pm
    A, lab, data, new, emb = fitted
    a, b, c, d = N_OLD, N_OLD + 1, N_OLD + 2, N_OLD + 3
    e = np.array([[a, 0], [a, 1], [a, 2], [b, a], [c, b]])
    g = pm.Graph.from_edges(e, n_items=N_OLD + 4)
    for kw in ({}, {"max_distance": np.inf}, {"max_distance": 2.0}, {"repulsive_penalty": None}):
        pm.seed(0)
        out = pm.embed_new_points(data, emb, g, **kw)
        assert out.shape == (4, 2) and bool(torch.isfinite(out).all()), kw


def test_options(fitted_weighted):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    A, lab, data, new, emb = fitted_weighted
    pm.seed(0)
    out = pm.embed_new_points(data, emb, new, repulsive_penalty=None)
    assert out.shape == (N_NEW, 2) and bool(torch.isfinite(out).all())
    assert _score(emb, lab, out) >= FLOOR - 0.05
    # a small explicit radius leaves fewer attractive edges than the default one
    mde_small, _ = recipes._new_points_mde(data, emb, new, max_distance=0.6)
    mde_def, _ = recipes._new_points_mde(data, emb, new)
    n_small = int((mde_small.distortion_function.weights > 0).sum())
    n_def = int((mde_def.distortion_function.weights > 0).sum())
    assert n_small < n_def
    out = pm.embed_new_points(data, emb, new, max_distance=0.6, n_neighbors=70)  # k > 64: the host route
    assert out.shape == (N_NEW, 2) and bool(torch.isfinite(out).all())
