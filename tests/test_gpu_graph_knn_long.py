"""Graph k-nearest neighbours for 1 <= k <= 256 on the device (`mde_graph_knn_long`, `mde_graph_knn_long_rows`) and
the routes that use them: `graph.k_nearest_neighbors_device_long`, `graph.knn_rows_device_long`, `preserve_neighbors`
and `laplacian_embedding` on a Graph, and `embed_new_points` on Graphs.

Every list must equal an fp64 scipy Dijkstra oracle with the (length, node index) order (`graph.knn_rows_host`), in
indices and in fp32 lengths, bit for bit; for k <= 64 it must equal `mde_graph_knn`.  The selection sorts segments of
up to LONG_SMEM keys in shared memory and radix-selects longer ones in global memory, so stars whose centre's segment
sits just below, at and above that size exercise both paths and the switch between them, with every length tied."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

pytestmark = pytest.mark.gpu

LONG_SMEM = 2048  # kLongSmem in mde_graph.cu
KS = (1, 15, 64, 65, 100, 256)


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


def _sbm(n, seed, weighted, communities=10, d_in=6, d_out=0.4):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, communities, n)
    members = [np.flatnonzero(lab == c) for c in range(communities)]
    src = np.repeat(np.arange(n), d_in)
    dst = np.empty_like(src)
    for c in range(communities):
        sel = lab[src] == c
        dst[sel] = rng.choice(members[c], sel.sum())
    e = np.concatenate([np.stack([src, dst], 1), rng.integers(0, n, (int(d_out * n), 2))])
    w = rng.uniform(0.5, 1.5, len(e)) if weighted else np.ones(len(e))
    return _sym(e, w, n)


def _path(n, seed):
    rng = np.random.default_rng(seed)
    return _sym(np.stack([np.arange(n - 1), np.arange(1, n)], 1), rng.uniform(0.5, 1.5, n - 1), n)


def _lattice(side):
    v = np.arange(side * side).reshape(side, side)
    e = np.concatenate([np.stack([v[:, :-1].ravel(), v[:, 1:].ravel()], 1),
                        np.stack([v[:-1].ravel(), v[1:].ravel()], 1)])
    return _sym(e, np.ones(len(e)), side * side)


def _star(n, weight=1.0):
    """Node 0 joined to every other node: its segment holds n - 1 nodes at one length, a leaf's n - 1 nodes at two."""
    return _sym(np.stack([np.zeros(n - 1, dtype=np.int64), np.arange(1, n)], 1), np.full(n - 1, weight), n)


GRAPHS = {
    "geometric": lambda: _geometric(3000, 8, 0, isolated=5, components=2),
    "sbm_unweighted": lambda: _sbm(3000, 3, False),
    "path": lambda: _path(1200, 4),
    "lattice": lambda: _lattice(50),
    "small": lambda: _geometric(150, 6, 6, isolated=2),   # k >= n - 1: padded rows
}


def _unweighted(A):
    return bool((A.data == 1.0).all())


def _device(A):
    from pymde_b200.preprocess import graph as G
    indptr, indices, w = G._device_csr(A, torch.device("cuda", 0))
    return indptr, indices, (None if _unweighted(A) else w)


def _stream():
    from pymde_b200 import util
    return util.stream_ptr(torch.device("cuda", 0))


def _search(csr, n, k, md, long=True, rows=None, batch=None):
    """mde_graph_knn(_long) or, with rows = (s0, s1), mde_graph_knn(_long)_rows; `batch` forces a workspace of exactly
    that batch (default: every source in one batch).  numpy (idx, len)."""
    _l, lib = _lib()
    indptr, indices, w = csr
    s0, s1 = rows or (0, n)
    b = batch or max(32, (s1 - s0 + 31) // 32 * 32)
    ws = torch.empty(int(lib.mde_graph_knn_ws_bytes(n, b)), dtype=torch.uint8, device="cuda")
    idx = torch.full((s1 - s0, k), -7, dtype=torch.int32, device="cuda")
    ln = torch.full((s1 - s0, k), -7.0, dtype=torch.float32, device="cuda")
    wp = None if w is None else w.data_ptr()
    tail = (md, idx.data_ptr(), ln.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    if rows is None:
        fn = lib.mde_graph_knn_long if long else lib.mde_graph_knn
        _l.check(fn(indptr.data_ptr(), indices.data_ptr(), wp, n, k, *tail))
    else:
        fn = lib.mde_graph_knn_long_rows if long else lib.mde_graph_knn_rows
        _l.check(fn(indptr.data_ptr(), indices.data_ptr(), wp, n, s0, s1, k, *tail))
    return idx.cpu().numpy(), ln.cpu().numpy()


def _oracle(A, md, k=256, s0=0, s1=None):
    """scipy Dijkstra and the (fp64 length, node index) order: `knn_rows_host`.  Its first k' columns are the k'-lists."""
    from pymde_b200.preprocess import graph as G
    return G.knn_rows_host(G.Graph(A), k, s0, A.shape[0] if s1 is None else s1, max_distance=md or None)


def _same(got, want, what):
    gi, gl = got
    wi, wl = want
    assert np.array_equal(gi, wi), what
    assert np.array_equal(gl.view(np.int32), wl.view(np.int32)), what


def _radius(A):
    return float(3 * np.quantile(sp.triu(A).data, 0.75))


# 1. against the fp64 oracle, and 2. against the k <= 64 search --------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_long_search_matches_dijkstra(name):
    A = GRAPHS[name]()
    n = A.shape[0]
    csr = _device(A)
    for md in (0.0, _radius(A)):
        wi, wl = _oracle(A, md)
        for k in KS:
            want = (wi[:, :k], wl[:, :k])
            full = _search(csr, n, k, md)
            _same(full, want, (name, md, k))
            for s0, s1 in [(0, 37), (n // 3, min(n, n // 3 + 200)), (n - 90, n)]:
                _same(_search(csr, n, k, md, rows=(s0, s1)), (wi[s0:s1, :k], wl[s0:s1, :k]), (name, md, k, s0, s1))
            if k <= 64:
                _same(_search(csr, n, k, md, long=False), full, (name, md, k, "mde_graph_knn"))


# 3. batches -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["geometric", "sbm_unweighted"])
def test_batches_give_the_same_lists(name):
    A = GRAPHS[name]()
    n = A.shape[0]
    csr = _device(A)
    for k in (15, 100, 256):
        one = _search(csr, n, k, 0.0)
        for batch in (32, 64):
            _same(_search(csr, n, k, 0.0, batch=batch), one, (name, k, batch))
        for s0, s1, batch in [(31, 33, 32), (63, 65, 64), (100, 1000, 96), (127, 1153, 32), (n - 70, n, 64)]:
            _same(_search(csr, n, k, 0.0, rows=(s0, s1), batch=batch), (one[0][s0:s1], one[1][s0:s1]),
                  (name, k, s0, s1, batch))


# 4. both selection paths, and ties ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [LONG_SMEM, LONG_SMEM + 1, LONG_SMEM + 2, 3 * LONG_SMEM + 17])
@pytest.mark.parametrize("weight", [1.0, 0.37])
def test_star_segments_around_the_shared_memory_capacity(n, weight):
    """The centre's segment holds n - 1 = LONG_SMEM - 1 .. LONG_SMEM + 1 (and 3 LONG_SMEM + 16) nodes, all at one
    length; a leaf's holds the centre at one length and n - 2 nodes tied at twice it."""
    A = _star(n, weight)
    csr = _device(A)
    wi, wl = _oracle(A, 0.0)
    for k in (1, 64, 65, 256):
        got = _search(csr, n, k, 0.0)
        _same(got, (wi[:, :k], wl[:, :k]), (n, weight, k))
        assert np.array_equal(got[0][0], np.arange(1, k + 1)), (n, k)  # the lowest indices among the tied leaves
        for s in (0, 1, n - 1):
            _same(_search(csr, n, k, 0.0, rows=(s, s + 1)), (wi[s:s + 1, :k], wl[s:s + 1, :k]), (n, weight, k, s))


def test_unweighted_lattice_ties():
    """Hop counts on a 200 x 200 grid: the k-th length is shared by up to ~4 x radius nodes."""
    A = _lattice(200)
    n = A.shape[0]
    csr = _device(A)
    rows = (n // 2 - 300, n // 2 + 300)
    for md in (0.0, 12.0):
        wi, wl = _oracle(A, md, 256, *rows)
        for k in (65, 100, 256):
            _same(_search(csr, n, k, md, rows=rows), (wi[:, :k], wl[:, :k]), (md, k))


# 5. the graph builder -------------------------------------------------------------------------------------------------
def test_builder_equals_the_host_knn_graph():
    from pymde_b200.preprocess import graph as G
    A = _geometric(3000, 8, 7)
    g = G.Graph(A)
    for md in (None, _radius(A)):
        got = G.k_nearest_neighbors_device_long(g, 100, max_distance=md, device="cuda")
        want = G.k_nearest_neighbors(g, 100, max_distance=md)
        assert isinstance(got, G.EdgeListGraph) and got.edges.is_cuda
        assert torch.equal(got.edges.cpu(), want.edges) and torch.equal(got.weights.cpu(), want.weights), md
        if md is None:
            assert got.n_edges >= 3000 * 50  # 100 entries per node


# 6. recipes -----------------------------------------------------------------------------------------------------------
def _refuse_host(monkeypatch):
    from pymde_b200.preprocess import graph as G

    def refuse(*a, **kw):
        raise AssertionError("a host shortest-path search ran")

    monkeypatch.setattr(csgraph, "dijkstra", refuse)
    monkeypatch.setattr(G, "k_nearest_neighbors", refuse)
    monkeypatch.setattr(G, "knn_rows_host", refuse)


@pytest.mark.parametrize("max_distance", [None, np.inf])
@pytest.mark.parametrize("recipe", ["preserve_neighbors", "laplacian_embedding"])
def test_recipes_build_on_the_device(recipe, max_distance, monkeypatch):
    """At the default radius (None) most lists end inside it; unlimited, every node has 100 neighbours."""
    import pymde_b200 as pm
    g = pm.Graph(_geometric(4000, 8, 9))  # continuous weights: no tied lengths

    def build():
        pm.seed(0)
        return getattr(pm, recipe)(g, embedding_dim=2, n_neighbors=100, max_distance=max_distance, device="cuda")

    with monkeypatch.context() as m:
        _refuse_host(m)
        dev = build()
    m2 = pytest.MonkeyPatch()
    m2.setenv("PYMDE_B200_SHORTEST_PATHS", "host")
    try:
        host = build()
    finally:
        m2.undo()
    assert torch.equal(dev.edges, host.edges.to(dev.edges.device))
    assert torch.equal(dev.distortion_function.weights, host.distortion_function.weights.to(dev.edges.device))
    if max_distance is not None:
        assert int((dev.distortion_function.weights > 0).sum()) >= 4000 * 50
    dev.embed(max_iter=30)
    st = dev.solve_stats
    if recipe == "preserve_neighbors":
        assert st.average_distortions[-1] < st.average_distortions[0]
    else:  # the spectral initialisation is already the Laplacian embedding's optimum
        assert st.average_distortions[-1] <= st.average_distortions[0] * (1 + 1e-4), st.average_distortions


# 7. new points --------------------------------------------------------------------------------------------------------
N_OLD, N_NEW = 8000, 800


def _split(A, n_old):
    from pymde_b200.preprocess import Graph
    U = sp.triu(A, k=1).tocoo()
    old = (U.row < n_old) & (U.col < n_old)
    e = np.stack([U.row, U.col], 1)
    return (Graph.from_edges(e[old], U.data[old], n_items=n_old),
            Graph.from_edges(e[~old], U.data[~old], n_items=A.shape[0]))


@pytest.fixture(scope="module", params=["sbm_unweighted", "sbm_weighted"])
def fitted(request):
    import pymde_b200 as pm
    A = _sbm(N_OLD + N_NEW, 21, request.param == "sbm_weighted")
    data, new = _split(A, N_OLD)
    pm.seed(0)
    emb = pm.preserve_neighbors(data).embed()
    return A, data, new, emb


def test_new_points_at_k_100(fitted, monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    from pymde_b200.preprocess import graph as G
    A, data, new, emb = fitted
    md = float(3 * torch.quantile(torch.cat([data.distances, new.distances]), 0.75))
    want, _ = G.knn_rows_host(G.Graph(A), 100, N_OLD, N_OLD + N_NEW, max_distance=md)
    _refuse_host(monkeypatch)

    def refuse(*a, **kw):
        raise AssertionError("a full graph k-NN search ran")

    monkeypatch.setattr(G, "k_nearest_neighbors_device", refuse)
    monkeypatch.setattr(G, "k_nearest_neighbors_device_long", refuse)
    got = recipes._graph_new_lists(data, new, 100, None, torch.device("cuda", 0))
    assert got.is_cuda and np.array_equal(got.cpu().numpy(), want)
    mde, items = recipes._new_points_mde(data, emb, new, n_neighbors=100)
    X = mde.embed()
    assert torch.equal(X[N_NEW:], emb[items[N_NEW:]])
    assert bool(torch.isfinite(X).all())
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    pm.seed(0)
    a = pm.embed_new_points(data, emb, new, n_neighbors=100)
    pm.seed(0)
    b = pm.embed_new_points(data, emb, new, n_neighbors=100)
    assert a.shape == (N_NEW, 2) and torch.equal(a, b)
