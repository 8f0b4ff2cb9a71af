"""CPU: the row-range graph k-nearest-neighbour search (`mde_graph_knn_rows`, include/mde_b200.h) is exported, additive
(the ABI version is still 1), reuses `mde_graph_knn_ws_bytes` and refuses bad arguments before any launch; the host
row search picks the (fp64 length, node index) smallest pairs; and `embed_new_points` on Graphs assembles the union
of the two graphs and rejects bad input before it touches a device."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null: never dereferenced, every call below returns before a CUDA call


def _call(n=1000, s_begin=0, s_end=10, k=5, indptr=FAKE, indices=FAKE, weights=FAKE, out_i=FAKE, out_d=FAKE,
          ws=FAKE, ws_bytes=None, max_distance=0.0):
    lib = _lib.load()
    if ws_bytes is None:
        ws_bytes = int(lib.mde_graph_knn_ws_bytes(n, 32)) if 1 <= n < (1 << 31) else 1 << 40
    return lib.mde_graph_knn_rows(indptr, indices, weights, n, s_begin, s_end, k, max_distance, out_i, out_d, ws,
                                  ws_bytes, None)


def test_symbol_is_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    assert "mde_graph_knn_rows" in _lib.SIGNATURES and lib.mde_graph_knn_rows is not None
    assert "int mde_graph_knn_rows(" in header
    assert "mde_graph_knn_rows_ws_bytes" not in header  # the full search's size function serves both


def test_bad_arguments_are_rejected_without_a_launch():
    lib = _lib.load()
    INVALID = _lib.MDE_E_INVALID
    launches = int(lib.mde_launch_count())
    max_k = int(lib.mde_graph_knn_max_k())
    assert max_k == 64
    for kw in ("indptr", "indices", "out_i", "out_d", "ws"):
        assert _call(**{kw: None}) == INVALID, kw
    for n in (0, -1, 1 << 31):
        assert _call(n=n, s_end=0) == INVALID, n
    for s_begin, s_end in [(-1, 5), (0, 1001), (999, 1001), (6, 5), (1000, 999)]:
        assert _call(s_begin=s_begin, s_end=s_end) == INVALID, (s_begin, s_end)
    for k in (0, -1, max_k + 1, 1000):
        assert _call(k=k) == INVALID, k
    need = int(lib.mde_graph_knn_ws_bytes(1000, 32))
    assert _call(ws_bytes=need - 1) == INVALID
    assert _call(ws_bytes=0) == INVALID
    # an empty range is checked like any other
    assert _call(s_begin=7, s_end=7, k=0) == INVALID
    assert _call(s_begin=7, s_end=7, ws_bytes=need - 1) == INVALID
    assert _call(s_begin=7, s_end=7, out_i=None) == INVALID
    assert int(lib.mde_launch_count()) == launches


def test_an_empty_range_returns_without_a_launch():
    lib = _lib.load()
    launches = int(lib.mde_launch_count())
    for n, s in [(1000, 0), (1000, 500), (1000, 1000), (1, 0), (1, 1)]:
        assert _call(n=n, s_begin=s, s_end=s) == 0, (n, s)
    # weights NULL (unit weights) is allowed; a finite radius changes nothing about the checks
    assert _call(s_begin=3, s_end=3, weights=None, max_distance=2.5) == 0
    assert _call(s_begin=3, s_end=3, k=64) == 0
    assert int(lib.mde_launch_count()) == launches


@pytest.mark.parametrize("n", [1, 33, 1000, 10 ** 6])
def test_workspace_size_is_the_full_searchs(n):
    lib = _lib.load()
    need = int(lib.mde_graph_knn_ws_bytes(n, 32))
    assert need == int(lib.mde_graph_sssp_ws_bytes(n, 32)) > 0
    assert _call(n=n, s_begin=0, s_end=0, ws_bytes=need) == 0
    assert _call(n=n, s_begin=0, s_end=0, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    # the tile is n B entries whatever the row count: the size grows with n and the batch, in steps of 32
    sizes = [int(lib.mde_graph_knn_ws_bytes(n, b)) for b in (32, 64, 96, 1024)]
    assert all(b > a for a, b in zip(sizes, sizes[1:]))
    assert sizes[1] - sizes[0] >= n * 32 * (4 * 8 + 4)
    assert int(lib.mde_graph_knn_ws_bytes(n, 48)) < 0


# ---- the host row search ----------------------------------------------------------------------------------------------
def _lex_oracle(D, rows, k):
    """Stable argsort restatement: per row the k smallest (length, column) pairs, the row's own node excluded."""
    D = D.copy()
    D[np.arange(len(rows)), rows] = np.inf
    order = np.argsort(D, axis=1, kind="stable")[:, :k]
    d = np.take_along_axis(D, order, 1)
    if order.shape[1] < k:
        pad = k - order.shape[1]
        order = np.pad(order, ((0, 0), (0, pad)))
        d = np.pad(d, ((0, 0), (0, pad)), constant_values=np.inf)
    return np.where(np.isfinite(d), order, -1).astype(np.int32), d


@pytest.mark.parametrize("k", [1, 3, 15, 64, 100])
def test_smallest_pairs_break_ties_by_index(k):
    from pymde_b200.preprocess.graph import _smallest_pairs
    rng = np.random.default_rng(k)
    for n, c in [(40, 7), (200, 30), (1000, 5)]:
        D = rng.integers(0, 6, (c, n)).astype(np.float64)  # many ties
        D[rng.random((c, n)) < 0.3] = np.inf
        D[0, :] = np.inf                                     # a row that reaches nothing
        D[1, :] = 1.0                                        # a row of equal lengths
        rows = rng.integers(0, n, c)
        got_i, got_d = _smallest_pairs(D, rows, k)
        want_i, want_d = _lex_oracle(D, rows, k)
        assert np.array_equal(got_i, want_i), (n, c)
        assert np.array_equal(got_d, want_d), (n, c)


def _geometric(n, k, seed, weighted=True, isolated=0):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 2))
    _, idx = cKDTree(pts).query(pts, k=k + 1)
    e = np.unique(np.sort(np.stack([np.repeat(np.arange(n), k), idx[:, 1:].ravel()], 1), axis=1), axis=0)
    e = e[(e < n - isolated).all(1)]
    w = np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1).astype(np.float32) if weighted else np.ones(len(e))
    U = sp.coo_matrix((w.astype(np.float32), (e[:, 0], e[:, 1])), shape=(n, n)).tocsr()
    return (U + U.T).tocsr()


@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("limit", [None, 0.08, np.inf])
def test_host_row_search_matches_dijkstra(weighted, limit):
    from pymde_b200.preprocess import graph as G
    n = 600
    A = _geometric(n, 5, 1, weighted=weighted, isolated=4)
    lim = 3.0 if (limit == 0.08 and not weighted) else limit
    D = csgraph.dijkstra(A.astype(np.float64), directed=False, limit=np.inf if lim is None else lim)
    for k in (1, 15, 64, 80):
        for s_begin, s_end in [(0, n), (n - 1, n), (250, 333), (n - 4, n), (10, 10)]:
            rows = np.arange(s_begin, s_end)
            want_i, want_d = _lex_oracle(D[rows], rows, k)
            got_i, got_d = G.knn_rows_host(G.Graph(A), k, s_begin, s_end, max_distance=lim)
            assert got_i.shape == (s_end - s_begin, k) and got_i.dtype == np.int32 and got_d.dtype == np.float32
            assert np.array_equal(got_i, want_i), (k, s_begin, s_end)
            assert np.array_equal(got_d, want_d.astype(np.float32)), (k, s_begin, s_end)


def test_host_row_search_rejects_bad_arguments():
    from pymde_b200.preprocess import graph as G
    g = G.Graph(_geometric(50, 3, 2))
    for k, a, b in [(0, 0, 5), (3, -1, 5), (3, 5, 4), (3, 0, 51)]:
        with pytest.raises(ValueError):
            G.knn_rows_host(g, k, a, b)


# ---- the union graph and the checks of embed_new_points ---------------------------------------------------------------
def _split(A, n_old):
    """(data, new_data) Graphs of a symmetric adjacency: the fitted block, and every edge touching a node >= n_old."""
    from pymde_b200.preprocess import Graph
    U = sp.triu(A, k=1).tocoo()
    old = (U.row < n_old) & (U.col < n_old)
    e = np.stack([U.row, U.col], 1)
    data = Graph.from_edges(e[old], U.data[old], n_items=n_old)
    new = Graph.from_edges(e[~old], U.data[~old], n_items=A.shape[0])
    return data, new


@pytest.mark.parametrize("weighted", [True, False])
def test_union_is_the_graph_the_pieces_came_from(weighted):
    from pymde_b200 import recipes
    n, n_old = 500, 430
    A = _geometric(n, 6, 3, weighted=weighted, isolated=3)
    data, new = _split(A, n_old)
    recipes._check_new_graph(data, new)
    U = recipes._union_graph(data, new)
    assert U.shape == (n, n) and U.has_canonical_format
    # numpy restatement: the fitted block in the top-left corner, the new edges everywhere else, no overlap
    dense = np.zeros((n, n), dtype=np.float32)
    dense[:n_old, :n_old] = data.adjacency_matrix.toarray()
    extra = new.adjacency_matrix.toarray()
    assert not (extra[:n_old, :n_old] != 0).any()
    dense += extra
    assert np.array_equal(U.toarray(), dense)
    assert np.array_equal(U.toarray(), A.toarray())
    # the default radius: preserve_neighbors' rule on the union equals the rule on the two edge lists
    from pymde_b200.preprocess import Graph
    whole = float(3 * torch.quantile(Graph(U).distances, 0.75))
    parts = float(3 * torch.quantile(torch.cat([data.distances, new.distances]), 0.75))
    assert whole == parts
    # isolated new nodes and an empty new graph
    bare = Graph.from_edges(np.zeros((0, 2), dtype=np.int64), n_items=n_old + 5)
    U2 = recipes._union_graph(data, bare)
    assert U2.shape == (n_old + 5, n_old + 5) and U2.nnz == data.adjacency_matrix.nnz


def test_graph_input_is_checked_before_the_device():
    import pymde_b200 as pm
    from pymde_b200 import recipes
    n, n_old = 300, 250
    data, new = _split(_geometric(n, 5, 4), n_old)
    emb = torch.zeros((n_old, 2))
    X = np.zeros((n_old, 4), dtype=np.float32)
    # a Graph mixed with a matrix, either way round
    with pytest.raises(ValueError, match="both"):
        pm.embed_new_points(data, emb, X[:10])
    with pytest.raises(ValueError, match="both"):
        pm.embed_new_points(X, emb, new)
    with pytest.raises(ValueError, match="both"):
        pm.embed_new_points(sp.csr_matrix(X), emb, new)
    # fewer nodes in new_data than in data
    small = pm.Graph.from_edges(np.array([[0, 1]]), n_items=n_old - 1)
    with pytest.raises(ValueError, match="nodes"):
        pm.embed_new_points(data, emb, small)
    # an edge between two fitted nodes
    U = sp.triu(new.adjacency_matrix, k=1).tocoo()
    bad = pm.Graph.from_edges(np.concatenate([np.stack([U.row, U.col], 1), [[0, 1]]]),
                              np.concatenate([U.data, [1.0]]), n_items=n)
    with pytest.raises(ValueError, match="only the edges that touch a new node"):
        pm.embed_new_points(data, emb, bad)
    # the embedding
    with pytest.raises(ValueError, match="rows"):
        pm.embed_new_points(data, emb[:-1], new)
    with pytest.raises(ValueError, match="2-D"):
        pm.embed_new_points(data, emb[:, 0], new)
    with pytest.raises(ValueError, match="2-D"):
        pm.embed_new_points(data, emb[None], new)
    with pytest.raises(ValueError, match="2-D"):
        recipes._new_points_mde(data, emb.tolist(), new)
