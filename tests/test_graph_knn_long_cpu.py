"""CPU: the graph k-nearest-neighbour searches for 64 < k <= 256 (`mde_graph_knn_long`, `mde_graph_knn_long_rows`,
include/mde_b200.h) are exported, additive (the ABI version is still 1, the k <= 64 entries keep their bound), refuse
bad arguments before any launch, and the Python wrappers refuse k outside [1, 256] before they touch a device."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null: never dereferenced, every call below returns before a CUDA call


def _full(n=1000, k=100, indptr=FAKE, indices=FAKE, weights=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE, ws_bytes=None,
          max_distance=0.0):
    lib = _lib.load()
    if ws_bytes is None:
        ws_bytes = int(lib.mde_graph_knn_ws_bytes(n, 32)) if 1 <= n < (1 << 31) else 1 << 40
    return lib.mde_graph_knn_long(indptr, indices, weights, n, k, max_distance, out_i, out_d, ws, ws_bytes, None)


def _rows(n=1000, s_begin=0, s_end=10, k=100, indptr=FAKE, indices=FAKE, weights=FAKE, out_i=FAKE, out_d=FAKE,
          ws=FAKE, ws_bytes=None, max_distance=0.0):
    lib = _lib.load()
    if ws_bytes is None:
        ws_bytes = int(lib.mde_graph_knn_ws_bytes(n, 32)) if 1 <= n < (1 << 31) else 1 << 40
    return lib.mde_graph_knn_long_rows(indptr, indices, weights, n, s_begin, s_end, k, max_distance, out_i, out_d,
                                       ws, ws_bytes, None)


def test_symbols_are_exported_and_the_bounds_are_kept():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    assert int(lib.mde_graph_knn_long_max_k()) == 256
    assert int(lib.mde_graph_knn_max_k()) == 64
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in ("mde_graph_knn_long_max_k", "mde_graph_knn_long", "mde_graph_knn_long_rows"):
        assert name in _lib.SIGNATURES and getattr(lib, name) is not None, name
        assert "int %s(" % name in header, name
    assert "mde_graph_knn_long_ws_bytes" not in header  # the k <= 64 searches' size function serves both


def test_bad_arguments_are_rejected_without_a_launch():
    lib = _lib.load()
    INVALID = _lib.MDE_E_INVALID
    launches = int(lib.mde_launch_count())
    for call in (_full, _rows):
        for kw in ("indptr", "indices", "out_i", "out_d", "ws"):
            assert call(**{kw: None}) == INVALID, (call.__name__, kw)
        for k in (0, -1, 257, 1000):
            assert call(k=k) == INVALID, (call.__name__, k)
        for n in (0, -1, 1 << 31):
            assert call(n=n, **({"s_end": 0} if call is _rows else {})) == INVALID, (call.__name__, n)
        need = int(lib.mde_graph_knn_ws_bytes(1000, 32))
        assert call(ws_bytes=need - 1) == INVALID, call.__name__
        assert call(ws_bytes=0) == INVALID, call.__name__
    for s_begin, s_end in [(-1, 5), (0, 1001), (999, 1001), (6, 5), (1000, 999)]:
        assert _rows(s_begin=s_begin, s_end=s_end) == INVALID, (s_begin, s_end)
    # an empty range is checked like any other
    assert _rows(s_begin=7, s_end=7, k=257) == INVALID
    assert _rows(s_begin=7, s_end=7, ws_bytes=int(lib.mde_graph_knn_ws_bytes(1000, 32)) - 1) == INVALID
    assert _rows(s_begin=7, s_end=7, out_i=None) == INVALID
    # the k <= 64 entries still refuse k = 65
    assert lib.mde_graph_knn(FAKE, FAKE, FAKE, 1000, 65, 0.0, FAKE, FAKE, FAKE,
                             int(lib.mde_graph_knn_ws_bytes(1000, 32)), None) == INVALID
    assert lib.mde_graph_knn_rows(FAKE, FAKE, FAKE, 1000, 0, 10, 65, 0.0, FAKE, FAKE, FAKE,
                                  int(lib.mde_graph_knn_ws_bytes(1000, 32)), None) == INVALID
    assert int(lib.mde_launch_count()) == launches


def test_an_empty_range_returns_without_a_launch():
    lib = _lib.load()
    launches = int(lib.mde_launch_count())
    for n, s in [(1000, 0), (1000, 500), (1000, 1000), (1, 0), (1, 1)]:
        for k in (1, 65, 256):
            assert _rows(n=n, s_begin=s, s_end=s, k=k) == 0, (n, s, k)
    assert _rows(s_begin=3, s_end=3, weights=None, max_distance=2.5) == 0
    assert int(lib.mde_launch_count()) == launches


def _graph():
    from pymde_b200.preprocess import Graph
    rng = np.random.default_rng(0)
    n = 200
    e = np.stack([np.arange(n - 1), np.arange(1, n)], 1)
    U = sp.coo_matrix((rng.uniform(0.5, 1.5, n - 1).astype(np.float32), (e[:, 0], e[:, 1])), shape=(n, n)).tocsr()
    return Graph((U + U.T).tocsr())


@pytest.mark.parametrize("k", [0, 257])
def test_wrappers_refuse_k_before_the_device(k, monkeypatch):
    from pymde_b200 import util
    from pymde_b200.preprocess import graph as G

    def refuse(*a, **kw):
        raise AssertionError("the device was touched")

    monkeypatch.setattr(util, "cuda_device", refuse)
    monkeypatch.setattr(G, "_device_csr", refuse)
    g = _graph()
    with pytest.raises(ValueError, match="between 1 and 256"):
        G.k_nearest_neighbors_device_long(g, k)
    with pytest.raises(ValueError, match="between 1 and 256"):
        G.knn_rows_device_long(g, k, 0, 10)
    # the k <= 64 wrappers keep their bound
    with pytest.raises(ValueError, match="between 1 and 64"):
        G.k_nearest_neighbors_device(g, 65)
    with pytest.raises(ValueError, match="between 1 and 64"):
        G.knn_rows_device(g, 65, 0, 10)
    with pytest.raises(ValueError):
        G.knn_rows_device_long(g, 100, 5, 4)


def test_recipes_route_by_k():
    """The long device search serves 64 < k <= 256 on a graph the device searches take, and nothing else."""
    from pymde_b200 import recipes
    from pymde_b200.preprocess import generic
    A = _graph().adjacency_matrix
    big = sp.random(1000, 1000, density=0.01, format="csr", random_state=0)
    on_device = generic._graph_on_device(big)
    for k, want in [(1, False), (64, False), (65, True), (100, True), (256, True), (257, False)]:
        assert recipes._graph_knn_long(big, k) == (want and on_device), k
        assert not recipes._graph_knn_long(A, k), k  # 200 nodes: tiny graphs stay on the host
