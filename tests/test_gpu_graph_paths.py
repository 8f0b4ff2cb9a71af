"""Weighted shortest paths (`mde_graph_sssp`) and graph k-nearest neighbours (`mde_graph_knn`) on the device.
Arbiter: scipy.sparse.csgraph's Dijkstra in fp64 (what the host path calls), with the (length, node index) k-NN rule
and the splitmix64 retention rule restated here in numpy.  Lengths must agree bit for bit after the cast to fp32."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

pytestmark = pytest.mark.gpu

MASK = (1 << 64) - 1


def _geometric(n, k, seed, isolated=0, components=1):
    """Undirected geometric k-NN graph with Euclidean fp32 weights; `components` well separated clusters, and the
    last `isolated` nodes without edges."""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 2))
    pts[:, 0] += 10.0 * (np.arange(n) % components)
    _, idx = cKDTree(pts).query(pts, k=k + 1)
    e = np.stack([np.repeat(np.arange(n), k), idx[:, 1:].ravel()], 1)
    e = np.unique(np.sort(e, axis=1), axis=0)
    if isolated:
        e = e[(e < n - isolated).all(1)]
    w = np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1).astype(np.float32)
    U = sp.coo_matrix((w, (e[:, 0], e[:, 1])), shape=(n, n)).tocsr()
    return (U + U.T).tocsr()


def _unweighted(n, k, seed):
    A = _geometric(n, k, seed)
    A.data[:] = 1.0
    return A


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK
    return x ^ (x >> 31)


def _retained(seed, n, s, v, retain):
    thresh = int(retain * 2.0 ** 64)
    return np.array([_splitmix64(seed ^ ((int(a) * n + int(b)) & MASK)) < thresh for a, b in zip(s, v)], bool)


def _oracle_pairs(A, limit=np.inf):
    """Finite upper triangle of scipy's undirected Dijkstra: edges sorted by (i, j) and fp32 lengths."""
    D = csgraph.dijkstra(A, directed=False, limit=limit)
    n = A.shape[0]
    iu = np.triu_indices(n, 1)
    finite = np.isfinite(D[iu])
    return np.stack([iu[0][finite], iu[1][finite]], 1), D[iu][finite].astype(np.float32)


def _oracle_knn(A, k, limit):
    """k smallest (fp64 length, node index) pairs per row, self excluded, padded with -1 / inf."""
    D = csgraph.dijkstra(A, directed=False, limit=np.inf if limit is None else limit)
    np.fill_diagonal(D, np.inf)
    order = np.argsort(D, axis=1, kind="stable")[:, :k]  # stable: equal lengths in node order
    d = np.take_along_axis(D, order, 1)
    idx = np.where(np.isfinite(d), order, -1).astype(np.int32)
    return idx, d.astype(np.float32)


def _lib():
    from pymde_b200 import _lib
    return _lib, _lib.load()


def _stream():
    from pymde_b200 import util
    return util.stream_ptr(torch.device("cuda", 0))


def _sssp_raw(A, batch=None, weighted=True, max_length=0.0, retain=1.0, seed=0):
    """mde_graph_sssp through the binding; `batch` forces a workspace of exactly that batch.  Sorted triples."""
    from pymde_b200.preprocess import graph as G
    _l, lib = _lib()
    dev = torch.device("cuda", 0)
    n = A.shape[0]
    indptr, indices, w = G._device_csr(A, dev)
    if not weighted:
        w = torch.ones_like(w)
    nb = lib.mde_graph_sssp_ws_bytes(n, batch) if batch else lib.mde_graph_sssp_ws_bytes(n, (n + 31) // 32 * 32)
    ws = torch.empty(int(nb), dtype=torch.uint8, device=dev)
    cap = n * (n - 1) // 2 + 1
    src, dst = (torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(2))
    ln = torch.empty(cap, dtype=torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    _l.check(lib.mde_graph_sssp(indptr.data_ptr(), indices.data_ptr(), w.data_ptr(), n, 0, n, float(max_length),
                                float(retain), C.c_uint64(seed), src.data_ptr(), dst.data_ptr(), ln.data_ptr(), cap,
                                count.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
    got = int(count.item())
    s, v, l = src[:got].long().cpu().numpy(), dst[:got].long().cpu().numpy(), ln[:got].cpu().numpy()
    o = np.lexsort((v, s))
    return np.stack([s[o], v[o]], 1), l[o]


def _knn_raw(A, k, max_distance=None, batch=None):
    from pymde_b200.preprocess import graph as G
    _l, lib = _lib()
    dev = torch.device("cuda", 0)
    n = A.shape[0]
    indptr, indices, w = G._device_csr(A, dev)
    wptr = None if bool((A.data == 1.0).all()) else w.data_ptr()
    nb = lib.mde_graph_knn_ws_bytes(n, batch or (n + 31) // 32 * 32)
    ws = torch.empty(int(nb), dtype=torch.uint8, device=dev)
    idx = torch.empty(n * k, dtype=torch.int32, device=dev)
    ln = torch.empty(n * k, dtype=torch.float32, device=dev)
    _l.check(lib.mde_graph_knn(indptr.data_ptr(), indices.data_ptr(), wptr, n, k,
                               0.0 if max_distance is None else float(max_distance), idx.data_ptr(), ln.data_ptr(),
                               ws.data_ptr(), ws.numel(), _stream()))
    return idx.view(n, k).cpu().numpy(), ln.view(n, k).cpu().numpy()


# 1. all pairs, weighted ---------------------------------------------------------------------------------------------
def test_all_pairs_weighted_match_dijkstra_exactly():
    from pymde_b200.preprocess import graph as G
    n = 3000  # not a multiple of any batch (multiples of 32)
    A = _geometric(n, 8, 0, isolated=7, components=2)
    want_e, want_l = _oracle_pairs(A)
    out = G.shortest_paths_device(G.Graph(A), retain_fraction=1.0, device="cuda")
    assert out.edges.device.type == "cuda"
    got_e = out.edges.cpu().numpy()
    assert got_e.shape == want_e.shape and np.array_equal(got_e, want_e)
    assert np.array_equal(out.distances.cpu().numpy(), want_l)
    # many small batches: every batch must leave the distance tile clean for the next one
    e32, l32 = _sssp_raw(A, batch=32)
    assert np.array_equal(e32, want_e) and np.array_equal(l32, want_l)


# 2. limit and sampling ----------------------------------------------------------------------------------------------
def test_limit_and_sampling():
    from pymde_b200.preprocess import graph as G
    n = 3000
    A = _geometric(n, 8, 1)
    g = G.Graph(A)
    limit = 0.12
    want_e, want_l = _oracle_pairs(A, limit=limit)
    full = G.shortest_paths_device(g, max_length=limit, device="cuda", seed=11)
    assert full.n_edges == len(want_e)
    assert np.array_equal(full.edges.cpu().numpy(), want_e) and np.array_equal(full.distances.cpu().numpy(), want_l)
    part = G.shortest_paths_device(g, max_length=limit, retain_fraction=0.25, device="cuda", seed=11)
    again = G.shortest_paths_device(g, max_length=limit, retain_fraction=0.25, device="cuda", seed=11)
    assert torch.equal(part.edges, again.edges) and torch.equal(part.distances, again.distances)
    assert abs(part.n_edges / full.n_edges - 0.25) < 0.01
    key_full = full.edges[:, 0] * n + full.edges[:, 1]
    key_part = part.edges[:, 0] * n + part.edges[:, 1]
    pos = torch.searchsorted(key_full, key_part)
    assert torch.equal(key_full[pos], key_part) and torch.equal(full.distances[pos], part.distances)
    # the sample is exactly the splitmix64 rule
    keep = _retained(11, n, want_e[:, 0], want_e[:, 1], 0.25)
    assert np.array_equal(part.edges.cpu().numpy(), want_e[keep])


# 3. the two engines agree -------------------------------------------------------------------------------------------
def test_unit_weight_engine_matches_hop_engine():
    _l, lib = _lib()
    n = 2500
    A = _unweighted(n, 5, 2)
    dev = torch.device("cuda", 0)
    for max_length, retain, seed in ((0, 1.0, 0), (6, 0.3, 5)):
        e_w, l_w = _sssp_raw(A, weighted=True, max_length=max_length, retain=retain, seed=seed)
        indptr = torch.tensor(A.indptr.astype(np.int32), device=dev)
        indices = torch.tensor(A.indices.astype(np.int32), device=dev)
        ws = torch.empty(int(lib.mde_graph_hops_ws_bytes(n)), dtype=torch.uint8, device=dev)
        cap = n * (n - 1) // 2 + 1
        src, dst = (torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(2))
        ln = torch.empty(cap, dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        _l.check(lib.mde_graph_hops(indptr.data_ptr(), indices.data_ptr(), n, 0, n, max_length, retain,
                                    C.c_uint64(seed), src.data_ptr(), dst.data_ptr(), ln.data_ptr(), cap,
                                    count.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
        got = int(count.item())
        s, v, l = src[:got].long().cpu().numpy(), dst[:got].long().cpu().numpy(), ln[:got].cpu().numpy()
        o = np.lexsort((v, s))
        assert len(e_w) > 0
        assert np.array_equal(np.stack([s[o], v[o]], 1), e_w) and np.array_equal(l[o], l_w)


# 4. asymmetric and parallel entries, negative weights ---------------------------------------------------------------
def test_asymmetric_and_parallel_entries_match_undirected_dijkstra():
    from pymde_b200.preprocess import graph as G
    n = 1500
    S = _geometric(n, 6, 3)
    U = sp.triu(S, k=1, format="csr")          # every edge stored once, in one direction only
    want_e, want_l = _oracle_pairs(U)
    out = G.shortest_paths_device(G.Graph(U), device="cuda")
    assert np.array_equal(out.edges.cpu().numpy(), want_e) and np.array_equal(out.distances.cpu().numpy(), want_l)
    # parallel entries of different weights: raw CSR duplicates, the shorter one must win in both directions.
    # (float64 data holding fp32 values: scipy's Dijkstra sums duplicates when it has to convert the dtype)
    coo = S.tocoo()
    rng = np.random.default_rng(4)
    pick = rng.random(coo.nnz) < 0.3
    rows = np.concatenate([coo.row, coo.row[pick]])
    cols = np.concatenate([coo.col, coo.col[pick]])
    data = np.concatenate([coo.data, (coo.data[pick] * rng.uniform(0.3, 2.0, pick.sum())).astype(np.float32)])
    data = data.astype(np.float64)
    order = np.argsort(rows, kind="stable")
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))])
    P = sp.csr_matrix((data[order], cols[order], indptr), shape=(n, n))
    assert not P.has_canonical_format
    want_e, want_l = _oracle_pairs(P)
    out = G.shortest_paths_device(G.Graph(P), device="cuda")
    assert np.array_equal(out.edges.cpu().numpy(), want_e) and np.array_equal(out.distances.cpu().numpy(), want_l)
    # negative weights are rejected before any launch
    N = S.copy()
    N.data[5] = -N.data[5]
    _l, lib = _lib()
    launches = int(lib.mde_launch_count())
    with pytest.raises(ValueError):
        G.shortest_paths_device(G.Graph(N), device="cuda")
    with pytest.raises(ValueError):
        G.k_nearest_neighbors_device(G.Graph(N), 5, device="cuda")
    assert int(lib.mde_launch_count()) == launches


# 5. graph k-NN ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("finite", [False, True])
def test_graph_knn_matches_oracle(weighted, finite):
    n = 3000
    A = _geometric(n, 8, 5, isolated=3, components=2) if weighted else _unweighted(n, 4, 6)
    limit = None
    if finite:
        limit = float(3 * np.quantile(sp.triu(A).data, 0.75)) if weighted else 3.0
    for k in (1, 5, 15, 64):
        want_i, want_l = _oracle_knn(A, k, limit)
        got_i, got_l = _knn_raw(A, k, limit)
        assert np.array_equal(got_i, want_i), (k, np.argwhere(got_i != want_i)[:5])
        assert np.array_equal(got_l, want_l), k
    # several batches give the same answer
    got_i, got_l = _knn_raw(A, 15, limit, batch=64)
    want_i, want_l = _oracle_knn(A, 15, limit)
    assert np.array_equal(got_i, want_i) and np.array_equal(got_l, want_l)


def test_graph_knn_device_equals_host():
    from pymde_b200.preprocess import graph as G
    n = 2000
    g = G.Graph(_geometric(n, 8, 7))
    maxd = 3 * float(torch.quantile(g.distances, 0.75))
    for k, md in ((15, maxd), (10, None)):
        dev = G.k_nearest_neighbors_device(g, k, max_distance=md, device="cuda")
        host = G.k_nearest_neighbors(g, k, max_distance=md)
        assert dev.edges.device.type == "cuda"
        assert torch.equal(dev.edges.cpu(), host.edges)
        assert torch.equal(dev.weights.cpu(), host.weights)
        assert set(np.unique(dev.weights.cpu().numpy())) <= {1.0, 2.0}


def test_generic_knn_above_max_k_uses_host():
    from pymde_b200.preprocess import generic
    from pymde_b200.preprocess import graph as G
    _l, lib = _lib()
    n = 400
    g = G.Graph(_geometric(n, 8, 8))
    k = int(lib.mde_graph_knn_max_k()) + 6
    got = generic.k_nearest_neighbors(g, k, device="cuda")
    want = G.k_nearest_neighbors(g, k)
    assert isinstance(got, G.Graph)
    assert torch.equal(got.edges, want.edges) and torch.equal(got.weights, want.weights)
    dev = generic.k_nearest_neighbors(g, 15, device="cuda")
    assert isinstance(dev, G.EdgeListGraph) and dev.edges.device.type == "cuda"


# 6. recipes stay on the device --------------------------------------------------------------------------------------
def test_recipes_on_a_weighted_graph_stay_on_device():
    import pymde_b200 as pm
    n = 3000
    g = pm.preprocess.Graph(_geometric(n, 8, 9))

    def build(recipe, **kw):
        pm.seed(0)
        return recipe(g, embedding_dim=2, device="cuda", **kw)

    for recipe, kw, attr in ((pm.preserve_distances, {"max_distances": 5e5}, "deviations"),
                             (pm.preserve_neighbors, {}, "weights")):
        mde = build(recipe, **kw)
        again = build(recipe, **kw)
        assert mde.edges.device.type == "cuda"
        assert torch.equal(mde.edges, again.edges)
        assert torch.equal(getattr(mde.distortion_function, attr), getattr(again.distortion_function, attr))
        mde.embed(max_iter=30)
        st = mde.solve_stats
        assert st.average_distortions[-1] < st.average_distortions[0]


# 7. bad arguments ---------------------------------------------------------------------------------------------------
def test_bad_arguments_are_rejected_without_a_launch():
    _l, lib = _lib()
    INVALID = _l.MDE_E_INVALID
    dev = torch.device("cuda", 0)
    n = 100
    A = _geometric(n, 4, 10)
    from pymde_b200.preprocess import graph as G
    indptr, indices, w = G._device_csr(A, dev)
    ip, ix, wp = indptr.data_ptr(), indices.data_ptr(), w.data_ptr()
    good = int(lib.mde_graph_sssp_ws_bytes(n, 32))
    ws = torch.empty(good, dtype=torch.uint8, device=dev)
    out = torch.empty(4 * n * n, dtype=torch.int32, device=dev)
    ln = torch.empty(n * n, dtype=torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    st = _stream()
    assert lib.mde_graph_sssp_ws_bytes(n, 0) < 0 and lib.mde_graph_sssp_ws_bytes(n, 48) < 0
    launches = int(lib.mde_launch_count())

    def sssp(**kw):
        a = dict(indptr=ip, indices=ix, weights=wp, n=n, s0=0, s1=n, ml=0.0, retain=1.0, seed=C.c_uint64(0),
                 src=out.data_ptr(), dst=out.data_ptr() + 4 * n * n, ln=ln.data_ptr(), cap=n * n,
                 count=count.data_ptr(), ws=ws.data_ptr(), wsb=good, stream=st)
        a.update(kw)
        return lib.mde_graph_sssp(*a.values())

    assert sssp(indptr=None) == INVALID
    assert sssp(indices=None) == INVALID
    assert sssp(count=None) == INVALID
    assert sssp(ws=None) == INVALID
    assert sssp(src=None) == INVALID
    assert sssp(n=1 << 31) == INVALID
    assert sssp(n=0) == INVALID
    assert sssp(s0=-1) == INVALID
    assert sssp(s1=n + 1) == INVALID
    assert sssp(s0=10, s1=5) == INVALID
    assert sssp(wsb=good - 1) == INVALID

    def knn(**kw):
        a = dict(indptr=ip, indices=ix, weights=wp, n=n, k=5, md=0.0, idx=out.data_ptr(), ln=ln.data_ptr(),
                 ws=ws.data_ptr(), wsb=int(lib.mde_graph_knn_ws_bytes(n, 32)), stream=st)
        a.update(kw)
        return lib.mde_graph_knn(*a.values())

    assert knn(k=0) == INVALID
    assert knn(k=int(lib.mde_graph_knn_max_k()) + 1) == INVALID
    assert knn(indptr=None) == INVALID
    assert knn(idx=None) == INVALID
    assert knn(ln=None) == INVALID
    assert knn(ws=None) == INVALID
    assert knn(n=1 << 31) == INVALID
    assert knn(wsb=int(lib.mde_graph_knn_ws_bytes(n, 32)) - 1) == INVALID
    assert int(lib.mde_launch_count()) == launches
    # and the same arguments, corrected, run
    assert knn() == 0 and sssp() == 0
