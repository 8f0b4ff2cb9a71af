"""GPU: the neighbour-graph builder (`mde_knn_graph_count` / `mde_knn_graph_emit`) gives exactly the edges and weights of
`Graph.from_edges`, and the recipes that assemble their graphs on the device build the same problems, bit for bit, as
with the host `Graph`."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu


def _host(idx):
    """Graph.from_edges of the directed pairs (i, idx[i, s]), the arbiter."""
    from pymde_b200.preprocess.graph import Graph
    idx = np.asarray(idx)
    n, k = idx.shape
    i = np.repeat(np.arange(n), k)
    j = idx.ravel().astype(np.int64)
    keep = j >= 0
    g = Graph.from_edges(np.stack([i[keep], j[keep]], 1).reshape(-1, 2), None, n_items=n)
    return g.edges, g.weights


def _device(idx):
    from pymde_b200.preprocess.graph import knn_edge_list
    g = knn_edge_list(torch.as_tensor(np.asarray(idx), dtype=torch.int32, device="cuda"), len(idx))
    return g.edges.cpu(), g.weights.cpu()


def _assert_same(idx):
    e_ref, w_ref = _host(idx)
    e, w = _device(idx)
    assert e.dtype == torch.int64 and w.dtype == torch.float32
    assert torch.equal(e, e_ref)
    assert torch.equal(w, w_ref)
    return e, w


def _random_lists(n, k, seed, holes=0.0):
    rng = np.random.default_rng(seed)
    idx = (np.arange(n)[:, None] + rng.integers(1, n, (n, k))) % n  # never the row itself; repeats allowed
    if holes:
        idx[rng.random((n, k)) < holes] = -1
    return idx.astype(np.int32)


@pytest.mark.parametrize("k", [1, 15, 24, 25, 64])
def test_random_lists_match_from_edges(k):
    _assert_same(_random_lists(5000, k, k))


@pytest.mark.parametrize("k", [1, 15, 24, 25, 64])
def test_lists_with_holes_and_empty_rows(k):
    idx = _random_lists(3000, k, 100 + k, holes=0.3)
    idx[::7] = -1  # rows with no entry at all
    idx[5, :] = -1
    _assert_same(idx)


@pytest.mark.parametrize("k", [1, 15, 24, 25, 64])
def test_fully_reciprocal_lists(k):
    rng = np.random.default_rng(k)
    for n in sorted({2, max(2, k // 2), k + 1}):
        idx = np.full((n, k), -1, dtype=np.int32)
        for i in range(n):
            others = rng.permutation([j for j in range(n) if j != i])[:k]
            slots = rng.permutation(k)[:len(others)]  # -1 anywhere in the row
            idx[i, slots] = others
        e, w = _assert_same(idx)
        assert e.shape[0] == n * (n - 1) // 2 and bool((w == 2).all())


def test_duplicates_inside_a_row_are_counted():
    n, k = 2000, 24
    idx = _random_lists(n, k, 4)
    idx[:, 1::2] = idx[:, 0::2]  # every entry twice
    idx[:, 20:] = idx[:, :1]     # one entry six times
    e, w = _assert_same(idx)
    assert float(w.max()) >= 6
    small = np.array([[1, 1, 2, 1], [0, 0, -1, 2], [1, -1, -1, -1]], dtype=np.int32)
    e, w = _assert_same(small)
    assert e.tolist() == [[0, 1], [0, 2], [1, 2]] and w.tolist() == [5.0, 1.0, 2.0]


def test_a_hub_listed_by_every_row():
    n, k, hub = 200_000, 15, 12345
    idx = _random_lists(n, k, 5)
    idx[:, 3] = hub
    idx[hub] = _random_lists(n, k, 6)[hub]
    e, w = _assert_same(idx)
    assert int(((e[:, 0] == hub) | (e[:, 1] == hub)).sum()) >= n - 1


def test_no_entries_at_all():
    for n, k in ((1, 1), (1, 64), (1000, 15)):
        e, w = _assert_same(np.full((n, k), -1, dtype=np.int32))
        assert e.shape == (0, 2) and w.shape == (0,)


@pytest.mark.parametrize("bad", ["self", "n", "below"])
def test_bad_entries_raise(bad):
    idx = _random_lists(1000, 15, 7)
    idx[417, 9] = {"self": 417, "n": 1000, "below": -2}[bad]
    with pytest.raises(ValueError):
        _device(idx)


def _raw(idx, fill):
    """The two C calls on a workspace pre-filled with `fill`."""
    from pymde_b200 import _lib
    lib = _lib.load()
    n, k = idx.shape
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_graph_ws_bytes(n, k, C.byref(need)))
    ws = torch.full((need.value + 1024,), fill, dtype=torch.uint8, device="cuda")
    off = (-ws.data_ptr()) % 1024
    p = C.c_int64(0)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mde_knn_graph_count(idx.data_ptr(), n, k, ws.data_ptr() + off, need.value, C.byref(p), s))
    e = torch.full((p.value, 2), -5, dtype=torch.int64, device="cuda")
    w = torch.full((p.value,), -5.0, dtype=torch.float32, device="cuda")
    _lib.check(lib.mde_knn_graph_emit(n, k, ws.data_ptr() + off, need.value, e.data_ptr(), w.data_ptr(), s))
    torch.cuda.synchronize()
    return e.cpu(), w.cpu()


@pytest.mark.parametrize("k", [15, 64])
def test_deterministic_whatever_the_workspace_held(k):
    raw = _random_lists(20000, k, 8, holes=0.1)
    raw[:, 0] = 77
    raw[77, 0] = 78
    idx = torch.as_tensor(raw, device="cuda")
    e_ref, w_ref = _host(raw)
    runs = [_raw(idx, 0x00), _raw(idx, 0xFF), _raw(idx, 0x00), _device(raw)]
    for e, w in runs:
        assert torch.equal(e, e_ref) and torch.equal(w, w_ref)


def _blobs(n, d, seed, dup=0):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((6, d)) * 5
    X = centers[rng.integers(0, 6, n)] + rng.standard_normal((n, d))
    if dup:
        X[-dup:] = X[:dup]  # duplicate rows: zero distances
    return X.astype(np.float32)


def _sparse(X):
    X = X.copy()
    X[np.abs(X) < 1.0] = 0
    return sp.csr_matrix(X)


@pytest.mark.parametrize("search", ["dense", "sparse", "approx", "approx_sparse", "gemm"])
@pytest.mark.parametrize("max_distance", [None, 4.0])
@pytest.mark.parametrize("k", [15, 50])
def test_search_outputs_match_the_host_graph(monkeypatch, search, max_distance, k):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    X = _blobs(3000, 12, 9)
    data = _sparse(X) if "sparse" in search else X
    if search.startswith("approx"):
        monkeypatch.setenv("PYMDE_B200_KNN_SPARSE" if "sparse" in search else "PYMDE_B200_KNN", "approx")
    if search == "gemm":
        monkeypatch.setenv("PYMDE_B200_KNN", "gemm")
    pm.seed(1)
    g_ref = dm.k_nearest_neighbors(data, k, max_distance=max_distance)
    pm.seed(1)
    g = dm.k_nearest_neighbors_device(data, k, max_distance=max_distance)
    assert g.edges.is_cuda and g.weights.is_cuda and g.n_items == 3000
    assert torch.equal(g.edges.cpu(), g_ref.edges)
    assert torch.equal(g.weights.cpu(), g_ref.weights)
    if max_distance is not None:
        assert g.n_edges < pm.preprocess.data_matrix.k_nearest_neighbors_device(data, k).n_edges


def test_device_knn_refuses_k_above_64():
    from pymde_b200.preprocess import data_matrix as dm
    with pytest.raises(ValueError):
        dm.k_nearest_neighbors_device(_blobs(200, 4, 1), 65)


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("retain", [0.3, 1.0])
def test_distance_graph_matches_the_host_graph(sparse, retain):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    X = _blobs(700, 10, 2, dup=40)
    X[5] = np.nan  # a NaN row: NaN distances are kept
    data = _sparse(X) if sparse else X
    pm.seed(4)
    g_ref = dm.distances(data, retain_fraction=retain)
    pm.seed(4)
    g = dm.distances_device(data, retain_fraction=retain)
    assert torch.equal(g.edges.cpu(), g_ref.edges)
    assert torch.equal(g.distances.cpu().view(torch.int32), g_ref.distances.view(torch.int32))  # NaN included
    assert bool(g.distances.isnan().any())
    assert g.n_edges < 700 * 699 // 2 * retain  # the duplicate rows' zeros are dropped


# --- recipes: device graph step against the host Graph ----------------------------------------------------------------

def _host_graph_steps(monkeypatch):
    from pymde_b200.preprocess import data_matrix as dm

    def knn(data, k, max_distance=None, device=None):
        return dm.k_nearest_neighbors(data, k, max_distance=max_distance, device=device)

    def dist(data, retain_fraction=1.0, device=None):
        return dm.distances(data, retain_fraction=retain_fraction, device=device)

    monkeypatch.setattr(dm, "k_nearest_neighbors_device", knn)
    monkeypatch.setattr(dm, "distances_device", dist)


def _problem(make, seed):
    import pymde_b200 as pm
    pm.seed(seed)
    mde = make()
    f = mde.distortion_function
    data = f.weights if hasattr(f, "weights") else f.deviations
    return mde.edges.clone(), data.clone(), getattr(mde, "_X_init", None)


def _recipes(data, n):
    import pymde_b200 as pm
    anchors = torch.arange(0, n, 97, device="cuda")
    values = torch.randn(anchors.shape[0], 2, generator=torch.Generator().manual_seed(0)).cuda()
    return {
        "neighbors_centered": lambda: pm.preserve_neighbors(data, constraint=pm.Centered()),
        "neighbors_standardized": lambda: pm.preserve_neighbors(data, constraint=pm.Standardized()),
        "neighbors_anchored": lambda: pm.preserve_neighbors(data, constraint=pm.Anchored(anchors, values)),
        "neighbors_max_distance": lambda: pm.preserve_neighbors(data, n_neighbors=24, max_distance=5.0),
        "laplacian": lambda: pm.laplacian_embedding(data),
        "distances_sampled": lambda: pm.preserve_distances(data, max_distances=2e5),
        "distances_all": lambda: pm.preserve_distances(data),
    }


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("recipe", ["neighbors_centered", "neighbors_standardized", "neighbors_anchored",
                                    "neighbors_max_distance", "laplacian", "distances_sampled", "distances_all"])
def test_recipes_are_bit_identical_to_the_host_graph(monkeypatch, sparse, recipe):
    n = 1500 if recipe.startswith("distances") else 4000
    X = _blobs(n, 16, 11, dup=30)
    data = _sparse(X) if sparse else X
    make = _recipes(data, n)[recipe]
    dev = _problem(make, 7)
    with monkeypatch.context() as m:
        _host_graph_steps(m)
        host = _problem(make, 7)
    again = _problem(make, 7)
    for a, b, c in zip(dev, host, again):
        if a is None:
            assert b is None and c is None
            continue
        assert torch.equal(a, c)  # run to run
        assert torch.equal(a, b)  # device graph step == host Graph
    if recipe.startswith("distances"):
        assert bool((dev[1] > 0).all())  # the duplicate rows' zero distances were dropped


@pytest.mark.parametrize("sparse", [False, True])
def test_recipes_build_no_scipy_graph(monkeypatch, sparse):
    import pymde_b200 as pm
    from pymde_b200.preprocess.graph import Graph

    def refuse(*args, **kwargs):
        raise AssertionError("a host Graph was built")

    n = 2500
    X = _blobs(n, 16, 12)
    data = _sparse(X) if sparse else X
    monkeypatch.setattr(Graph, "__init__", refuse)
    monkeypatch.setattr(Graph, "from_edges", staticmethod(refuse))
    pm.seed(0)
    for mde in (pm.preserve_neighbors(data), pm.laplacian_embedding(data), pm.preserve_distances(data)):
        assert mde.edges.is_cuda and mde.edges.shape[0] > n
