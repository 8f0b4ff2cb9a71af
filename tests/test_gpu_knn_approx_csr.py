"""Row f3, sparse and approximate: NN-descent over CSR rows (`mde_knn_approx_csr`, csrc/mde_knn_approx.cu).

Contract: k distinct rows per row, never the row itself, ascending by (squared distance, index), with the distances
of `mde_knn_csr` / `mde_knn_csr_wide` (the fp64 sum rounded once); bit-identical results for the same (CSR, k, seed),
whatever the workspace held; recall against the exact sparse search; opt-in routing through
PYMDE_B200_KNN_SPARSE=approx, which PYMDE_B200_KNN=approx does not imply."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.test_gpu_knn_sparse import _clustered, _exact_d2, _random_csr, _ulps

pytestmark = pytest.mark.gpu


def _approx(A, k, seed=1, fill=None, iterations=False):
    from pymde_b200 import _lib
    from pymde_b200.preprocess import data_matrix as dm
    lib = _lib.load()
    (indptr, indices, values), (n, d) = dm._to_device_csr(A, "cuda")
    nnz = int(indices.shape[0])
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_approx_csr_ws_bytes(n, d, nnz, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    if fill is not None:
        ws.fill_(fill)
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    it = C.c_int(-1)
    _lib.check(lib.mde_knn_approx_csr_ex(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), n, d, nnz, k,
                                         C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(), p, need.value,
                                         torch.cuda.current_stream().cuda_stream, C.byref(it)))
    torch.cuda.synchronize()
    return (idx, d2, it.value) if iterations else (idx, d2)


def _exact(A, k):
    from pymde_b200.preprocess import data_matrix as dm
    csr, shape = dm._to_device_csr(A, "cuda")
    return dm.knn_sparse_device(csr, shape, k)


def _check_contract(A, k, idx, d2):
    """Validity, distinctness, (distance, index) order, and distances equal to the fp64 sum rounded once (up to the
    last place another summation order can move)."""
    n = A.shape[0]
    got = idx.long()
    assert int(got.min()) >= 0 and int(got.max()) < n
    assert not bool((got == torch.arange(n, device="cuda")[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())
    dd, ii = d2[:, 1:], idx[:, 1:]
    dp, ip = d2[:, :-1], idx[:, :-1]
    assert bool(((dd > dp) | ((dd == dp) & (ii > ip))).all())
    X = torch.tensor(A.toarray(), device="cuda", dtype=torch.float64)
    ex = _exact_d2(X, torch.arange(n, device="cuda"), got).float().cpu().numpy()
    u = _ulps(d2.cpu().numpy(), ex)
    assert u.max() <= 1 and (u == 0).mean() >= 0.9999


def _with_long_row(n, d, long_nnz, seed):
    A = _random_csr(n, d, 0.01, seed).tolil()
    rng = np.random.default_rng(seed + 1)
    A[n // 2, rng.choice(d, long_nnz, replace=False)] = rng.standard_normal(long_nnz).astype(np.float32)
    A = A.tocsr()
    A.sort_indices()
    return A


def _with_empty_rows():
    A = _random_csr(600, 400, 0.05, seed=1).tolil()
    A[np.arange(5, 600, 7)] = 0
    A = A.tocsr()
    A.eliminate_zeros()
    return A


def _with_duplicates():
    base = _random_csr(500, 2000, 0.03, seed=2)
    return sp.vstack([base, base[:100]]).tocsr()


AWKWARD = {
    "n2": (lambda: _random_csr(2, 5, 0.5, seed=3), 1),
    "d1": (lambda: _random_csr(300, 1, 0.7, seed=4), 5),
    "k64": (lambda: _random_csr(4099, 3000, 0.01, seed=5), 64),
    "empty_rows": (_with_empty_rows, 10),
    "duplicates": (_with_duplicates, 6),
    "all_zero": (lambda: sp.csr_matrix((200, 50), dtype=np.float32), 5),
    "long_row": (lambda: _with_long_row(3000, 30000, 20000, seed=6), 15),
}


@pytest.mark.parametrize("case", sorted(AWKWARD))
def test_output_contract_on_awkward_shapes(case):
    make, k = AWKWARD[case]
    A = make()
    idx, d2 = _approx(A, k)
    _check_contract(A, k, idx, d2)
    if case == "all_zero":
        assert bool((d2 == 0).all())
    if case == "duplicates":  # a copy is at distance 0: whatever else the search found, it found the copy
        assert bool((d2[:100, 0] == 0).all()) and bool((d2[500:, 0] == 0).all())


@pytest.mark.parametrize("n,d,density,k", [(2, 5, 0.5, 1), (20, 300, 0.1, 7), (33, 400, 0.05, 24), (30, 1, 0.5, 15),
                                           (60, 500, 0.05, 30), (97, 2000, 0.02, 64), (97, 50, 0.0, 40)])
def test_exact_when_the_lists_hold_every_row(n, d, density, k):
    """n - 1 <= 32 (k <= 24) or n - 1 <= 96 (k > 24): every list holds every other row, so the result is the exact
    sparse search's, bit for bit, ties included (both are fully determined)."""
    A = _random_csr(n, d, density, seed=3 * n + k)
    idx, d2 = _approx(A, k)
    ri, rd = _exact(A, k)
    assert torch.equal(idx, ri)
    assert torch.equal(d2.view(torch.int32), rd.view(torch.int32))


def _recall_checks(idx, d2, ri, rd, floor=0.97):
    k = idx.shape[1]
    a = torch.sort(idx.long(), 1)[0]
    b = torch.sort(ri.long(), 1)[0]
    hits = (a[:, :, None] == b[:, None, :]).any(2).float().sum(1)
    recall = float(hits.mean()) / k
    assert recall >= floor, recall
    # an approximate list never beats the true j-th distance
    assert bool((d2 >= rd).all())
    # rows whose set is the exact set carry the exact search's bits
    same = (a == b).all(1)
    assert bool(torch.equal(d2[same].view(torch.int32), rd[same].view(torch.int32)))
    return recall


def _low_dim_clusters(n, d, nnz_row, n_centres, intrinsic, seed):
    """The sparse counterpart of the dense tests' mixture: each row keeps its cluster centre's support, and its values
    move along `intrinsic` random directions of that cluster plus noise of 1e-2.  (`_clustered`'s isotropic noise in
    all nnz_row values is NN-descent's weak case: every row of a cluster is nearly equidistant from every other.)"""
    rng = np.random.default_rng(seed)
    cols = np.stack([rng.choice(d, nnz_row, replace=False) for _ in range(n_centres)])
    vals = rng.standard_normal((n_centres, nnz_row)) * 4
    basis = rng.standard_normal((n_centres, intrinsic, nnz_row)) / np.sqrt(nnz_row)
    lab = rng.integers(0, n_centres, n)
    z = rng.standard_normal((n, intrinsic))
    v = vals[lab] + np.einsum("ni,nif->nf", z, basis[lab]) + 1e-2 * rng.standard_normal((n, nnz_row))
    r = np.repeat(np.arange(n), nnz_row)
    return sp.csr_matrix((v.astype(np.float32).ravel(), (r, cols[lab].ravel())), shape=(n, d))


@pytest.fixture(scope="module")
def clustered():
    return _low_dim_clusters(50000, 20000, 30, 100, 6, seed=12)


@pytest.mark.parametrize("k", [15, 24, 50])
def test_recall_on_a_clustered_sparse_matrix(clustered, k):
    idx, d2 = _approx(clustered, k, seed=5)
    ri, rd = _exact(clustered, k)  # mde_knn_csr for k <= 24, mde_knn_csr_wide for k = 50
    recall = _recall_checks(idx, d2, ri, rd)
    print("k = %d: recall %.4f" % (k, recall))


def test_determinism_seed_and_workspace(clustered):
    k = 15
    i1, d1 = _approx(clustered, k, seed=9, fill=0x00)
    i2, d2 = _approx(clustered, k, seed=9, fill=0xFF)
    i3, d3 = _approx(clustered, k, seed=9)
    assert torch.equal(i1, i2) and torch.equal(i1, i3)
    assert torch.equal(d1.view(torch.int32), d2.view(torch.int32))
    assert torch.equal(d1.view(torch.int32), d3.view(torch.int32))
    # another seed: another run, the same quality
    i4, d4 = _approx(clustered, k, seed=12345)
    ri, rd = _exact(clustered, k)
    _recall_checks(i4, d4, ri, rd)


def test_iterations_are_reported():
    A = _clustered(5000, 3000, 20, 100, seed=13)
    _, _, it = _approx(A, 10, iterations=True)
    assert 1 <= it <= 13  # max(5, ceil(log2 5000))
    _, _, it = _approx(_random_csr(30, 100, 0.1, seed=1), 10, iterations=True)
    assert it == 0  # every list holds every row from the start


def test_k_nearest_neighbors_routes_to_the_approximate_sparse_search(monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import preprocess
    from pymde_b200.preprocess import data_matrix as dm
    A = _clustered(3000, 5000, 20, 100, seed=2)
    monkeypatch.setenv("PYMDE_B200_KNN_SPARSE", "approx")
    for k in (10, 30):
        pm.seed(7)
        g1 = preprocess.k_nearest_neighbors(A, k=k)
        pm.seed(7)
        csr, shape = dm._to_device_csr(A, "cuda")
        idx, d2 = dm.knn_approx_sparse_device(csr, shape, k)
        g2 = dm._knn_graph(idx, d2, 3000, None, torch.device("cuda"))
        assert np.array_equal(np.asarray(g1.edges.cpu()), np.asarray(g2.edges.cpu()))
        np.testing.assert_array_equal(np.asarray(g1.distances.cpu()), np.asarray(g2.distances.cpu()))


def _refuse(*a, **kw):
    raise AssertionError("approximate sparse search taken without PYMDE_B200_KNN_SPARSE=approx")


@pytest.mark.parametrize("knn_mode", [None, "approx"])
def test_without_the_sparse_variable_the_search_stays_exact(monkeypatch, knn_mode):
    """Unset, and with PYMDE_B200_KNN=approx alone (documented to keep sparse input exact)."""
    from pymde_b200 import preprocess
    from pymde_b200.preprocess import data_matrix as dm
    monkeypatch.delenv("PYMDE_B200_KNN_SPARSE", raising=False)
    if knn_mode is None:
        monkeypatch.delenv("PYMDE_B200_KNN", raising=False)
    else:
        monkeypatch.setenv("PYMDE_B200_KNN", knn_mode)
    monkeypatch.setattr(dm, "knn_approx_sparse_device", _refuse)
    monkeypatch.setattr(dm, "knn_approx_device", _refuse)
    A = _clustered(1500, 4000, 20, 100, seed=4)
    g = preprocess.k_nearest_neighbors(A, k=7)
    idx, d2 = _exact(A, 7)
    ref = dm._knn_graph(idx, d2, 1500, None, torch.device("cuda"))
    assert np.array_equal(np.asarray(g.edges.cpu()), np.asarray(ref.edges.cpu()))


def test_preserve_neighbors_is_reproducible_and_embeds(monkeypatch):
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_KNN_SPARSE", "approx")
    A = _clustered(4000, 6000, 20, 150, seed=8)
    runs = []
    for _ in range(2):
        pm.seed(3)
        mde = pm.preserve_neighbors(A, embedding_dim=2, verbose=False, device="cuda")
        runs.append((mde.edges.cpu().numpy(), mde.distortion_function.weights.cpu().numpy()))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert np.array_equal(runs[0][1], runs[1][1])
    Y = mde.embed(max_iter=20)
    assert Y.shape == (4000, 2) and bool(torch.isfinite(Y).all())


def test_no_densifying_at_400_gb_dense_size(monkeypatch):
    from pymde_b200 import preprocess
    monkeypatch.setenv("PYMDE_B200_KNN_SPARSE", "approx")
    A = _clustered(100_000, 1_000_000, 10, 2000, seed=9)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    g = preprocess.k_nearest_neighbors(A, k=10)
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 2 * 2 ** 30, peak
    assert g.n_items == 100_000 and g.edges.shape[0] >= 100_000 * 10 // 2
