"""Row f3 for 24 < k <= 64: `mde_knn_wide` and `mde_knn_csr_wide` (csrc/mde_knn.cu, csrc/mde_knn_sparse.cu: a
running top-96 per query row in shared memory) against fp64 brute forces, against the k <= 24 searches where both
apply, and through `k_nearest_neighbors` and the recipes."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.test_gpu_knn import _brute64 as _brute64_dense
from tests.test_gpu_knn import _compare as _compare_dense
from tests.test_gpu_knn_sparse import _clustered, _random_csr, _ulps

pytestmark = pytest.mark.gpu


def _lib():
    from pymde_b200 import _lib as L
    return L, L.load()


def _ws(nbytes):
    ws = torch.empty(nbytes + 1024, dtype=torch.uint8, device="cuda")
    return ws, ws.data_ptr() + (-ws.data_ptr()) % 1024


def _dense(X, k, wide):
    """One call of mde_knn_wide (wide) or mde_knn, whatever k is."""
    L, lib = _lib()
    X = X.contiguous()
    n, d = X.shape
    need = C.c_size_t(0)
    L.check((lib.mde_knn_wide_ws_bytes if wide else lib.mde_knn_ws_bytes)(n, d, C.byref(need)))
    ws, p = _ws(need.value)
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    L.check((lib.mde_knn_wide if wide else lib.mde_knn)(X.data_ptr(), n, d, k, idx.data_ptr(), d2.data_ptr(), p,
                                                          need.value, None))
    torch.cuda.synchronize()
    return idx, d2


def _sparse(A, k, wide):
    """One call of mde_knn_csr_wide (wide) or mde_knn_csr."""
    from pymde_b200.preprocess import data_matrix as dm
    L, lib = _lib()
    (ip, ix, v), (n, d) = dm._to_device_csr(A, "cuda")
    nnz = int(ix.shape[0])
    need = C.c_size_t(0)
    L.check((lib.mde_knn_csr_wide_ws_bytes if wide else lib.mde_knn_csr_ws_bytes)(n, d, nnz, C.byref(need)))
    ws, p = _ws(need.value)
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    L.check((lib.mde_knn_csr_wide if wide else lib.mde_knn_csr)(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz,
                                                                  k, idx.data_ptr(), d2.data_ptr(), p, need.value,
                                                                  None))
    return idx, d2


def _brute_all_pairs(A, k):
    """fp64 brute force over all pairs: sum (q - x)^2 of the densified rows in fp64, rounded once to fp32, the k
    smallest by (distance, index) -- the fully determined result of the sparse searches, up to the order of the fp64
    sums."""
    X = torch.tensor(A.toarray(), dtype=torch.float64, device="cuda")
    n, d = X.shape
    D = torch.empty((n, n), dtype=torch.float32, device="cuda")
    step = max(1, (1 << 27) // (n * d))
    for s0 in range(0, n, step):
        D[s0:s0 + step] = ((X[s0:s0 + step, None, :] - X[None, :, :]) ** 2).sum(-1).float()
    D.fill_diagonal_(float("inf"))
    val, idx = torch.sort(D, dim=1, stable=True)  # stable: equal distances stay in index order
    return idx[:, :k].cpu().numpy(), val[:, :k].cpu().numpy()


def _dense_matrix(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn((n, d), generator=g, device="cuda")
    if d == 784:  # MNIST-like: clipped, many exact zeros
        X = torch.where(X < 0.3, torch.zeros_like(X), X.clamp(max=1.0)).contiguous()
    return X


@pytest.mark.parametrize("n,d,k", [(65, 7, 64), (130, 64, 40), (1000, 65, 64), (2500, 200, 25), (4099, 784, 50)])
def test_wide_dense_matches_fp64_brute_force(n, d, k):
    from pymde_b200.preprocess import data_matrix as dm
    X = _dense_matrix(n, d, n + d)
    idx, d2 = dm.knn_device(X, k)  # k > 24 selects mde_knn_wide
    _compare_dense(X, k, idx, d2)
    if k == n - 1:  # every other row is a neighbour
        assert bool((torch.sort(idx.long(), 1)[0].sum(1) == n * (n - 1) // 2 - torch.arange(n, device="cuda")).all())


def test_wide_dense_duplicates_and_far_offsets():
    g = torch.Generator(device="cuda").manual_seed(7)
    base = torch.randn((700, 48), generator=g, device="cuda")
    X = torch.cat([base, base[:100]], 0) + 30.0
    k = 40
    idx, d2 = _dense(X, k, wide=True)
    # _compare's checks, except that a duplicated pair often straddles the k-th place at k = 40: fewer rows have a
    # clear gap behind the k-th neighbour than _compare expects of generic data
    val, ref = _brute64_dense(X, k)
    got = idx.long()
    assert not bool((got == torch.arange(800, device="cuda")[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())
    gd = ((X.double()[:, None, :] - X.double()[got]) ** 2).sum(-1)
    np.testing.assert_allclose(gd.cpu().numpy(), val[:, :k].cpu().numpy(), rtol=2e-6, atol=1e-9)
    np.testing.assert_allclose(d2.double().cpu().numpy(), gd.cpu().numpy(), rtol=2e-6, atol=1e-9)
    assert bool((d2[:, 1:] >= d2[:, :-1]).all())
    clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-9
    assert bool((s == torch.sort(ref, 1)[0]).all(1)[clear].all()) and float(clear.float().mean()) > 0.75
    assert bool((d2[:100, 0] == 0).all()) and bool((idx[:100, 0].long() == torch.arange(700, 800, device="cuda")).all())
    assert bool((d2[700:, 0] == 0).all()) and bool((idx[700:, 0].long() == torch.arange(0, 100, device="cuda")).all())


@pytest.mark.parametrize("k", [1, 15, 24])
def test_wide_dense_equals_narrow_search(k):
    for n, d in ((1000, 65), (3000, 784)):
        X = _dense_matrix(n, d, 11 * k + n)
        i1, d1 = _dense(X, k, wide=False)
        i2, d2 = _dense(X, k, wide=True)
        assert torch.equal(d1, d2)  # bit-identical: the same re-rank arithmetic on the same candidates
        r, c = torch.nonzero(i1 != i2, as_tuple=True)
        # a differing index sits inside an exact tie: its distance occurs twice in the row, or is the k-th (tied
        # with a row outside the list)
        tied = ((d1[r] == d1[r, c][:, None]).sum(1) >= 2) | (d1[r, c] == d1[r, k - 1])
        assert bool(tied.all())


def _sparse_cases():
    empty = _random_csr(300, 400, 0.05, seed=1).tolil()
    empty[np.arange(5, 300, 7)] = 0
    empty = empty.tocsr()
    empty.eliminate_zeros()
    base = _random_csr(500, 2000, 0.03, seed=2)
    return {
        "random": _random_csr(1000, 3000, 0.02, seed=21),
        "dense_random": _random_csr(600, 500, 1.0, seed=22),
        "clustered": _clustered(1500, 20000, 30, 25, seed=23, size=60),
        "empty_rows": empty,
        "duplicated_rows": sp.vstack([base, base[:100]]).tocsr(),
        "no_nonzeros": sp.csr_matrix((200, 50), dtype=np.float32),
    }


_CASES = None


@pytest.mark.parametrize("name", ["random", "dense_random", "clustered", "empty_rows", "duplicated_rows",
                                  "no_nonzeros"])
@pytest.mark.parametrize("k", [25, 40, 64])
def test_wide_sparse_matches_fp64_brute_force(name, k):
    global _CASES
    if _CASES is None:
        _CASES = _sparse_cases()
    A = _CASES[name]
    from pymde_b200.preprocess import data_matrix as dm
    csr, shape = dm._to_device_csr(A, "cuda")
    idx, d2 = dm.knn_sparse_device(csr, shape, k)  # k > 24 selects mde_knn_csr_wide
    ri, rd = _brute_all_pairs(A, k)
    got_i, got_d = idx.cpu().numpy(), d2.cpu().numpy()
    assert _ulps(got_d, rd).max() <= 1
    # the order is (distance, index) of the device's once-rounded fp64 sums; a 1-ulp difference of the host's sum can
    # only swap rows whose distances are within that ulp
    same = (got_i == ri).all(1)
    if not same.all():
        bad = np.nonzero(~same)[0]
        assert (_ulps(got_d[bad], rd[bad]).max(1) >= 1).all()
        assert (np.sort(got_i[bad], 1) == np.sort(ri[bad], 1)).mean() > 0.99 or len(bad) < 3
    assert same.mean() > 0.999


@pytest.mark.parametrize("k", [10, 24])
def test_wide_sparse_equals_narrow_search(k):
    for A in (_random_csr(1000, 20000, 0.01, seed=31), _clustered(3003, 20000, 30, 273, seed=5, size=11)):
        i1, d1 = _sparse(A, k, wide=False)
        i2, d2 = _sparse(A, k, wide=True)
        assert torch.equal(i1, i2) and torch.equal(d1, d2)


def test_wide_sparse_never_densifies():
    from pymde_b200 import preprocess
    A = _clustered(100_000, 1_000_000, 10, 2000, seed=9)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    g = preprocess.k_nearest_neighbors(A, k=40)
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 2 * 2 ** 30, peak
    assert g.n_items == 100_000 and g.edges.shape[0] >= 100_000 * 40 // 2


def test_wide_k_nearest_neighbors_matches_gemm_path_away_from_ties(monkeypatch):
    from pymde_b200 import preprocess
    rng = np.random.default_rng(3)
    X = rng.standard_normal((1500, 32)).astype(np.float32)
    g1 = preprocess.k_nearest_neighbors(X, k=30)
    monkeypatch.setenv("PYMDE_B200_KNN", "gemm")
    g2 = preprocess.k_nearest_neighbors(X, k=30)
    e1 = set(map(tuple, np.asarray(g1.edges.cpu()).tolist()))
    e2 = set(map(tuple, np.asarray(g2.edges.cpu()).tolist()))
    assert len(e1 ^ e2) <= 0.001 * len(e1)  # the GEMM path is not exact near ties


def test_wide_recipes_accept_csr():
    import pymde_b200 as pm
    from pymde_b200 import util
    A = _clustered(1204, 5000, 20, 172, seed=7, size=7)
    util.seed(0)
    m1 = pm.preserve_neighbors(A, n_neighbors=30, init="random", device="cuda")
    util.seed(0)
    m2 = pm.preserve_neighbors(A.toarray(), n_neighbors=30, init="random", device="cuda")
    assert bool((m1.edges == m2.edges).all())
    X = m1.embed(max_iter=30)
    assert X.shape == (1204, 2) and bool(torch.isfinite(X).all())


def test_wide_abi_rejections():
    L, lib = _lib()
    assert lib.mde_knn_wide_max_k() == 64
    n, d = 70, 4
    X = torch.randn((n, d), device="cuda")
    oi = torch.empty((n, 70), dtype=torch.int32, device="cuda")
    od = torch.empty((n, 70), dtype=torch.float32, device="cuda")
    need = C.c_size_t(0)
    assert lib.mde_knn_wide_ws_bytes(n, d, C.byref(need)) == 0 and need.value > 0
    ws, p = _ws(need.value + 1024)

    def dense(k, ptr=p, nbytes=need.value):
        return lib.mde_knn_wide(X.data_ptr(), n, d, k, oi.data_ptr(), od.data_ptr(), ptr, nbytes, None)

    assert dense(64) == 0
    torch.cuda.synchronize()
    for k in (0, 65, n):
        assert dense(k) == L.MDE_E_INVALID
    assert dense(30, nbytes=need.value - 1) == L.MDE_E_INVALID
    assert dense(30, ptr=p + 256) == L.MDE_E_INVALID

    A = _random_csr(n, 8, 0.5, seed=11)
    A.sort_indices()
    nnz = A.nnz
    assert lib.mde_knn_csr_wide_ws_bytes(n, 8, nnz, C.byref(need)) == 0 and need.value > 0
    ws2, p2 = _ws(need.value + 1024)

    def sparse(indices, k=30, ptr=p2, nbytes=need.value):
        ip = torch.tensor(A.indptr, dtype=torch.int64, device="cuda")
        ix = torch.tensor(indices, dtype=torch.int32, device="cuda")
        v = torch.tensor(A.data, dtype=torch.float32, device="cuda")
        return lib.mde_knn_csr_wide(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, 8, nnz, k, oi.data_ptr(),
                                    od.data_ptr(), ptr, nbytes, None)

    assert sparse(A.indices) == 0
    for k in (0, 65, n):
        assert sparse(A.indices, k=k) == L.MDE_E_INVALID
    assert sparse(A.indices, nbytes=need.value - 1) == L.MDE_E_INVALID
    assert sparse(A.indices, ptr=p2 + 256) == L.MDE_E_INVALID
    r = int(np.argmax(np.diff(A.indptr)))
    bad = A.indices.copy()
    bad[A.indptr[r]], bad[A.indptr[r] + 1] = bad[A.indptr[r] + 1], bad[A.indptr[r]]
    assert sparse(bad) == L.MDE_E_INVALID
    bad = A.indices.copy()
    bad[-1] = 8
    assert sparse(bad) == L.MDE_E_INVALID
