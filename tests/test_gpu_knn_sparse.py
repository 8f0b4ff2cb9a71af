"""Row f3 on sparse input: `mde_knn_csr` and `mde_pair_dist_csr` (csrc/mde_knn_sparse.cu) against fp64 brute force.

Contract: the k nearest other rows, ordered by (distance, index), with the exact squared distance summed in fp64
and rounded once to fp32.  The reference (pymde/preprocess/data_matrix.py:19,99) accepts scipy.sparse input for
the k-NN and the pair distances without densifying it."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu


def _random_csr(n, d, density, seed):
    rng = np.random.default_rng(seed)
    A = sp.random(n, d, density=density, format="csr", dtype=np.float32, random_state=rng)
    A.data = rng.standard_normal(A.nnz).astype(np.float32)
    return A


def _knn(A, k):
    from pymde_b200.preprocess import data_matrix as dm
    csr, shape = dm._to_device_csr(A, "cuda")
    return dm.knn_sparse_device(csr, shape, k)


def _exact_d2(Xd, rows, cols):
    """fp64 sum (x_r - x_c)^2 for rows [n] against cols [n, m], in row chunks."""
    out = torch.empty(cols.shape, dtype=torch.float64, device=Xd.device)
    step = max(1, (1 << 26) // (cols.shape[1] * Xd.shape[1]))
    for s0 in range(0, cols.shape[0], step):
        r = rows[s0:s0 + step]
        out[s0:s0 + step] = ((Xd[r][:, None, :] - Xd[cols[s0:s0 + step]]) ** 2).sum(-1)
    return out


def _brute64(X, k):
    """Exact fp64 search: candidates from the fp64 norm expansion (k + 9 of them), then sum (q - x)^2 in fp64.
    Returns the k + 1 smallest squared distances (the extra one measures the gap behind the k-th) and the indices
    of the k smallest, by (distance, index)."""
    Xd = X.double()
    n = X.shape[0]
    kk = min(n - 1, k + 9)
    sq = (Xd * Xd).sum(1)
    cand = torch.empty((n, kk), dtype=torch.int64, device=X.device)
    for s0 in range(0, n, 1024):
        d2 = sq[s0:s0 + 1024, None] + sq[None, :] - 2.0 * Xd[s0:s0 + 1024] @ Xd.T
        d2[torch.arange(d2.shape[0]), torch.arange(s0, s0 + d2.shape[0])] = float("inf")
        cand[s0:s0 + 1024] = torch.topk(d2, kk, dim=1, largest=False)[1]
    exact = _exact_d2(Xd, torch.arange(n, device=X.device), cand)
    cand, pos = torch.sort(cand, dim=1)  # stable sort by value below keeps index order among equal distances
    exact = torch.gather(exact, 1, pos)
    val, pos = torch.sort(exact, dim=1, stable=True)
    idx = torch.gather(cand, 1, pos)
    return val[:, :min(kk, k + 1)], idx[:, :k]


def _ulps(a, b):
    """Distance in units of the last place between fp32 arrays of non-negative values."""
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _compare(A, k, idx, d2, min_clear=0.9):
    n = A.shape[0]
    X = torch.tensor(A.toarray(), device="cuda")
    val, ref = _brute64(X, k)
    got = idx.long()
    assert int(got.min()) >= 0 and int(got.max()) < n
    assert not bool((got == torch.arange(n, device="cuda")[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())  # no repeats
    # distances: the fp64 sum rounded once to fp32 (the fp64 sums differ in order only, so a last-place difference
    # after the rounding is possible, and rare)
    ex = _exact_d2(X.double(), torch.arange(n, device="cuda"), got).float().cpu().numpy()
    dg = d2.cpu().numpy()
    u = _ulps(dg, ex)
    assert u.max() <= 1 and (u == 0).mean() >= 0.9999
    # ordered by (distance, index)
    dd, ii = d2[:, 1:], idx[:, 1:]
    dp, ip = d2[:, :-1], idx[:, :-1]
    assert bool(((dd > dp) | ((dd == dp) & (ii > ip))).all())
    # the k smallest: distances as the brute force, and the same rows wherever the k-th is clearly separated
    assert _ulps(dg, val[:, :k].float().cpu().numpy()).max() <= 1
    if val.shape[1] > k:
        clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-9
        same = (torch.sort(got, 1)[0] == torch.sort(ref, 1)[0]).all(1)
        assert bool(same[clear].all()) and float(clear.float().mean()) >= min_clear
        if bool(clear.any()):
            exact_order = (got == ref).all(1)
            assert float(exact_order[clear].float().mean()) > 0.99


@pytest.mark.parametrize("n,d,density,k", [(2, 5, 0.5, 1), (33, 1000, 0.05, 5), (1000, 20000, 0.01, 15),
                                           (4099, 3000, 0.1, 24), (600, 5000, 1.0, 10)])
def test_knn_csr_matches_fp64_brute_force(n, d, density, k):
    A = _random_csr(n, d, density, seed=n + d)
    idx, d2 = _knn(A, k)
    _compare(A, k, idx, d2)


def test_empty_rows_are_mutually_at_zero_resolved_by_index():
    A = _random_csr(300, 400, 0.05, seed=1).tolil()
    empty = np.arange(5, 300, 7)
    A[empty] = 0
    A = A.tocsr()
    A.eliminate_zeros()
    k = 10
    idx, d2 = _knn(A, k)
    for r in empty:
        want = [e for e in empty if e != r][:k]
        assert idx[r].tolist() == want
        assert bool((d2[r] == 0).all())
    # the other rows share few features, so their nearest rows are the empty ones, all at ||x||^2: again by index
    full = np.setdiff1d(np.arange(300), empty)
    at_norm = (d2[full] == d2[full, -1:]).all(1).cpu().numpy()
    assert at_norm.mean() > 0.5
    assert (idx[full[at_norm]].cpu().numpy() == empty[:k]).all()
    _compare(A, k, idx, d2, min_clear=0.0)


def test_duplicated_rows_find_their_copy_first():
    base = _random_csr(500, 2000, 0.03, seed=2)
    A = sp.vstack([base, base[:100]]).tocsr()
    idx, d2 = _knn(A, 6)
    assert bool((d2[:100, 0] == 0).all())
    assert bool((idx[:100, 0].long() == torch.arange(500, 600, device="cuda")).all())
    assert bool((idx[500:, 0].long() == torch.arange(0, 100, device="cuda")).all())
    # a row sharing no feature with a duplicated pair sees both copies at the same distance: no clear k-th gap there
    _compare(A, 6, idx, d2, min_clear=0.8)


def test_large_magnitude_values():
    A = _random_csr(700, 3000, 0.05, seed=3)
    A.data = (A.data * 1e6 + np.sign(A.data) * 3e6).astype(np.float32)
    idx, d2 = _knn(A, 8)
    _compare(A, 8, idx, d2)


def test_matrix_without_nonzeros():
    A = sp.csr_matrix((200, 50), dtype=np.float32)
    idx, d2 = _knn(A, 5)
    want = torch.tensor([[c for c in range(7) if c != r][:5] for r in range(200)], device="cuda")
    assert bool((idx.long() == want).all()) and bool((d2 == 0).all())


def test_tile_pairs_sharing_no_feature_block():
    """Four groups of 256 rows on disjoint 64-feature blocks: most (query tile, candidate tile) pairs share no K
    block, so their cross terms are exactly 0 without a single wgmma.  The offset keeps every group's rows nearer
    to each other than to any other group's."""
    rng = np.random.default_rng(4)
    blocks = []
    for g in range(4):
        B = np.zeros((256, 4096), np.float32)
        B[:, 1024 * g:1024 * g + 64] = rng.standard_normal((256, 64)).astype(np.float32) + 3.0
        blocks.append(B)
    A = sp.csr_matrix(np.concatenate(blocks))
    idx, d2 = _knn(A, 7)
    _compare(A, 7, idx, d2)
    group = torch.arange(1024, device="cuda") // 256
    assert bool((group[idx.long()] == group[:, None]).all())


def _clustered(n, d, nnz_row, n_centres, seed, size=None):
    """Rows drawn around sparse cluster centres: each row keeps its centre's support, with noisy values.  With
    `size`, every cluster has exactly `size` rows (shuffled), so a k-NN with k = size - 1 has clear k-th gaps."""
    rng = np.random.default_rng(seed)
    cols = np.stack([rng.choice(d, nnz_row, replace=False) for _ in range(n_centres)])
    vals = rng.standard_normal((n_centres, nnz_row)).astype(np.float32) * 4
    lab = rng.integers(0, n_centres, n) if size is None else rng.permutation(np.repeat(np.arange(n_centres), size))
    c = cols[lab].ravel()
    v = (vals[lab] + 0.1 * rng.standard_normal((n, nnz_row))).astype(np.float32).ravel()
    r = np.repeat(np.arange(n), nnz_row)
    return sp.csr_matrix((v, (r, c)), shape=(n, d))


def test_k_nearest_neighbors_sparse_matches_gemm_path(monkeypatch):
    from pymde_b200 import preprocess
    A = _clustered(3003, 20000, 30, 273, seed=5, size=11)
    g1 = preprocess.k_nearest_neighbors(A, k=10)
    monkeypatch.setenv("PYMDE_B200_KNN", "gemm")
    g2 = preprocess.k_nearest_neighbors(A, k=10)
    assert g1.n_items == g2.n_items == 3003
    e1 = np.asarray(g1.edges.cpu()); e2 = np.asarray(g2.edges.cpu())
    assert e1.shape == e2.shape and (e1 == e2).all()
    np.testing.assert_array_equal(np.asarray(g1.weights.cpu()), np.asarray(g2.weights.cpu()))


def test_k_nearest_neighbors_sparse_max_distance():
    from pymde_b200 import preprocess
    A = _random_csr(800, 500, 0.05, seed=6)
    idx, d2 = _knn(A, 5)
    md = float(d2.sqrt().median())
    g = preprocess.k_nearest_neighbors(A, k=5, max_distance=md)
    keep = (d2.sqrt() <= md).cpu().numpy()
    e = np.stack([np.repeat(np.arange(800), 5)[keep.ravel()], idx.cpu().numpy().ravel()[keep.ravel()]], 1)
    want = set(map(tuple, np.sort(e, 1).tolist()))
    assert set(map(tuple, np.asarray(g.edges.cpu()).tolist())) == want


def test_recipes_accept_csr():
    import pymde_b200 as pm
    from pymde_b200 import util
    A = _clustered(1204, 5000, 20, 172, seed=7, size=7)
    util.seed(0)  # the same negative edges for both
    m1 = pm.preserve_neighbors(A, n_neighbors=6, init="random", device="cuda")
    util.seed(0)
    m2 = pm.preserve_neighbors(A.toarray(), n_neighbors=6, init="random", device="cuda")
    assert bool((m1.edges == m2.edges).all())
    X = m1.embed(max_iter=30)
    assert X.shape == (1204, 2) and bool(torch.isfinite(X).all())
    lap = pm.laplacian_embedding(A, device="cuda")
    assert lap.edges.shape[0] > 0
    B = _random_csr(400, 3000, 0.02, seed=8)
    p1 = pm.preserve_distances(B, device="cuda")
    p2 = pm.preserve_distances(B.toarray(), device="cuda")
    assert bool((p1.edges == p2.edges).all())
    np.testing.assert_allclose(p1.distortion_function.deviations.cpu().numpy(),
                               p2.distortion_function.deviations.cpu().numpy(), rtol=2e-6, atol=1e-6)


def test_no_densifying_at_400_gb_dense_size():
    from pymde_b200 import preprocess
    A = _clustered(100_000, 1_000_000, 10, 2000, seed=9)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    g = preprocess.k_nearest_neighbors(A, k=10)
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 2 * 2 ** 30, peak
    assert g.n_items == 100_000 and g.edges.shape[0] >= 100_000 * 10 // 2


def test_pair_dist_csr_all_pairs():
    from pymde_b200.preprocess import data_matrix as dm
    A = _random_csr(3000, 5000, 0.02, seed=10)
    csr, shape = dm._to_device_csr(A, "cuda")
    pairs = torch.triu_indices(3000, 3000, 1, device="cuda").T.contiguous()
    got = dm._pair_dist_csr(csr, shape, pairs)
    Xd = torch.tensor(A.toarray(), device="cuda", dtype=torch.float64)
    want = torch.empty_like(got)
    step = 1 << 14
    for s0 in range(0, pairs.shape[0], step):
        p = pairs[s0:s0 + step]
        want[s0:s0 + step] = (Xd[p[:, 0]] - Xd[p[:, 1]]).norm(dim=1).float()
    u = _ulps(got.cpu().numpy(), want.cpu().numpy())
    assert u.max() <= 1 and (u == 0).mean() >= 0.9999


def test_abi_rejections():
    from pymde_b200 import _lib
    from pymde_b200.preprocess import data_matrix as dm
    lib = _lib.load()
    A = _random_csr(10, 8, 0.5, seed=11)
    A.sort_indices()
    n, d, nnz = 10, 8, A.nnz
    assert nnz >= 4 and all(A.indptr[1:] - A.indptr[:-1] >= 0)
    need = C.c_size_t(0)
    assert lib.mde_knn_csr_ws_bytes(n, d, nnz, C.byref(need)) == 0 and need.value > 0
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    oi = torch.empty((n, 25), dtype=torch.int32, device="cuda")
    od = torch.empty((n, 25), dtype=torch.float32, device="cuda")

    def run(indices, k=3, ws_bytes=need.value):
        ip = torch.tensor(A.indptr, dtype=torch.int64, device="cuda")
        ix = torch.tensor(indices, dtype=torch.int32, device="cuda")
        v = torch.tensor(A.data, dtype=torch.float32, device="cuda")
        return lib.mde_knn_csr(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz, k, oi.data_ptr(), od.data_ptr(),
                               p, ws_bytes, None)

    assert run(A.indices) == 0
    assert run(A.indices, k=25) == _lib.MDE_E_INVALID
    assert run(A.indices, ws_bytes=need.value - 1) == _lib.MDE_E_INVALID
    r = int(np.argmax(np.diff(A.indptr)))  # a row with at least two entries
    bad = A.indices.copy()
    bad[A.indptr[r]], bad[A.indptr[r] + 1] = bad[A.indptr[r] + 1], bad[A.indptr[r]]
    assert run(bad) == _lib.MDE_E_INVALID
    bad = A.indices.copy()
    bad[-1] = d
    assert run(bad) == _lib.MDE_E_INVALID
    csr, shape = dm._to_device_csr(A, "cuda")
    out = torch.empty(1, dtype=torch.float32, device="cuda")
    pairs = torch.tensor([[0, n]], dtype=torch.int64, device="cuda")
    assert lib.mde_pair_dist_csr(csr[0].data_ptr(), csr[1].data_ptr(), csr[2].data_ptr(), n, d, pairs.data_ptr(), 1,
                                 out.data_ptr(), None) == _lib.MDE_E_INVALID
