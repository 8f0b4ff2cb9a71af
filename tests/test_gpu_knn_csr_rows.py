"""The row-range sparse exact search (`mde_knn_csr_rows`, csrc/mde_knn_sparse.cu) against the full sparse searches:
row r of a search of rows [row_begin, row_end) must be row row_begin + r of `mde_knn_csr` / `mde_knn_csr_wide` /
`mde_knn_csr_long` bit for bit, indices and distances, ties included -- with the candidate sweep split into slices
and without, on ranges that do and do not start on a tile, on uniform, Zipf-column, zero-row, tied and
disjoint-vocabulary matrices.  `embed_new_points` on sparse input takes it and never the full search."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

KS = [1, 7, 15, 24, 25, 40, 64, 65, 100, 256]


def _ranges(n):
    out = [(0, 1), (n - 1, n), (37, 41), (1000, 1300), (n - 3000, n), (0, n)]
    return [(a, b) for a, b in out if 0 <= a < b <= n]


def rows_search(csr, shape, k, rb, re):
    """(idx, d2) from mde_knn_csr_rows on a workspace filled with 0xA5 and outputs filled with -7."""
    from pymde_b200 import _lib
    lib = _lib.load()
    ip, ix, v = csr
    n, d = shape
    nnz = int(ix.shape[0])
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_csr_rows_ws_bytes(n, d, nnz, re - rb, k, C.byref(need)))
    ws = torch.full((need.value + 1024,), 0xA5, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.full((re - rb, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((re - rb, k), -7.0, dtype=torch.float32, device="cuda")
    _lib.check(lib.mde_knn_csr_rows(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz, rb, re, k, idx.data_ptr(),
                                    d2.data_ptr(), p, need.value, None))
    torch.cuda.synchronize()
    return idx, d2


def _slices(n, rows, k):
    from pymde_b200 import _lib
    return _lib.load().mde_dbg_knn_csr_slices(n, rows, k)


def _check_rows(A, ks, ranges=None, seen=None):
    from pymde_b200.preprocess import data_matrix as dm
    csr, shape = dm._to_device_csr(A, torch.device("cuda"))
    n = shape[0]
    for k in ks:
        if k > n - 1:
            continue
        full_i, full_d = dm.knn_sparse_device(csr, shape, k)
        for rb, re in ranges or _ranges(n):
            i, d2 = rows_search(csr, shape, k, rb, re)
            assert torch.equal(i, full_i[rb:re]), (n, k, rb, re)
            assert torch.equal(d2, full_d[rb:re]), (n, k, rb, re)
            if seen is not None:
                seen.add(_slices(n, re - rb, k))


# --- data families --------------------------------------------------------------------------------------------------

def uniform(n, d=2000, density=0.01, seed=0):
    rng = np.random.default_rng(seed)
    return sp.random(n, d, density=density, format="csr", random_state=rng, dtype=np.float32)


def zipf(n, d=3000, per_row=40, seed=1, binary=False):
    """Columns drawn with probability ~ 1 / rank^1.1, as the terms of a TF-IDF or count matrix."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, d + 1) ** 1.1
    p /= p.sum()
    cols = rng.choice(d, size=(n, per_row), p=p)
    rows = np.repeat(np.arange(n), per_row)
    vals = np.ones(n * per_row, np.float32) if binary else rng.random(n * per_row).astype(np.float32)
    A = sp.csr_matrix((vals, (rows, cols.reshape(-1))), shape=(n, d))
    A.sum_duplicates()
    if binary:
        A.data[:] = np.minimum(A.data, 3.0)  # small counts: many equal distances
    return A


def zero_rows(n, seed=2):
    A = uniform(n, seed=seed).tolil()
    rng = np.random.default_rng(seed)
    for r in rng.choice(n, n // 5, replace=False):
        A.rows[r], A.data[r] = [], []
    for r in range(min(n, 1000), min(n, 1300)):  # a run of whole zero tiles
        A.rows[r], A.data[r] = [], []
    return A.tocsr()


def duplicates(n, seed=3):
    """Binary count rows, each repeated: exact duplicates and many exact ties."""
    base = zipf((n + 3) // 4, d=500, per_row=12, seed=seed, binary=True)
    rng = np.random.default_rng(seed)
    return base[rng.integers(0, base.shape[0], n)].tocsr()


def two_vocabularies(n, seed=4):
    """The first half of the rows uses 512 frequent columns, the second 2 560 rare ones: after the features are
    ordered by document frequency the two halves occupy disjoint K blocks, so their tile pairs intersect in none."""
    rng = np.random.default_rng(seed)
    h = n // 2
    a = sp.random(h, 512, density=40 / 512, format="csr", random_state=rng, dtype=np.float32)
    b = sp.random(n - h, 2560, density=40 / 2560, format="csr", random_state=rng, dtype=np.float32)
    return sp.block_diag([a, b], format="csr").astype(np.float32)


FAMILIES = {"uniform": uniform, "zipf": zipf, "zero_rows": zero_rows, "duplicates": duplicates,
            "two_vocabularies": two_vocabularies}


# --- tests ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [130, 5000, 40000])
def test_rows_equal_the_full_search(n):
    seen = set()
    A = uniform(n, d=2000, density=0.01 if n < 40000 else 0.005)
    _check_rows(A, KS, seen=seen)
    if n >= 5000:
        assert 1 in seen and max(seen) > 1, seen  # both split and unsplit sweeps ran


@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_rows_on_every_data_family(name):
    A = FAMILIES[name](5000)
    _check_rows(A, [1, 15, 40, 100], ranges=[(0, 1), (37, 41), (1000, 1300), (2500, 2700), (2000, 5000), (0, 5000)])


def test_slice_rule_covers_both_cases():
    assert _slices(5000, 4, 15) > 1 and _slices(5000, 300, 40) > 1
    assert _slices(40000, 40000, 15) == 1 and _slices(5000, 300, 100) == 1


@pytest.mark.parametrize("k", [1, 15, 40, 100])
@pytest.mark.parametrize("n,rb,re", [(130, 0, 130), (2000, 37, 41), (2000, 1500, 2000)])
def test_rows_agree_with_an_fp64_brute_force(n, rb, re, k):
    from pymde_b200.preprocess import data_matrix as dm
    if k > n - 1:
        return
    A = uniform(n, d=300, density=0.05, seed=5)
    csr, shape = dm._to_device_csr(A, torch.device("cuda"))
    idx, d2 = rows_search(csr, shape, k, rb, re)
    X = A.toarray().astype(np.float64)
    D = ((X[rb:re, None, :] - X[None, :, :]) ** 2).sum(-1)
    D[np.arange(re - rb), np.arange(rb, re)] = np.inf
    order = np.argsort(D, axis=1, kind="stable")
    got = idx.long().cpu().numpy()
    # fp64 sums rounded once to fp32
    np.testing.assert_allclose(d2.double().cpu().numpy(), np.take_along_axis(D, got, 1), rtol=1e-7, atol=0)
    ref = np.take_along_axis(D, order[:, :k + 1], 1)
    np.testing.assert_allclose(d2.double().cpu().numpy(), ref[:, :k], rtol=1e-7, atol=0)
    clear = ref[:, k] - ref[:, k - 1] > 1e-5 * ref[:, k] if k < n - 1 else np.ones(re - rb, bool)
    for r in np.nonzero(clear)[0]:
        assert set(got[r]) == set(order[r, :k])


def test_malformed_csr_is_refused():
    from pymde_b200 import _lib
    lib = _lib.load()
    A = uniform(600, d=100, density=0.05, seed=6)
    ip = torch.from_numpy(A.indptr.astype(np.int64)).cuda()
    ix = A.indices.astype(np.int32).copy()
    r = int(np.argmax(np.diff(A.indptr) >= 2))
    ix[A.indptr[r]], ix[A.indptr[r] + 1] = ix[A.indptr[r] + 1], ix[A.indptr[r]]  # not increasing within a row
    ix = torch.from_numpy(ix).cuda()
    v = torch.from_numpy(A.data.astype(np.float32)).cuda()
    n, d, nnz = 600, 100, int(A.nnz)
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_csr_rows_ws_bytes(n, d, nnz, 100, 15, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    oi = torch.full((100, 15), -7, dtype=torch.int32, device="cuda")
    od = torch.full((100, 15), -7.0, dtype=torch.float32, device="cuda")
    code = lib.mde_knn_csr_rows(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz, 200, 300, 15, oi.data_ptr(),
                                od.data_ptr(), p, need.value, None)
    assert code == _lib.MDE_E_INVALID
    assert bool((oi == -7).all()) and bool((od == -7.0).all())


def test_knn_rows_device_routes_sparse_input_to_the_row_search(monkeypatch):
    from pymde_b200.preprocess import data_matrix as dm
    A = zipf(3000)
    csr, shape = dm._to_device_csr(A, torch.device("cuda"))
    full = {k: dm.knn_sparse_device(csr, shape, k) for k in (15, 100)}

    def refuse(*args, **kwargs):
        raise AssertionError("the full sparse search ran")

    monkeypatch.setattr(dm, "knn_sparse_device", refuse)
    for k, (fi, fd) in full.items():
        i, d2 = dm.knn_rows_device(A, k, 2000, 3000)
        assert i.dtype == torch.int32
        assert torch.equal(i, fi[2000:]) and torch.equal(d2, fd[2000:])


def test_embed_new_points_on_sparse_input_matches_the_full_search_route(monkeypatch):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    data = zipf(6000, seed=7)
    new = zipf(400, seed=8)
    pm.seed(0)
    emb = pm.preserve_neighbors(data, embedding_dim=2).embed()
    original = dm.knn_sparse_device

    def refuse(*args, **kwargs):
        raise AssertionError("the full sparse search ran")

    with monkeypatch.context() as m:
        m.setattr(dm, "knn_sparse_device", refuse)
        pm.seed(0)
        got = pm.embed_new_points(data, emb, new)

    def full_then_slice(csr, shape, k, row_begin, row_end):  # the route before the row search
        idx, d2 = original(csr, shape, k)
        return idx[row_begin:row_end].contiguous(), d2[row_begin:row_end].contiguous()

    with monkeypatch.context() as m:
        m.setattr(dm, "knn_sparse_rows_device", full_then_slice)
        pm.seed(0)
        want = pm.embed_new_points(data, emb, new)
    assert got.shape == (400, 2) and bool(torch.isfinite(got).all())
    assert torch.equal(got, want)
