"""Row f3 for 64 < k <= 256: `mde_knn_long` and `mde_knn_csr_long` (csrc/mde_knn.cu, csrc/mde_knn_sparse.cu: a
running top-288 per query row in shared memory) against fp64 brute forces and against the wide searches where both
apply; the long neighbour-graph builder against `Graph.from_edges`; and both through `k_nearest_neighbors` and the
recipes, without densifying sparse input."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.test_gpu_knn import _brute64 as _brute64_dense
from tests.test_gpu_knn import _compare as _compare_dense
from tests.test_gpu_knn_graph import _assert_same, _blobs, _random_lists
from tests.test_gpu_knn_graph import _sparse as _blobs_sparse
from tests.test_gpu_knn_sparse import _clustered, _random_csr, _ulps
from tests.test_gpu_knn_wide import _brute_all_pairs, _dense_matrix, _ws

pytestmark = pytest.mark.gpu

KS = [65, 100, 128, 200, 256]


def _lib():
    from pymde_b200 import _lib as L
    return L, L.load()


def _dense(X, k, entry):
    """One call of mde_knn_long ("long") or mde_knn_wide ("wide")."""
    L, lib = _lib()
    X = X.contiguous()
    n, d = X.shape
    need = C.c_size_t(0)
    L.check(getattr(lib, "mde_knn_%s_ws_bytes" % entry)(n, d, C.byref(need)))
    ws, p = _ws(need.value)
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    L.check(getattr(lib, "mde_knn_%s" % entry)(X.data_ptr(), n, d, k, idx.data_ptr(), d2.data_ptr(), p, need.value,
                                               None))
    torch.cuda.synchronize()
    return idx, d2


def _sparse(A, k, entry):
    """One call of mde_knn_csr_long ("long") or mde_knn_csr_wide ("wide")."""
    from pymde_b200.preprocess import data_matrix as dm
    L, lib = _lib()
    (ip, ix, v), (n, d) = dm._to_device_csr(A, "cuda")
    nnz = int(ix.shape[0])
    need = C.c_size_t(0)
    L.check(getattr(lib, "mde_knn_csr_%s_ws_bytes" % entry)(n, d, nnz, C.byref(need)))
    ws, p = _ws(need.value)
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    L.check(getattr(lib, "mde_knn_csr_%s" % entry)(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz, k,
                                                   idx.data_ptr(), d2.data_ptr(), p, need.value, None))
    return idx, d2


def _assert_tie_only_differences(i1, d1, i2, d2):
    """Bit-identical distances; an index may differ only inside an exact tie (its distance occurs twice in the row,
    or equals the last one, tied with a row outside the list)."""
    assert torch.equal(d1, d2)
    r, c = torch.nonzero(i1 != i2, as_tuple=True)
    k = d1.shape[1]
    tied = ((d1[r] == d1[r, c][:, None]).sum(1) >= 2) | (d1[r, c] == d1[r, k - 1])
    assert bool(tied.all())


# --- dense -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,d,k", [(1000, 65, 65), (1500, 32, 100), (2001, 200, 128), (2500, 784, 200),
                                   (3001, 64, 256), (257, 16, 256)])
def test_long_dense_matches_fp64_brute_force(n, d, k):
    from pymde_b200.preprocess import data_matrix as dm
    X = _dense_matrix(n, d, 7 * n + d)
    idx, d2 = dm.knn_device(X, k)  # k > 64 selects mde_knn_long
    _compare_dense(X, k, idx, d2)
    if k == n - 1:  # every other row is a neighbour
        assert bool((torch.sort(idx.long(), 1)[0].sum(1) == n * (n - 1) // 2 - torch.arange(n, device="cuda")).all())


def test_long_dense_duplicates_and_far_offsets():
    g = torch.Generator(device="cuda").manual_seed(8)
    base = torch.randn((900, 48), generator=g, device="cuda")
    X = torch.cat([base, base[:100]], 0) + 30.0
    n, k = 1000, 100
    idx, d2 = _dense(X, k, "long")
    val, ref = _brute64_dense(X, k)
    got = idx.long()
    assert not bool((got == torch.arange(n, device="cuda")[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())
    gd = ((X.double()[:, None, :] - X.double()[got]) ** 2).sum(-1)
    np.testing.assert_allclose(gd.cpu().numpy(), val[:, :k].cpu().numpy(), rtol=2e-6, atol=1e-9)
    np.testing.assert_allclose(d2.double().cpu().numpy(), gd.cpu().numpy(), rtol=2e-6, atol=1e-9)
    assert bool((d2[:, 1:] >= d2[:, :-1]).all())
    clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-9
    assert bool((s == torch.sort(ref, 1)[0]).all(1)[clear].all()) and float(clear.float().mean()) > 0.75
    # the duplicate comes first, at distance 0 (an exact tie broken by index against any other zero)
    assert bool((d2[:100, 0] == 0).all()) and bool((idx[:100, 0].long() == torch.arange(900, 1000, device="cuda")).all())
    assert bool((d2[900:, 0] == 0).all()) and bool((idx[900:, 0].long() == torch.arange(0, 100, device="cuda")).all())


@pytest.mark.parametrize("n,d", [(3000, 64), (2000, 784), (1111, 7)])
def test_long_dense_prefix_is_the_wide_search(n, d):
    X = _dense_matrix(n, d, 3 * n + d)
    iw, dw = _dense(X, 64, "wide")
    il, dl = _dense(X, 256, "long")
    _assert_tie_only_differences(iw, dw, il[:, :64].contiguous(), dl[:, :64].contiguous())
    i64, d64 = _dense(X, 64, "long")
    _assert_tie_only_differences(iw, dw, i64, d64)


# --- sparse ------------------------------------------------------------------------------------------------------------

def _sparse_cases():
    empty = _random_csr(300, 400, 0.05, seed=41).tolil()
    empty[np.arange(5, 300, 7)] = 0
    empty = empty.tocsr()
    empty.eliminate_zeros()
    base = _random_csr(500, 2000, 0.03, seed=42)
    return {
        "random": _random_csr(1000, 3000, 0.02, seed=43),
        "clustered_text": _clustered(1500, 20000, 30, 25, seed=44, size=60),
        "empty_rows": empty,
        "duplicated_rows": sp.vstack([base, base[:100]]).tocsr(),
        "no_nonzeros": sp.csr_matrix((200, 50), dtype=np.float32),
        "one_feature": _random_csr(601, 1, 0.6, seed=45),
    }


_CASES = {}


def _case(name):
    """(matrix, fp64 brute force at k = min(256, n - 1)); the brute force is a stable sort, so its prefixes are the
    brute forces of the smaller k."""
    if not _CASES:
        for key, A in _sparse_cases().items():
            _CASES[key] = [A, None]
    entry = _CASES[name]
    if entry[1] is None:
        entry[1] = _brute_all_pairs(entry[0], min(256, entry[0].shape[0] - 1))
    return entry


@pytest.mark.parametrize("name", ["random", "clustered_text", "empty_rows", "duplicated_rows", "no_nonzeros",
                                  "one_feature"])
@pytest.mark.parametrize("k", KS)
def test_long_sparse_matches_fp64_brute_force(name, k):
    from pymde_b200.preprocess import data_matrix as dm
    A, (ri, rd) = _case(name)
    k = min(k, A.shape[0] - 1)
    csr, shape = dm._to_device_csr(A, "cuda")
    idx, d2 = dm.knn_sparse_device(csr, shape, k)  # k > 64 selects mde_knn_csr_long
    ri, rd = ri[:, :k], rd[:, :k]
    got_i, got_d = idx.cpu().numpy(), d2.cpu().numpy()
    # the device sums in fp64 in its own column order and rounds once: a last-place difference from the host's fp64
    # sum is possible, and only such a difference may reorder rows
    assert _ulps(got_d, rd).max() <= 1
    same = (got_i == ri).all(1)
    if not same.all():
        bad = np.nonzero(~same)[0]
        assert (_ulps(got_d[bad], rd[bad]).max(1) >= 1).all()
    assert same.mean() > 0.999
    if name == "no_nonzeros":  # every distance is 0: the k lowest other indices, in order
        assert (got_d == 0).all()
        assert (got_i == ri).all()


@pytest.mark.parametrize("name", ["random", "clustered_text", "duplicated_rows", "empty_rows"])
def test_long_sparse_prefix_is_the_wide_search(name):
    A = _case(name)[0]
    iw, dw = _sparse(A, 64, "wide")
    il, dl = _sparse(A, 256, "long")
    assert torch.equal(iw, il[:, :64]) and torch.equal(dw, dl[:, :64])
    i64, d64 = _sparse(A, 64, "long")
    assert torch.equal(iw, i64) and torch.equal(dw, d64)


def test_sparse_input_is_never_densified(monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import preprocess

    def refuse(self, *args, **kwargs):
        raise AssertionError("a sparse matrix was densified")

    for name in dir(sp):
        cls = getattr(sp, name)
        if isinstance(cls, type) and hasattr(cls, "toarray"):
            monkeypatch.setattr(cls, "toarray", refuse)
            monkeypatch.setattr(cls, "todense", refuse)
    A = _clustered(4000, 100_000, 20, 40, seed=12)
    with pytest.raises(AssertionError):
        A.toarray()
    g = preprocess.k_nearest_neighbors(A, k=200)
    assert g.n_items == 4000 and g.edges.shape[0] >= 4000 * 200 // 2
    pm.seed(0)
    mde = pm.preserve_neighbors(A, n_neighbors=100, device="cuda")
    assert mde.edges.is_cuda and mde.edges.shape[0] >= 4000 * 100 // 2


# --- routing -----------------------------------------------------------------------------------------------------------

def test_long_k_nearest_neighbors_matches_gemm_path_away_from_ties(monkeypatch):
    from pymde_b200 import preprocess
    rng = np.random.default_rng(4)
    X = rng.standard_normal((2000, 32)).astype(np.float32)
    g1 = preprocess.k_nearest_neighbors(X, k=150)  # dense input: the GEMM path above k = 64
    monkeypatch.setenv("PYMDE_B200_KNN", "approx")  # ... and mde_knn_long with the opt-in
    g2 = preprocess.k_nearest_neighbors(X, k=150)
    e1 = set(map(tuple, np.asarray(g1.edges.cpu()).tolist()))
    e2 = set(map(tuple, np.asarray(g2.edges.cpu()).tolist()))
    assert len(e1 ^ e2) <= 0.001 * len(e1)  # the GEMM path is not exact near ties


@pytest.mark.parametrize("sparse", [False, True])
def test_approx_modes_take_the_exact_long_search_above_64(monkeypatch, sparse):
    from pymde_b200.preprocess import data_matrix as dm
    X = _blobs(1500, 12, 5)
    data = _blobs_sparse(X) if sparse else X
    if sparse:
        i1, d1, _ = dm._search(data, 100, torch.device("cuda"))
    else:
        i1, d1 = dm.knn_device(torch.from_numpy(X).cuda(), 100)
    monkeypatch.setenv("PYMDE_B200_KNN_SPARSE" if sparse else "PYMDE_B200_KNN", "approx")
    i2, d2, _ = dm._search(data, 100, torch.device("cuda"))
    assert i1.dtype == i2.dtype == torch.int32  # a search kernel, not the GEMM path
    assert torch.equal(i1, i2) and torch.equal(d1, d2)


# --- graph -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [65, 128, 256])
def test_long_lists_match_from_edges(k):
    n = 3000
    idx = _random_lists(n, k, 200 + k, holes=0.2)
    idx[::11] = -1                      # rows with no entry at all
    idx[1::5, 1::2] = idx[1::5, 0:k - 1:2]  # duplicates inside rows
    idx[:, -1] = 13                     # a hub: every row lists row 13 ...
    idx[13, -1] = -1                    # ... except row 13 itself
    idx[7, :] = 3                       # one value k times (a multiplicity of up to 256)
    e, w = _assert_same(idx)
    assert float(w.max()) >= k


def test_long_fully_reciprocal_lists():
    n, k = 257, 256
    idx = np.stack([np.array([j for j in range(n) if j != i]) for i in range(n)]).astype(np.int32)
    idx = np.stack([np.random.default_rng(i).permutation(r) for i, r in enumerate(idx)])
    e, w = _assert_same(idx)
    assert e.shape[0] == n * (n - 1) // 2 and bool((w == 2).all())


def test_csr_workspace_grows_with_n_and_nnz():
    L, lib = _lib()

    def ws(n, d, nnz, entry="long"):
        need = C.c_size_t(0)
        L.check(getattr(lib, "mde_knn_csr_%s_ws_bytes" % entry)(n, d, nnz, C.byref(need)))
        return need.value

    base = ws(10000, 5000, 100000)
    assert base % 1024 == 0 and ws(10000, 5000, 0) > 0
    assert ws(20000, 5000, 100000) > base and ws(10000, 5000, 200000) > base
    assert base - ws(10000, 5000, 100000, "wide") >= 1536 * 10000 - 4096  # 288 candidates per row against 96


def test_csr_workspace_too_small_or_misaligned_is_rejected():
    L, lib = _lib()
    need = C.c_size_t(0)
    L.check(lib.mde_knn_csr_long_ws_bytes(1000, 30, 500, C.byref(need)))
    fake = 1 << 20  # never dereferenced: the workspace check comes first

    def call(nnz, ws, nbytes):
        return lib.mde_knn_csr_long(fake, fake, fake, 1000, 30, nnz, 100, fake, fake, ws, nbytes, None)

    assert call(500, fake, need.value - 1) == L.MDE_E_INVALID
    assert call(500, fake + 512, need.value) == L.MDE_E_INVALID
    assert call(600, fake, need.value) == L.MDE_E_INVALID  # more non-zeros


def test_device_knn_long_refuses_k_above_256():
    from pymde_b200.preprocess import data_matrix as dm
    with pytest.raises(ValueError):
        dm.k_nearest_neighbors_device_long(_blobs(300, 4, 1), 257)


@pytest.mark.parametrize("search", ["dense", "sparse", "approx", "gemm"])
@pytest.mark.parametrize("max_distance", [None, 4.0])
@pytest.mark.parametrize("k", [1, 65, 200])
def test_device_knn_long_matches_the_host_graph(monkeypatch, search, max_distance, k):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    X = _blobs(2000, 12, 19)
    data = _blobs_sparse(X) if search == "sparse" else X
    if search in ("approx", "gemm"):
        monkeypatch.setenv("PYMDE_B200_KNN", search)
    pm.seed(1)
    g_ref = dm.k_nearest_neighbors(data, k, max_distance=max_distance)
    pm.seed(1)
    g = dm.k_nearest_neighbors_device_long(data, k, max_distance=max_distance)
    assert g.edges.is_cuda and g.weights.is_cuda and g.n_items == 2000
    assert torch.equal(g.edges.cpu(), g_ref.edges)
    assert torch.equal(g.weights.cpu(), g_ref.weights)


@pytest.mark.parametrize("sparse", [False, True])
def test_preserve_neighbors_100_matches_the_host_graph_and_embeds(monkeypatch, sparse):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    X = _blobs(3000, 16, 21, dup=20)
    data = _blobs_sparse(X) if sparse else X

    def problem():
        pm.seed(3)
        mde = pm.preserve_neighbors(data, n_neighbors=100, device="cuda")
        f = mde.distortion_function
        return mde, mde.edges.clone(), (f.weights if hasattr(f, "weights") else f.deviations).clone()

    mde, e_dev, w_dev = problem()
    calls = []

    def host(data, k, max_distance=None, device=None):
        calls.append(k)
        return dm.k_nearest_neighbors(data, k, max_distance=max_distance, device=device)

    with monkeypatch.context() as m:
        m.setattr(dm, "k_nearest_neighbors_device_long", host)
        _, e_host, w_host = problem()
    assert calls == [100]  # above 64 the recipe assembles the graph with the long builder
    assert torch.equal(e_dev, e_host) and torch.equal(w_dev, w_host)
    Y = mde.embed(max_iter=40)
    assert Y.shape == (3000, 2) and bool(torch.isfinite(Y).all())
    assert np.isfinite(float(mde.distortions().mean()))
