"""The row-range exact search (`mde_knn_rows`, `mde_knn16_rows`, csrc/mde_knn.cu) against the full searches: row r of
a search of rows [row_begin, row_end) must be row row_begin + r of `mde_knn` / `mde_knn_wide` (or their 16-bit
entries) bit for bit, indices and distances, ties included -- with the candidate sweep split into slices and without,
on ranges that do and do not start on a tile, on offset and far-clustered data (the certificate and the direct
search) and on exact duplicates.  `knn_rows_device` routes k > 64 and scipy.sparse input to the rows of the
corresponding full search."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.test_gpu_knn_offset import family

pytestmark = pytest.mark.gpu

KS = [1, 7, 15, 24, 25, 40, 64]
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def _ranges(n):
    out = [(0, 1), (n - 1, n), (37, 41), (1000, 1300), (n - 3000, n), (0, n)]
    return [(a, b) for a, b in out if 0 <= a < b <= n]


def rows_search(X, k, rb, re):
    """(idx, d2, rows searched directly) from mde_knn_rows / mde_knn16_rows, on a workspace filled with 0xA5."""
    from pymde_b200 import _lib
    lib = _lib.load()
    half = X.dtype in (torch.float16, torch.bfloat16)
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check((lib.mde_knn16_rows_ws_bytes if half else lib.mde_knn_rows_ws_bytes)(n, d, re - rb, k, C.byref(need)))
    ws = torch.full((need.value + 1024,), 0xA5, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.full((re - rb, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((re - rb, k), -7.0, dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    if half:
        code = lib.mde_knn16_rows(X.data_ptr(), _lib.DTYPE_FP16 if X.dtype == torch.float16 else _lib.DTYPE_BF16, n, d,
                                  rb, re, k, idx.data_ptr(), d2.data_ptr(), p, need.value, None, C.byref(fb))
    else:
        code = lib.mde_knn_rows(X.data_ptr(), n, d, rb, re, k, idx.data_ptr(), d2.data_ptr(), p, need.value, None,
                                C.byref(fb))
    _lib.check(code)
    torch.cuda.synchronize()
    assert 0 <= fb.value <= re - rb
    return idx, d2, fb.value


def _data(n, d=24, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((10, d), generator=g, device="cuda") * 3.0
    lab = torch.randint(0, 10, (n,), generator=g, device="cuda")
    return (c[lab] + torch.randn((n, d), generator=g, device="cuda")).contiguous()


def _check_rows(X, k, ranges):
    from pymde_b200.preprocess import data_matrix as dm
    full_i, full_d = dm.knn_device(X, k)
    for rb, re in ranges:
        i, d2, _ = rows_search(X, k, rb, re)
        assert torch.equal(i, full_i[rb:re]), (k, rb, re)
        assert torch.equal(d2, full_d[rb:re]), (k, rb, re)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("n", [130, 5000, 40000])
def test_rows_equal_the_full_search(n, dtype):
    X = _data(n).to(dtype)
    for k in KS:
        if k <= n - 1:
            _check_rows(X, k, _ranges(n))


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("name", ["off1000_d32", "far_r1000_d16", "far_r30_d8", "dup_off500", "pixels"])
def test_rows_on_offset_far_and_tied_data(name, dtype):
    X = torch.from_numpy(family(name)).cuda()
    X = X.to(dtype)  # (16-bit: coarse values far from the origin, many exact ties)
    n = X.shape[0]
    for k in (15, 40):
        _check_rows(X, k, [(0, 1), (37, 41), (1000, 1300), (n - 3000, n), (0, n)])


def test_fallback_rows_are_reported():
    from tests.test_gpu_knn_offset import search
    for k in (15, 40):
        # far-apart tight clusters: the scores cannot separate the neighbours, most rows are searched directly; the
        # full range reports what the full search's _ex entry reports
        X = torch.from_numpy(family("far_r30_d8", n=3001, seed=k)).cuda()
        _, _, fb = rows_search(X, k, 0, 3001)
        _, _, fb_full = search(X, k)
        assert fb == fb_full and fb > 0.5 * 3001, (fb, fb_full)
    X = _data(20000)
    for k in (15, 40):
        _, _, fb = rows_search(X, k, 1000, 2000)
        assert fb <= 10, fb  # ordinary data stays on the tensor cores


@pytest.mark.parametrize("k", [1, 15, 40])
@pytest.mark.parametrize("n,rb,re", [(130, 0, 130), (2000, 37, 41), (2000, 1500, 2000)])
def test_rows_agree_with_an_fp64_brute_force(n, rb, re, k):
    X = _data(n, d=16, seed=3)
    idx, d2, _ = rows_search(X, k, rb, re)
    Xd = X.double().cpu().numpy()
    D = ((Xd[rb:re, None, :] - Xd[None, :, :]) ** 2).sum(-1)
    D[np.arange(re - rb), np.arange(rb, re)] = np.inf
    order = np.argsort(D, axis=1, kind="stable")
    got = idx.long().cpu().numpy()
    np.testing.assert_allclose(d2.double().cpu().numpy(), np.take_along_axis(D, got, 1), rtol=2e-6, atol=1e-9)
    ref = np.take_along_axis(D, order[:, :k + 1], 1)
    np.testing.assert_allclose(d2.double().cpu().numpy(), ref[:, :k], rtol=2e-6, atol=1e-9)
    clear = ref[:, k] - ref[:, k - 1] > 4e-6 * ref[:, k] if k < n - 1 else np.ones(re - rb, bool)
    for r in np.nonzero(clear)[0]:
        assert set(got[r]) == set(order[r, :k])


@pytest.mark.parametrize("k", [65, 100])
def test_large_k_takes_the_gemm_rows(k):
    from pymde_b200.preprocess import data_matrix as dm
    X = _data(3000)
    full_i, full_d = dm._gemm_search(X, k)
    for rb, re in [(0, 1), (37, 41), (1000, 1300), (2999, 3000), (0, 3000)]:
        i, d2 = dm.knn_rows_device(X, k, rb, re)
        assert i.dtype == torch.int64
        assert torch.equal(i, full_i[rb:re]) and torch.equal(d2, full_d[rb:re])


@pytest.mark.parametrize("k", [15, 40, 100])
def test_sparse_input_takes_the_full_sparse_search(k):
    from pymde_b200.preprocess import data_matrix as dm
    rng = np.random.default_rng(4)
    A = sp.random(2500, 300, density=0.05, format="csr", random_state=rng, dtype=np.float32)
    full_i, full_d = dm.knn_sparse_device(*dm._to_device_csr(A, torch.device("cuda")), k)
    for rb, re in [(0, 1), (37, 41), (1000, 1300), (0, 2500)]:
        i, d2 = dm.knn_rows_device(A, k, rb, re)
        assert torch.equal(i, full_i[rb:re]) and torch.equal(d2, full_d[rb:re])


def test_dense_routes_are_always_exact(monkeypatch):
    from pymde_b200.preprocess import data_matrix as dm
    X = _data(5000)
    monkeypatch.setenv("PYMDE_B200_KNN", "approx")
    full_i, full_d = dm.knn_device(X, 15)
    i, d2 = dm.knn_rows_device(X, 15, 4000, 5000)
    assert torch.equal(i, full_i[4000:]) and torch.equal(d2, full_d[4000:])
    with pytest.raises(ValueError):
        dm.knn_rows_device(X, 15, 10, 10)
    with pytest.raises(ValueError):
        dm.knn_rows_device(X, 5000, 0, 10)
