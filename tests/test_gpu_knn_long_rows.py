"""The long row-range exact search (`mde_knn_long_rows`, `mde_knn16_long_rows`, `mde_knn8_long_rows`,
csrc/mde_knn.cu) against the full long searches: row r of a search of rows [row_begin, row_end) must be row
row_begin + r of `mde_knn_long` / `mde_knn16_long` / `mde_knn8_long` bit for bit, indices and distances, ties
included -- with the candidate sweep split into slices and merged by the radix select, and without, on ranges that do
and do not start on a tile, on offset, far-clustered, tied and pixel data (the certificate and the direct search);
the fallback count of the full range equals the full search's; the rows agree with an fp64 brute force; an 8-bit
matrix is searched without an fp32 copy; and `embed_new_points` at n_neighbors = 100 takes the route for 16-bit and
8-bit stacks and keeps the GEMM rows for fp32."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_gpu_knn_offset import family

pytestmark = pytest.mark.gpu

KS = [1, 65, 100, 200, 256]
DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.uint8, torch.int8]
IDS = ["fp32", "fp16", "bf16", "u8", "s8"]


def _ranges(n):
    out = [(0, 1), (n - 1, n), (37, 41), (1000, 1300), (n - 3000, n), (0, n)]
    return sorted({(a, b) for a, b in out if 0 <= a < b <= n})


def _entry(X):
    """(name prefix, leading arguments) of X's dtype."""
    from pymde_b200 import _lib
    if X.dtype == torch.float32:
        return "mde_knn", (X.data_ptr(),)
    code = {torch.float16: _lib.DTYPE_FP16, torch.bfloat16: _lib.DTYPE_BF16, torch.uint8: _lib.DTYPE_U8,
            torch.int8: _lib.DTYPE_S8}[X.dtype]
    return ("mde_knn8" if X.dtype in (torch.uint8, torch.int8) else "mde_knn16"), (X.data_ptr(), code)


def _workspace(nbytes):
    ws = torch.full((nbytes + 1024,), 0xA5, dtype=torch.uint8, device="cuda")
    return ws, ws.data_ptr() + (-ws.data_ptr()) % 1024


def full_long(X, k):
    """(idx, d2, rows searched directly) of the full long search (`_long_ex`) on a workspace filled with 0xA5."""
    from pymde_b200 import _lib
    lib = _lib.load()
    name, args = _entry(X)
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check(getattr(lib, name + "_long_ws_bytes")(n, d, C.byref(need)))
    ws, p = _workspace(need.value)
    idx = torch.full((n, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((n, k), -7.0, dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    _lib.check(getattr(lib, name + "_long_ex")(*args, n, d, k, idx.data_ptr(), d2.data_ptr(), p, need.value, None,
                                               C.byref(fb)))
    torch.cuda.synchronize()
    assert 0 <= fb.value <= n
    return idx, d2, fb.value


def long_rows(X, k, rb, re):
    """(idx, d2, rows searched directly) of the long row search on a workspace filled with 0xA5."""
    from pymde_b200 import _lib
    lib = _lib.load()
    name, args = _entry(X)
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check(getattr(lib, name + "_long_rows_ws_bytes")(n, d, re - rb, k, C.byref(need)))
    ws, p = _workspace(need.value)
    idx = torch.full((re - rb, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((re - rb, k), -7.0, dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    _lib.check(getattr(lib, name + "_long_rows")(*args, n, d, rb, re, k, idx.data_ptr(), d2.data_ptr(), p,
                                                 need.value, None, C.byref(fb)))
    torch.cuda.synchronize()
    assert 0 <= fb.value <= re - rb
    return idx, d2, fb.value


def _to(X, dtype):
    """X (fp32) in `dtype`; an 8-bit type gets an affine quantisation of X to its range."""
    if dtype in (torch.uint8, torch.int8):
        lo, hi = X.min(), X.max()
        q = torch.round((X - lo) / (hi - lo).clamp_min(1e-30) * 255.0)
        return (q if dtype == torch.uint8 else q - 128.0).to(dtype).contiguous()
    return X.to(dtype).contiguous()


def _data(n, d=24, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((10, d), generator=g, device="cuda") * 3.0
    lab = torch.randint(0, 10, (n,), generator=g, device="cuda")
    return (c[lab] + torch.randn((n, d), generator=g, device="cuda")).contiguous()


def _check_rows(X, k, ranges):
    full_i, full_d, _ = full_long(X, k)
    for rb, re in ranges:
        i, d2, _ = long_rows(X, k, rb, re)
        assert torch.equal(i, full_i[rb:re]), (k, rb, re)
        assert torch.equal(d2, full_d[rb:re]), (k, rb, re)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("n", [130, 5000, 40000])
def test_rows_equal_the_full_long_search(n, dtype):
    from pymde_b200 import _lib
    lib = _lib.load()
    X = _to(_data(n), dtype)
    ranges = _ranges(n)
    # both sides of the split: S > 1 on the short ranges, S = 1 once the query tiles fill the SMs
    slices = {lib.mde_dbg_knn_long_slices(n, re - rb, 100) for rb, re in ranges}
    assert max(slices) > 1 and (n < 132 * 64 or min(slices) == 1)
    for k in KS:
        if k <= n - 1:
            _check_rows(X, k, ranges)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", ["off1000_d32", "far_r1000_d16", "far_r30_d8", "dup_off500", "pixels"])
def test_rows_on_offset_far_tied_and_pixel_data(name, dtype):
    X = _to(torch.from_numpy(family(name)).cuda(), dtype)
    n = X.shape[0]
    for k in (65, 150):
        _check_rows(X, k, [(0, 1), (37, 41), (1000, 1300), (n - 3000, n), (0, n)])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.uint8], ids=["fp32", "fp16", "u8"])
def test_fallback_rows_are_reported(dtype):
    from pymde_b200 import _lib
    for k in (65, 150):
        # far-apart tight clusters: the scores cannot separate the neighbours, many rows are searched directly; the
        # full range (split into S = 2 slices at n = 3 001) reports what the full search's _ex entry reports
        X = _to(torch.from_numpy(family("far_r30_d8", n=3001, seed=k)).cuda(), dtype)
        assert _lib.load().mde_dbg_knn_long_slices(3001, 3001, k) == 2
        _, _, fb = long_rows(X, k, 0, 3001)
        _, _, fb_full = full_long(X, k)
        assert fb == fb_full, (fb, fb_full)
    X = _to(_data(20000), dtype)
    for k in (65, 150):
        _, _, fb = long_rows(X, k, 1000, 2000)
        assert fb <= 10, fb  # ordinary data stays on the tensor cores


@pytest.mark.parametrize("k", [65, 128, 256])
@pytest.mark.parametrize("n,rb,re", [(300, 0, 300), (2000, 37, 41), (2000, 1500, 2000)])
def test_rows_agree_with_an_fp64_brute_force(n, rb, re, k):
    X = _data(n, d=16, seed=3)
    idx, d2, _ = long_rows(X, k, rb, re)
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


def test_8bit_input_is_searched_without_an_fp32_copy():
    from pymde_b200.preprocess import data_matrix as dm
    n, d = 200000, 256
    X = _to(_data(n, d=d, seed=5), torch.uint8)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    idx, d2 = dm.knn_rows_device_long(X, 100, n - 1000, n)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - before
    assert idx.dtype == torch.int32 and idx.shape == (1000, 100)
    assert peak < n * d * 4, (peak, n * d * 4)
    i2, dd2, _ = long_rows(X, 100, n - 1000, n)
    assert torch.equal(idx, i2) and torch.equal(d2, dd2)


def test_wrapper_routes():
    from pymde_b200.preprocess import data_matrix as dm
    import scipy.sparse as sp
    X = _data(3000)
    # a float64 matrix is searched in fp32, a numpy matrix is uploaded
    i, d2 = dm.knn_rows_device_long(X.double(), 100, 37, 41)
    fi, fd, _ = full_long(X, 100)
    assert i.dtype == torch.int32 and torch.equal(i, fi[37:41]) and torch.equal(d2, fd[37:41])
    i, d2 = dm.knn_rows_device_long(X.cpu().numpy(), 100, 37, 41)
    assert torch.equal(i, fi[37:41]) and torch.equal(d2, fd[37:41])
    # scipy.sparse: the sparse row search
    A = sp.random(2000, 300, density=0.05, format="csr", random_state=0, dtype=np.float32)
    i, d2 = dm.knn_rows_device_long(A, 100, 100, 300)
    si, sd = dm.knn_sparse_rows_device(*dm._to_device_csr(A, torch.device("cuda")), 100, 100, 300)
    assert torch.equal(i, si) and torch.equal(d2, sd)


# --- embed_new_points at n_neighbors = 100 -------------------------------------------------------------------------

N_OLD, N_NEW, D = 20000, 2000, 32
FLOOR = 0.97  # tests/test_gpu_new_points.py


@pytest.fixture(scope="module")
def fitted():
    import pymde_b200 as pm
    from tests.test_gpu_new_points import _blobs
    data, lab = _blobs(N_OLD, 1)
    new, new_lab = _blobs(N_NEW, 2)
    pm.seed(0)
    emb = pm.preserve_neighbors(data).embed()
    return data, lab, new, new_lab, emb


def _u8(x):
    return np.clip(np.round(x * 16.0 + 128.0), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("kind", ["fp32", "u8"])
def test_embed_new_points_at_100_neighbours(fitted, kind, monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    from pymde_b200.preprocess import data_matrix as dm
    from tests.test_gpu_new_points import _accuracy
    data, lab, new, new_lab, emb = fitted
    if kind == "u8":
        data, new = _u8(data), _u8(new)
    stacked = recipes._stacked_matrix(data, new, torch.device("cuda"))
    assert stacked.dtype == (torch.uint8 if kind == "u8" else torch.float32)

    def refuse(*a, **kw):
        raise AssertionError("the other route was called")
    if kind == "u8":
        # the search lists: the rows of the full long search, from the long row search and not the GEMM rows
        fi, fd, _ = full_long(stacked, 100)
        monkeypatch.setattr(dm, "knn_rows_device", refuse)
        i, d2 = recipes._dense_new_lists(stacked, 100, N_OLD, N_OLD + N_NEW)
        assert torch.equal(i, fi[N_OLD:]) and torch.equal(d2, fd[N_OLD:])
    else:
        # fp32 keeps the GEMM rows, which measured faster on it (DESIGN section 11.8)
        gi, gd = dm.knn_rows_device(stacked, 100, N_OLD, N_OLD + N_NEW)
        monkeypatch.setattr(dm, "knn_rows_device_long", refuse)
        i, d2 = recipes._dense_new_lists(stacked, 100, N_OLD, N_OLD + N_NEW)
        assert torch.equal(i, gi) and torch.equal(d2, gd)
    pm.seed(0)
    out = pm.embed_new_points(data, emb, new, n_neighbors=100)
    assert out.shape == (N_NEW, 2) and bool(torch.isfinite(out).all())
    acc = _accuracy(emb, lab, out, new_lab)
    print("accuracy at n_neighbors = 100 (%s): %.4f" % (kind, acc))
    assert acc >= FLOOR, acc
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    pm.seed(0)
    a = pm.embed_new_points(data, emb, new, n_neighbors=100)
    pm.seed(0)
    b = pm.embed_new_points(data, emb, new, n_neighbors=100)
    assert torch.equal(a, b)


def test_16bit_stacks_take_the_long_row_search(monkeypatch):
    from pymde_b200 import recipes
    from pymde_b200.preprocess import data_matrix as dm

    def refuse(*a, **kw):
        raise AssertionError("the GEMM rows were called")
    monkeypatch.setattr(dm, "knn_rows_device", refuse)
    for dtype in (torch.float16, torch.bfloat16, torch.int8):
        X = _to(_data(5000), dtype)
        fi, fd, _ = full_long(X, 150)
        i, d2 = recipes._dense_new_lists(X, 150, 4000, 5000)
        assert torch.equal(i, fi[4000:]) and torch.equal(d2, fd[4000:])
