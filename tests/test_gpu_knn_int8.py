"""8-bit data matrices (uint8, int8) on the dense k-nearest-neighbour searches (`mde_knn8*`, csrc/mde_knn.cu and
csrc/mde_knn_approx.cu): read in place, without an fp32 copy, ranked by exact integer scores on the tensor cores, and
with the bits the fp32 searches give on X.float(), through the C entries, `k_nearest_neighbors`, the device graph
builders, `embed_new_points` and the recipes."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EIGHT = [torch.uint8, torch.int8]
IDS = ["u8", "s8"]
KS = [1, 5, 24, 25, 64, 65, 256]
SHAPES = [(n, d) for n in (2, 129, 1000, 4097) for d in (1, 100, 128, 129, 784)]


def _lib():
    from pymde_b200 import _lib as L
    return L, L.load()


def _code(dtype):
    L, _ = _lib()
    return L.DTYPE_U8 if dtype == torch.uint8 else L.DTYPE_S8


def _range(dtype):
    return (0, 256) if dtype == torch.uint8 else (-128, 128)


def _matrix(n, d, seed, dtype, kind="full"):
    """Full-range values, or genotype-like ones (0 / 1 / 2, mostly 0: many exact ties), on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "geno":
        p = torch.rand((n, d), generator=g, device="cuda")
        X = (p > 0.7).to(torch.int32) + (p > 0.93).to(torch.int32)
        return X.to(dtype)
    lo, hi = _range(dtype)
    return torch.randint(lo, hi, (n, d), generator=g, device="cuda").to(dtype)


def _exact(X, k):
    from pymde_b200.preprocess import data_matrix as dm
    return dm.knn_device(X, k)


def _assert_same_as_upcast(X, k):
    i8, d8 = _exact(X, k)
    i32, d32 = _exact(X.float(), k)
    assert torch.equal(i8, i32) and torch.equal(d8, d32)
    return i8, d8


# --- exact searches ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("n,d", SHAPES)
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("kind", ["full", "geno"])
def test_exact_search_equals_the_fp32_search_on_the_upcast(dtype, n, d, k, kind):
    """The narrow (k <= 24), wide (<= 64) and long (<= 256) kernels, across tile and K-block edges."""
    k = min(k, n - 1)
    X = _matrix(n, d, 13 * n + d, dtype, kind)
    _assert_same_as_upcast(X, k)


def _brute_int64(X, k):
    """(indices, squared distances) in int64 numpy: ascending by (distance, index), the row itself excluded."""
    A = X.cpu().numpy().astype(np.int64)
    n = A.shape[0]
    sq = (A * A).sum(1)
    D = sq[:, None] + sq[None, :] - 2 * (A @ A.T)
    D[np.arange(n), np.arange(n)] = np.iinfo(np.int64).max
    order = np.lexsort((np.broadcast_to(np.arange(n), (n, n)), D), axis=1)[:, :k]
    return order, np.take_along_axis(D, order, 1)


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("d", [16, 100, 258])
@pytest.mark.parametrize("k", [10, 50, 200])
@pytest.mark.parametrize("kind", ["full", "geno"])
def test_exact_search_matches_int64_brute_force(dtype, d, k, kind):
    """d * 255^2 <= 2^24: the fp32 re-rank is exact, so the order is the exact one, ties broken by index."""
    X = _matrix(1500, d, 7 * d + k, dtype, kind)
    idx, d2 = _exact(X, k)
    ref_i, ref_d = _brute_int64(X, k)
    assert np.array_equal(idx.cpu().numpy().astype(np.int64), ref_i)
    assert np.array_equal(d2.cpu().numpy().astype(np.int64), ref_d)
    assert np.array_equal(d2.cpu().numpy(), ref_d.astype(np.float32))


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
def test_strided_and_cpu_input_is_searched_as_its_contiguous_copy(dtype):
    from pymde_b200.preprocess import data_matrix as dm
    X = _matrix(1000, 96, 3, dtype)
    Xs = X[:, ::2]  # non-contiguous
    i1, d1 = _exact(Xs, 20)
    i2, d2 = _exact(Xs.float().contiguous(), 20)
    assert torch.equal(i1, i2) and torch.equal(d1, d2)
    i3, d3, _ = dm._search(Xs.cpu(), 20, torch.device("cuda"))
    assert torch.equal(i1, i3) and torch.equal(d1, d3)
    i4, d4, _ = dm._search(Xs.cpu().numpy(), 20, torch.device("cuda"))
    assert torch.equal(i1, i4) and torch.equal(d1, d4)


# --- edge values -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("k", [5, 40, 150])
def test_extreme_zero_duplicate_rows_and_constant_columns(dtype, k):
    lo, hi = _range(dtype)
    X = _matrix(900, 130, 21 + k, dtype)
    X[:, 7] = hi - 1                      # constant columns
    X[:, 64] = lo
    X[10:14] = hi - 1                     # all-255 / all-127 rows
    X[20:24] = lo                         # all-0 / all-(-128) rows
    X[30:34] = 0                          # zero rows
    X[100:103] = X[99]                    # duplicates of row 99
    X[500:600] = X[400:500]               # 100 duplicated rows
    i, d2 = _assert_same_as_upcast(X, k)
    assert bool((d2[10, :3] == 0).all()) and bool((d2[99, :3] == 0).all())
    assert torch.equal(i[99, :3].long(), torch.tensor([100, 101, 102], device="cuda"))


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("k", [5, 40, 150])
def test_one_far_outlier_row(dtype, k):
    lo, hi = _range(dtype)
    X = _matrix(1200, 200, 5 + k, dtype, "geno")
    X[777] = hi - 1 if dtype == torch.uint8 else lo
    _assert_same_as_upcast(X, k)


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("k", [5, 30])
def test_d_max_and_one_column_more(dtype, k):
    """d = d_max takes the 8-bit route, d_max + 1 the fp32 route on X.float(): the same bits either way."""
    L, lib = _lib()
    d_max = lib.mde_knn8_max_d(_code(dtype))
    for d, n in ((d_max, 260), (d_max + 1, 260)):
        X = _matrix(n, d, d + k, dtype)
        _assert_same_as_upcast(X, k)
        entry = "mde_knn8" if k <= lib.mde_knn_max_k() else "mde_knn8_wide"
        need = C.c_size_t(0)
        L.check(getattr(lib, entry + "_ws_bytes")(n, d, C.byref(need)))
        ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
        out_i = torch.empty((n, k), dtype=torch.int32, device="cuda")
        out_d = torch.empty((n, k), dtype=torch.float32, device="cuda")
        fb = C.c_int(-1)
        code = getattr(lib, entry + "_ex")(X.data_ptr(), _code(dtype), n, d, k, out_i.data_ptr(), out_d.data_ptr(),
                                           ws.data_ptr() + (-ws.data_ptr()) % 1024, need.value,
                                           torch.cuda.current_stream().cuda_stream, C.byref(fb))
        if d > d_max:
            assert code == L.MDE_E_UNSUPPORTED and fb.value == -1
        else:
            assert code == 0 and 0 <= fb.value <= n
            i32, d32 = _exact(X.float(), k)
            assert torch.equal(out_i, i32) and torch.equal(out_d, d32)


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("entry,k", [("knn8", 15), ("knn8_wide", 50), ("knn8_long", 200)])
def test_fallback_rows_are_reported(dtype, entry, k):
    """The _ex entries count the rows the certificate sends to the direct search, with the bits of the fp32 route."""
    L, lib = _lib()
    n, d = 3000, 784
    X = _matrix(n, d, 9, dtype)
    need = C.c_size_t(0)
    L.check(getattr(lib, "mde_%s_ws_bytes" % entry)(n, d, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    out_i = torch.empty((n, k), dtype=torch.int32, device="cuda")
    out_d = torch.empty((n, k), dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    L.check(getattr(lib, "mde_%s_ex" % entry)(X.data_ptr(), _code(dtype), n, d, k, out_i.data_ptr(),
                                              out_d.data_ptr(), ws.data_ptr() + (-ws.data_ptr()) % 1024, need.value,
                                              torch.cuda.current_stream().cuda_stream, C.byref(fb)))
    assert 0 <= fb.value <= n
    i32, d32 = _exact(X.float(), k)
    assert torch.equal(out_i, i32) and torch.equal(out_d, d32)


# --- rows --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("k", [1, 15, 24, 25, 64])
@pytest.mark.parametrize("lo,hi", [(0, 1), (0, 4097), (1000, 1300), (4000, 4097), (129, 130)])
def test_rows_equal_the_rows_of_the_full_search(dtype, k, lo, hi):
    from pymde_b200.preprocess import data_matrix as dm
    X = _matrix(4097, 100, 3 * k + lo, dtype)
    full_i, full_d = _exact(X, k)
    i, d2 = dm.knn_rows_device(X, k, lo, hi)
    assert torch.equal(i, full_i[lo:hi]) and torch.equal(d2, full_d[lo:hi])
    i32, d32 = dm.knn_rows_device(X.float(), k, lo, hi)
    assert torch.equal(i, i32) and torch.equal(d2, d32)


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("source", ["cuda", "numpy"])
def test_embed_new_points_on_an_8_bit_pair_equals_the_float_pair(monkeypatch, dtype, source):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    X = _matrix(2300, 64, 77, dtype, "geno")
    data, new = X[:2000], X[2000:]
    if source == "numpy":
        data, new = data.cpu().numpy(), new.cpu().numpy()
    emb = torch.randn((2000, 2), generator=torch.Generator().manual_seed(1)).cuda()
    stacked = recipes._stacked_matrix(data, new, torch.device("cuda"))
    assert stacked.dtype == dtype
    fd, fn = X[:2000].float(), X[2000:].float()
    pm.seed(3)
    p8, it8 = recipes._new_points_mde(data, emb, new)
    pm.seed(3)
    p32, it32 = recipes._new_points_mde(fd, emb, fn)
    assert torch.equal(it8, it32) and torch.equal(p8.edges, p32.edges)
    f8, f32 = p8.distortion_function, p32.distortion_function
    assert torch.equal(f8.weights, f32.weights)
    pm.seed(4)
    a = pm.embed_new_points(data, emb, new)
    pm.seed(4)
    b = pm.embed_new_points(fd, emb, fn)
    assert torch.equal(a, b)


# --- NN-descent --------------------------------------------------------------------------------------------------------

def _approx8(X, k, seed, fill):
    L, lib = _lib()
    n, d = X.shape
    need = C.c_size_t(0)
    L.check(lib.mde_knn8_approx_ws_bytes(n, d, k, C.byref(need)))
    ws = torch.full((need.value + 1024,), fill, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    it = C.c_int(-1)
    L.check(lib.mde_knn8_approx_ex(X.data_ptr(), _code(X.dtype), n, d, k, C.c_uint64(seed), idx.data_ptr(),
                                   d2.data_ptr(), p, need.value, torch.cuda.current_stream().cuda_stream, C.byref(it)))
    torch.cuda.synchronize()
    return idx, d2, it.value


@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("k", [15, 24, 50, 64])
@pytest.mark.parametrize("kind", ["full", "geno"])
def test_nn_descent_equals_the_fp32_search_on_the_upcast(dtype, k, kind):
    from pymde_b200.preprocess import data_matrix as dm
    X = _matrix(4000, 40, 100 + k, dtype, kind)
    ref_i, ref_d = dm.knn_approx_device(X.float(), k, seed=12345)
    for fill in (0x00, 0xFF):
        i, d, it = _approx8(X, k, 12345, fill)
        assert it >= 1
        assert torch.equal(i, ref_i) and torch.equal(d, ref_d)
    i, d = dm.knn_approx_device(X, k, seed=12345)  # the Python entry takes the 8-bit route
    assert torch.equal(i, ref_i) and torch.equal(d, ref_d)


# --- routing and recipes -----------------------------------------------------------------------------------------------

def _pixels(n, d, seed):
    """MNIST-like uint8 pixels: cluster templates, noise, many exact zeros."""
    rng = np.random.default_rng(seed)
    centers = rng.random((6, d)) * 255
    X = centers[rng.integers(0, 6, n)] + rng.normal(0, 40, (n, d))
    X[X < 60] = 0
    return np.clip(X, 0, 255).astype(np.uint8)


SOURCES = ["u8-cuda", "u8-cpu", "u8-numpy", "s8-cuda", "s8-cpu", "s8-numpy"]


def _inputs(source, pixels):
    """(8-bit input in the given form, its fp32 upcast as a CPU tensor)."""
    A = pixels if source.startswith("u8") else (pixels.astype(np.int16) - 128).astype(np.int8)
    if source.endswith("numpy"):
        return A, torch.from_numpy(A.astype(np.float32))
    t = torch.from_numpy(A)
    return (t.cuda() if source.endswith("cuda") else t), t.float()


@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("mode", ["kernel", "approx", "gemm"])
@pytest.mark.parametrize("k", [15, 50, 100, 300])
def test_neighbour_graphs_equal_those_of_the_upcast(monkeypatch, source, mode, k):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    if mode != "kernel":
        monkeypatch.setenv("PYMDE_B200_KNN", mode)
    data, up = _inputs(source, _pixels(1200, 48, 31))

    def both(fn):
        pm.seed(4)
        a = fn(data)
        pm.seed(4)
        return a, fn(up)

    g8, g32 = both(lambda x: dm.k_nearest_neighbors(x, k))
    assert torch.equal(g8.edges, g32.edges) and torch.equal(g8.weights, g32.weights)
    if k <= 256:
        build = dm.k_nearest_neighbors_device if k <= 64 else dm.k_nearest_neighbors_device_long
        g8, g32 = both(lambda x: build(x, k))
        assert torch.equal(g8.edges, g32.edges) and torch.equal(g8.weights, g32.weights)

    def problem(x):
        mde = pm.preserve_neighbors(x, n_neighbors=k, init="random", device="cuda")
        f = mde.distortion_function
        return mde.edges.clone(), (f.weights if hasattr(f, "weights") else f.deviations).clone()

    (e8, w8), (e32, w32) = both(problem)
    assert torch.equal(e8, e32) and torch.equal(w8, w32)


@pytest.mark.parametrize("source", ["u8-cuda", "u8-numpy", "s8-cpu"])
@pytest.mark.parametrize("mode", ["kernel", "approx", "gemm"])
def test_laplacian_embedding_equals_that_of_the_upcast(monkeypatch, source, mode):
    import pymde_b200 as pm
    if mode != "kernel":
        monkeypatch.setenv("PYMDE_B200_KNN", mode)
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    data, up = _inputs(source, _pixels(900, 32, 41))
    out = []
    for x in (data, up):
        pm.seed(8)
        mde = pm.laplacian_embedding(x, n_neighbors=10, device="cuda")
        f = mde.distortion_function
        w = f.weights if hasattr(f, "weights") else f.deviations
        out.append((mde.edges.clone(), w.clone(), mde._X_init.clone(), mde.embed(max_iter=20).clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("max_distances", [5e7, 3e4])
def test_preserve_distances_equals_the_upcast(source, max_distances):
    import pymde_b200 as pm
    data, up = _inputs(source, _pixels(500, 20, 33))
    out = []
    for x in (data, up):
        pm.seed(6)
        mde = pm.preserve_distances(x, max_distances=max_distances, device="cuda")
        out.append((mde.edges.clone(), mde.distortion_function.deviations.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


# --- memory ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", EIGHT, ids=IDS)
@pytest.mark.parametrize("mode", ["kernel", "approx"])
def test_search_allocates_no_fp32_copy(monkeypatch, dtype, mode):
    from pymde_b200.preprocess import data_matrix as dm
    L, lib = _lib()
    n, d, k = 50_000, 768, 15
    if mode == "approx":
        monkeypatch.setenv("PYMDE_B200_KNN", "approx")
    X = _matrix(n, d, 1, dtype)
    need = C.c_size_t(0)
    if mode == "approx":
        L.check(lib.mde_knn8_approx_ws_bytes(n, d, k, C.byref(need)))
    else:
        L.check(lib.mde_knn8_ws_bytes(n, d, C.byref(need)))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx, d2, _ = dm._search(X, k, torch.device("cuda"))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    outputs = idx.numel() * 4 + d2.numel() * 4
    assert idx.dtype == torch.int32 and idx.shape == (n, k)
    assert peak <= need.value + outputs + (1 << 20), (peak, need.value, outputs)
    assert peak < need.value + outputs + 4 * n * d  # (an fp32 copy of X alone would exceed this)
