"""16-bit data matrices (fp16, bf16) on the dense k-nearest-neighbour searches (`mde_knn16*`, csrc/mde_knn.cu and
csrc/mde_knn_approx.cu): read in place, without an fp32 copy, and with the bits the fp32 searches give on X.float(),
through the C entries, `k_nearest_neighbors`, the device graph builders and the recipes."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_gpu_knn import _compare

pytestmark = pytest.mark.gpu

HALF = [torch.float16, torch.bfloat16]
KS = [1, 15, 24, 25, 50, 64, 65, 128, 256]
SHAPES = [(n, d) for n in (2, 129, 3001) for d in (1, 7, 64, 65, 784)]


def _lib():
    from pymde_b200 import _lib as L
    return L, L.load()


def _matrix(n, d, seed, dtype, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn((n, d), generator=g, device="cuda") * scale).to(dtype)


def _exact(X, k):
    from pymde_b200.preprocess import data_matrix as dm
    return dm.knn_device(X, k)


def _assert_same_as_upcast(X, k):
    i16, d16 = _exact(X, k)
    i32, d32 = _exact(X.float(), k)
    assert torch.equal(i16, i32) and torch.equal(d16, d32)
    return i16, d16


# --- exact searches ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", HALF, ids=["fp16", "bf16"])
@pytest.mark.parametrize("n,d", SHAPES)
@pytest.mark.parametrize("k", KS)
def test_exact_search_equals_the_fp32_search_on_the_upcast(dtype, n, d, k):
    if k > n - 1:
        pytest.skip("k > n - 1")
    X = _matrix(n, d, 11 * n + d, dtype)
    _assert_same_as_upcast(X, k)


@pytest.mark.parametrize("dtype", HALF, ids=["fp16", "bf16"])
@pytest.mark.parametrize("k", [15, 50, 200])
def test_exact_search_matches_fp64_brute_force(dtype, k):
    X = _matrix(4099, 784, 5, dtype)
    idx, d2 = _exact(X, k)
    _compare(X.float(), k, idx, d2)


@pytest.mark.parametrize("dtype", HALF, ids=["fp16", "bf16"])
def test_strided_and_cpu_input_is_searched_as_its_contiguous_copy(dtype):
    from pymde_b200.preprocess import data_matrix as dm
    X = _matrix(1000, 96, 3, dtype)
    Xs = X[:, ::2]  # non-contiguous
    i1, d1 = _exact(Xs, 20)
    i2, d2 = _exact(Xs.float().contiguous(), 20)
    assert torch.equal(i1, i2) and torch.equal(d1, d2)
    i3, d3, _ = dm._search(Xs.cpu(), 20, torch.device("cuda"))
    assert torch.equal(i1, i3) and torch.equal(d1, d3)


# --- NN-descent --------------------------------------------------------------------------------------------------------

def _approx16(X, k, seed, fill):
    L, lib = _lib()
    n, d = X.shape
    need = C.c_size_t(0)
    L.check(lib.mde_knn16_approx_ws_bytes(n, d, k, C.byref(need)))
    ws = torch.full((need.value + 1024,), fill, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    it = C.c_int(-1)
    code = L.DTYPE_FP16 if X.dtype == torch.float16 else L.DTYPE_BF16
    L.check(lib.mde_knn16_approx_ex(X.data_ptr(), code, n, d, k, C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(), p,
                                    need.value, torch.cuda.current_stream().cuda_stream, C.byref(it)))
    torch.cuda.synchronize()
    return idx, d2, it.value


@pytest.mark.parametrize("dtype", HALF, ids=["fp16", "bf16"])
@pytest.mark.parametrize("k", [15, 24, 50, 64])
def test_nn_descent_equals_the_fp32_search_on_the_upcast(dtype, k):
    from pymde_b200.preprocess import data_matrix as dm
    X = _matrix(4000, 40, 100 + k, dtype)
    ref_i, ref_d = dm.knn_approx_device(X.float(), k, seed=12345)
    for fill in (0x00, 0xFF):
        i, d, it = _approx16(X, k, 12345, fill)
        assert it >= 1
        assert torch.equal(i, ref_i) and torch.equal(d, ref_d)
    i, d = dm.knn_approx_device(X, k, seed=12345)  # the Python entry takes the 16-bit route
    assert torch.equal(i, ref_i) and torch.equal(d, ref_d)


# --- routing and recipes -----------------------------------------------------------------------------------------------

def _blobs(n, d, seed):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((6, d)) * 5
    return (centers[rng.integers(0, 6, n)] + rng.standard_normal((n, d))).astype(np.float32)


SOURCES = ["fp16-cuda", "fp16-cpu", "fp16-numpy", "bf16-cuda", "bf16-cpu"]


def _inputs(source, X32):
    """(16-bit input in the given form, its fp32 upcast as a CPU tensor)."""
    t = torch.from_numpy(X32)
    if source == "fp16-numpy":
        data = X32.astype(np.float16)
        return data, torch.from_numpy(data.astype(np.float32))
    dtype = torch.float16 if source.startswith("fp16") else torch.bfloat16
    h = t.to(dtype)
    return (h.cuda() if source.endswith("cuda") else h), h.float()


@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("mode", ["kernel", "approx", "gemm"])
@pytest.mark.parametrize("k", [15, 50, 100, 300])
def test_neighbour_graphs_equal_those_of_the_upcast(monkeypatch, source, mode, k):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    if mode != "kernel":
        monkeypatch.setenv("PYMDE_B200_KNN", mode)
    data, up = _inputs(source, _blobs(1200, 12, 31))

    def both(fn):
        pm.seed(4)
        a = fn(data)
        pm.seed(4)
        return a, fn(up)

    g16, g32 = both(lambda x: dm.k_nearest_neighbors(x, k))
    assert torch.equal(g16.edges, g32.edges) and torch.equal(g16.weights, g32.weights)
    if k <= 256:
        build = dm.k_nearest_neighbors_device if k <= 64 else dm.k_nearest_neighbors_device_long
        g16, g32 = both(lambda x: build(x, k))
        assert torch.equal(g16.edges, g32.edges) and torch.equal(g16.weights, g32.weights)

    def problem(x):
        mde = pm.preserve_neighbors(x, n_neighbors=k, init="random", device="cuda")
        f = mde.distortion_function
        return mde.edges.clone(), (f.weights if hasattr(f, "weights") else f.deviations).clone()

    (e16, w16), (e32, w32) = both(problem)
    assert torch.equal(e16, e32) and torch.equal(w16, w32)


@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("max_distances", [5e7, 3e4])
def test_preserve_distances_equals_the_upcast(source, max_distances):
    import pymde_b200 as pm
    data, up = _inputs(source, _blobs(500, 20, 33))
    out = []
    for x in (data, up):
        pm.seed(6)
        mde = pm.preserve_distances(x, max_distances=max_distances, device="cuda")
        out.append((mde.edges.clone(), mde.distortion_function.deviations.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


# --- memory ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", HALF, ids=["fp16", "bf16"])
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
        L.check(lib.mde_knn16_approx_ws_bytes(n, d, k, C.byref(need)))
    else:
        L.check(lib.mde_knn16_ws_bytes(n, d, C.byref(need)))
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


# --- edge values -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,k", [(33, 24), (97, 64), (289, 256)])
def test_fp16_extremes(n, k):
    """+-65504 next to values of order 1: with n - 1 candidates per list both routes keep every row, and the re-rank
    decides on identical fp32 values."""
    X = _matrix(n, 64, n, torch.float16)
    g = torch.Generator(device="cuda").manual_seed(2 * n)
    mask = torch.rand((n, 64), generator=g, device="cuda") < 0.03
    sign = torch.where(torch.rand((n, 64), generator=g, device="cuda") < 0.5, -1.0, 1.0)
    X = torch.where(mask, (65504.0 * sign).half(), X)
    assert bool((X.abs() == 65504).any())
    _assert_same_as_upcast(X, k)


@pytest.mark.parametrize("k", [10, 50, 150])
def test_fp16_subnormals(k):
    X = _matrix(1500, 64, 9, torch.float16, scale=2.0 ** -17)
    assert float((X.float().abs() < 2.0 ** -14).float().mean()) > 0.9  # mostly subnormal fp16
    _, d2 = _assert_same_as_upcast(X, k)
    assert bool((d2 > 0).all())


@pytest.mark.parametrize("scale", [2.0 ** 56, 2.0 ** -62])
@pytest.mark.parametrize("k", [10, 50, 150])
def test_bf16_exponents_near_the_fp32_limits(scale, k):
    X = _matrix(1500, 64, 10, torch.bfloat16, scale=scale)
    _, d2 = _assert_same_as_upcast(X, k)
    assert bool(torch.isfinite(d2).all()) and bool((d2 > 0).all())


@pytest.mark.parametrize("dtype", HALF, ids=["fp16", "bf16"])
@pytest.mark.parametrize("k", [5, 40, 100])
def test_duplicate_rows(dtype, k):
    """Groups of four identical rows (three copies of each of the first 100), fewer than the spare candidates of
    every list, so both routes hold every tie."""
    base = _matrix(600, 48, 17, dtype)
    X = torch.cat([base, base[:100], base[:100], base[:100]], 0)
    idx, d2 = _assert_same_as_upcast(X, k)
    assert bool((d2[:100, :3] == 0).all())
    # the copies of row i < 100 come first, by index
    want = torch.stack([torch.arange(600, 700), torch.arange(700, 800), torch.arange(800, 900)], 1).cuda()
    assert torch.equal(idx[:100, :3].long(), want)
