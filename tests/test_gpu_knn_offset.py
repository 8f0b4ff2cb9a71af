"""The dense exact k-nearest-neighbour searches on data far from the origin and on far-apart clusters, against fp64.

Every dense exact route ranks candidates by the norm expansion ||x||^2 - 2 q.x: the tensor-core searches (`mde_knn`,
`mde_knn_wide`, `mde_knn_long` and their 16-bit entries, csrc/mde_knn.cu) with bf16 x 3 (or 16-bit) cross terms, the
GEMM path of `data_matrix._search` with library matmuls.  When ||x||^2 is large against the neighbour distances the
scores are rounding noise (tests/test_knn_offset_cpu.py reproduces this on the CPU).  The searches centre the columns,
which removes a global offset, and certify every row: a row whose kept candidates cannot be shown to contain its k
nearest rows is searched directly.  So the result must be the exact one on every family below, whatever its offset or
clustering, and the families a centred search handles must rarely need the direct search.

Reference: the fp64 column-centred norm expansion picks k + 16 candidates per row, whose exact fp64 squared distances
rank them.  Contract checked (that of tests/test_gpu_knn.py): indices in range, no self neighbour, no repeat,
ascending fp32 distances within 2e-6 of the exact ones, the exact k smallest distances, and the reference's neighbour
set wherever the k-th and (k + 1)-th neighbours are separated by more than fp32 rounding."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 4000  # a multiple of neither 64 nor 128


# --- data families ---------------------------------------------------------------------------------------------------

def _clusters(rng, n, d, radius, spread, m=10):
    centres = rng.standard_normal((m, d))
    centres *= radius / np.linalg.norm(centres, axis=1, keepdims=True)
    return centres[rng.integers(0, m, n)] + spread * rng.standard_normal((n, d))


def family(name, n=N, seed=0):
    """float32 n x d data of a named family (numpy, seeded)."""
    rng = np.random.default_rng(seed)
    if name == "iso16":
        X = rng.standard_normal((n, 16))
    elif name == "latlong":  # latitude / longitude of points in one city
        X = np.array([40.7, -74.0]) + 0.05 * rng.standard_normal((n, 2))
    elif name == "off100_d8":
        X = 100.0 + rng.standard_normal((n, 8))
    elif name == "off1000_d32":
        X = 1000.0 + rng.standard_normal((n, 32))
    elif name == "far_r1000_d16":
        X = _clusters(rng, n, 16, 1000.0, 1.0)
    elif name == "far_r30_d8":
        X = _clusters(rng, n, 8, 30.0, 0.01)
    elif name == "far_r1000_d2":
        X = _clusters(rng, n, 2, 1000.0, 1.0)
    elif name == "far_r300_d64":
        X = _clusters(rng, n, 64, 300.0, 0.3)
    elif name == "dup_off500":  # exact duplicates (d^2 = 0 ties) far from the origin
        base = 500.0 + rng.standard_normal((n - n // 8, 16))
        X = np.concatenate([base, base[: n // 8]], 0)
    elif name == "relu_shift":  # non-negative features with a common shift
        X = np.maximum(rng.standard_normal((n, 64)), 0.0) + 20.0
    elif name == "pixels":  # 0 .. 255 images: ten templates with integer noise
        t = rng.integers(0, 256, (10, 64))
        X = np.clip(t[rng.integers(0, 10, n)] + rng.integers(-12, 13, (n, 64)), 0, 255)
    else:
        raise KeyError(name)
    return np.ascontiguousarray(X, dtype=np.float32)


# families whose exact distances are continuous: near-ties at the k-th neighbour are rare
TIE_RARE = ["iso16", "latlong", "off100_d8", "off1000_d32", "far_r1000_d16", "far_r30_d8", "far_r1000_d2",
            "far_r300_d64", "relu_shift"]
TIE_HEAVY = ["dup_off500", "pixels"]
OFFSET = ["latlong", "off100_d8", "off1000_d32"]  # a global offset: centring must keep the direct search rare
FAR = ["far_r1000_d16", "far_r30_d8", "far_r1000_d2", "far_r300_d64"]  # far-apart clusters: centring does not help


# --- fp64 reference and the contract ---------------------------------------------------------------------------------

def reference(X, k):
    """(exact fp64 squared distances [n, k + 1], indices [n, k]) of the k + 1 nearest rows of every row."""
    Xd = X.double()
    Xd = Xd - Xd.mean(0)
    n = X.shape[0]
    kc = min(n - 1, k + 16)
    sq = (Xd * Xd).sum(1)
    vals, idxs = [], []
    for s0 in range(0, n, 1024):
        Q = Xd[s0:s0 + 1024]
        score = sq[None, :] - 2.0 * Q @ Xd.T
        score[torch.arange(Q.shape[0]), torch.arange(s0, s0 + Q.shape[0])] = float("inf")
        cand = torch.topk(score, kc, dim=1, largest=False)[1]
        exact = ((Q[:, None, :] - Xd[cand]) ** 2).sum(-1)
        val, pos = torch.sort(exact, dim=1, stable=True)
        vals.append(val[:, :k + 1]); idxs.append(torch.gather(cand, 1, pos[:, :k]))
    return torch.cat(vals), torch.cat(idxs)


def check(X, k, idx, d2, tie_rare=True):
    n = X.shape[0]
    val, ref = reference(X, k)
    got = idx.long()
    assert got.shape == (n, k) and d2.shape == (n, k)
    assert int(got.min()) >= 0 and int(got.max()) < n
    assert not bool((got == torch.arange(n, device=got.device)[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())  # no repeats
    gd = ((X.double()[:, None, :] - X.double()[got]) ** 2).sum(-1)
    np.testing.assert_allclose(d2.double().cpu().numpy(), gd.cpu().numpy(), rtol=2e-6, atol=1e-9)
    np.testing.assert_allclose(gd.cpu().numpy(), val[:, :k].cpu().numpy(), rtol=2e-6, atol=1e-9)
    assert bool((d2[:, 1:] >= d2[:, :-1]).all())
    if val.shape[1] > k:
        clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-9
        same = (s == torch.sort(ref, 1)[0]).all(1)
        assert bool(same[clear].all())
        if tie_rare:
            assert float(clear.float().mean()) >= 0.95
        return clear, ref
    return None, ref


# --- the raw entries -------------------------------------------------------------------------------------------------

def route_of(k):
    return "_long" if k > 64 else "_wide" if k > 24 else ""


def search(X, k, route=None, fill=0xA5):
    """(idx, d2, rows searched directly) from the `_ex` entry of `route` (default: the one k selects), on a workspace
    filled with `fill`."""
    from pymde_b200 import _lib
    lib = _lib.load()
    half = X.dtype in (torch.float16, torch.bfloat16)
    name = ("knn16" if half else "knn") + (route_of(k) if route is None else route)
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check(getattr(lib, "mde_%s_ws_bytes" % name)(n, d, C.byref(need)))
    ws = torch.full((need.value + 1024,), fill, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.full((n, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((n, k), -7.0, dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    args = (X.data_ptr(), _lib.DTYPE_FP16 if X.dtype == torch.float16 else _lib.DTYPE_BF16) if half else (X.data_ptr(),)
    _lib.check(getattr(lib, "mde_%s_ex" % name)(*args, n, d, k, idx.data_ptr(), d2.data_ptr(), p, need.value, None,
                                                 C.byref(fb)))
    torch.cuda.synchronize()
    assert 0 <= fb.value <= n
    return idx, d2, fb.value


# --- the tensor-core searches ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [15, 64, 200])
@pytest.mark.parametrize("name", TIE_RARE + TIE_HEAVY)
def test_every_family_gives_the_exact_neighbours(name, k):
    from pymde_b200.preprocess import data_matrix as dm
    X = torch.from_numpy(family(name)).cuda()
    idx, d2 = dm.knn_device(X, k)
    check(X, k, idx, d2, tie_rare=name in TIE_RARE)
    if name == "dup_off500":  # every copied row finds its copy first, at distance exactly 0
        m = N // 8
        assert bool((d2[:m, 0] == 0).all())
        assert bool((idx[:m, 0].long() == torch.arange(N - m, N, device="cuda")).all())


@pytest.mark.parametrize("k", [1, 15, 24, 25, 64, 65, 200, 256])
@pytest.mark.parametrize("name", ["latlong", "far_r1000_d16", "far_r30_d8"])
def test_every_k_of_every_route(name, k):
    X = torch.from_numpy(family(name, n=3001, seed=k)).cuda()
    idx, d2, fb = search(X, k)
    check(X, k, idx, d2)
    if name in FAR:
        assert fb > 0.5 * X.shape[0]  # the scores cannot separate the neighbours: the certificate must fail


@pytest.mark.parametrize("name", OFFSET)
@pytest.mark.parametrize("k", [15, 64, 200])
def test_centring_keeps_offset_data_on_the_tensor_cores(name, k):
    X = torch.from_numpy(family(name)).cuda()
    idx, d2, fb = search(X, k)
    check(X, k, idx, d2)
    assert fb <= 0.01 * N, fb


@pytest.mark.parametrize("route", ["", "_wide", "_long"])
@pytest.mark.parametrize("name", ["latlong", "far_r1000_d16", "dup_off500"])
def test_smallest_n(name, route):
    """n = k + 2: every row's list holds every other row (certified without the direct search)."""
    k = {"": 24, "_wide": 64, "_long": 256}[route]
    X = torch.from_numpy(family(name, n=k + 2, seed=1)).cuda()
    idx, d2, fb = search(X, k, route)
    check(X, k, idx, d2, tie_rare=False)
    assert fb == 0


@pytest.mark.parametrize("route", ["", "_wide", "_long"])
def test_lower_routes_agree_with_the_direct_search(route):
    """A k any route takes, on far clusters: every row searched directly, the same bits on every route."""
    X = torch.from_numpy(family("far_r1000_d16", n=5555, seed=5)).cuda()  # clusters larger than the long lists
    i0, d0, _ = search(X, 20, "")
    i1, d1, fb = search(X, 20, route)
    assert fb > 0 and torch.equal(i0, i1) and torch.equal(d0, d1)


# --- 16-bit input ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [15, 64, 200])
@pytest.mark.parametrize("dtype,offset", [(torch.float16, 100.0), (torch.bfloat16, 64.0)], ids=["fp16", "bf16"])
def test_16bit_offset_data_gives_the_fp32_route(dtype, offset, k):
    """The 16-bit route returns the bits of the fp32 route on X.float(), ties included (fp16 at 100 is spaced 1/16 apart,
    bf16 at 64 0.5 apart: many exact ties)."""
    rng = np.random.default_rng(11)
    X = (offset + torch.from_numpy(rng.standard_normal((N, 16)).astype(np.float32))).to(dtype).cuda()
    i16, d16, _ = search(X, k)
    i32, d32, _ = search(X.float(), k)
    assert torch.equal(i16, i32) and torch.equal(d16, d32)
    check(X.float(), k, i16, d16, tie_rare=False)


# --- the GEMM path ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("how,k", [("default", 100), ("gemm", 15), ("gemm", 300)])
@pytest.mark.parametrize("name", ["latlong", "far_r1000_d16"])
def test_gemm_path(monkeypatch, name, how, k, tf32):
    from pymde_b200.preprocess import data_matrix as dm
    if how == "gemm":
        monkeypatch.setenv("PYMDE_B200_KNN", "gemm")
    else:
        monkeypatch.delenv("PYMDE_B200_KNN", raising=False)
    X = torch.from_numpy(family(name)).cuda()
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        idx, d2, n = dm._search(family(name), k, torch.device("cuda"))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    assert idx.dtype == torch.int64 and n == N  # the GEMM path
    check(X, k, idx, d2)


# --- graph builders --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [15, 100])
def test_graph_builders_on_latlong_data(k):
    from pymde_b200 import preprocess
    from pymde_b200.preprocess import data_matrix as dm
    from pymde_b200.preprocess.graph import Graph
    data = family("latlong")
    X = torch.from_numpy(data).cuda()
    idx, d2, _ = dm._search(data, k, torch.device("cuda"))
    clear, ref = check(X, k, idx, d2)
    # the fp64 reference graph (on a row whose k-th and (k + 1)-th neighbours are within fp32 rounding, either is right)
    ref = torch.where(clear[:, None], ref, idx.long())
    e = torch.stack([torch.arange(N, device="cuda")[:, None].expand_as(ref).reshape(-1), ref.reshape(-1)], 1)
    want = Graph.from_edges(e.cpu(), None, n_items=N)
    g = preprocess.k_nearest_neighbors(data, k=k)
    np.testing.assert_array_equal(np.asarray(g.edges.cpu()), np.asarray(want.edges.cpu()))
    np.testing.assert_array_equal(np.asarray(g.weights.cpu()), np.asarray(want.weights.cpu()))
    build = dm.k_nearest_neighbors_device if k <= 64 else dm.k_nearest_neighbors_device_long
    gd = build(data, k)
    np.testing.assert_array_equal(gd.edges.cpu().numpy(), np.asarray(want.edges.cpu()))
    np.testing.assert_array_equal(gd.weights.cpu().numpy(), np.asarray(want.weights.cpu()))


# --- ordinary data ---------------------------------------------------------------------------------------------------

def _ordinary(kind):
    g = torch.Generator(device="cuda").manual_seed(17)
    if kind == "iso":
        return torch.randn((4099, 65), generator=g, device="cuda")
    X = torch.randn((4099, 784), generator=g, device="cuda")  # MNIST-shaped: clipped, many exact zeros
    return torch.where(X < 0.3, torch.zeros_like(X), X.clamp(max=1.0)).contiguous()


@pytest.mark.parametrize("k", [15, 64, 200])
@pytest.mark.parametrize("kind", ["iso", "mnist"])
def test_ordinary_data_certifies_and_repeats_bit_for_bit(kind, k):
    X = _ordinary(kind)
    idx, d2, fb = search(X, k)
    print(kind, k, "rows searched directly:", fb)
    assert fb <= 0.01 * X.shape[0], fb
    check(X, k, idx, d2)
    i2, e2, fb2 = search(X, k, fill=0x00)
    assert fb2 == fb and torch.equal(idx, i2) and torch.equal(d2, e2)


@pytest.mark.parametrize("k", [15, 64])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_16bit_ordinary_data_stays_on_the_tensor_cores(dtype, k):
    """A 16-bit matrix near the origin keeps its exact operand: its rows certify as the fp32 ones do."""
    X = _ordinary("mnist").to(dtype)
    idx, d2, fb = search(X, k)
    print(dtype, k, "rows searched directly:", fb)
    assert fb <= 0.01 * X.shape[0], fb
    i32, d32, _ = search(X.float(), k)
    assert torch.equal(idx, i32) and torch.equal(d2, d32)
