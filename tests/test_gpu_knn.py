"""Row f3: the wgmma k-nearest-neighbour kernel (`mde_knn`, csrc/mde_knn.cu) against an fp64 brute force.

The reference's neighbour search (pymde/preprocess/data_matrix.py:91-178) delegates to scikit-learn / pynndescent;
its contract is "the k nearest rows in Euclidean distance", which is what is checked here: identical neighbour sets
(up to exact ties), ascending order, exact fp32 squared distances, no self neighbours."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _brute64(X, k):
    """Exact fp64 search: candidates from the fp64 norm expansion (k + 9 of them), then sum (q - x)^2 in fp64.
    Returns the k + 1 smallest squared distances (the extra one measures the gap behind the k-th) and the indices."""
    Xd = X.double()
    n = X.shape[0]
    kk = min(n - 1, k + 9)
    sq = (Xd * Xd).sum(1)
    d2 = sq[:, None] + sq[None, :] - 2.0 * Xd @ Xd.T
    d2.fill_diagonal_(float("inf"))
    cand = torch.topk(d2, kk, dim=1, largest=False)[1]
    exact = torch.empty((n, kk), dtype=torch.float64, device=X.device)
    for s0 in range(0, n, 256):
        exact[s0:s0 + 256] = ((Xd[s0:s0 + 256, None, :] - Xd[cand[s0:s0 + 256]]) ** 2).sum(-1)
    val, pos = torch.sort(exact, dim=1)
    idx = torch.gather(cand, 1, pos)
    k1 = min(kk, k + 1)
    return val[:, :k1], idx[:, :k]


def _compare(X, k, idx, d2):
    n = X.shape[0]
    val, ref = _brute64(X, k)
    got = idx.long()
    assert int(got.min()) >= 0 and int(got.max()) < n
    assert not bool((got == torch.arange(n, device="cuda")[:, None]).any())
    assert bool((torch.sort(got, 1)[0][:, 1:] != torch.sort(got, 1)[0][:, :-1]).all())  # no repeats
    gd = ((X.double()[:, None, :] - X.double()[got]) ** 2).sum(-1)
    # distances of the returned neighbours = the k smallest exact distances, to fp32 rounding of the re-rank (a pair
    # closer than that may come out in either order), in ascending order of the fp32 values
    np.testing.assert_allclose(gd.cpu().numpy(), val[:, :k].cpu().numpy(), rtol=2e-6, atol=1e-9)
    np.testing.assert_allclose(d2.double().cpu().numpy(), gd.cpu().numpy(), rtol=2e-6, atol=1e-9)
    assert bool((d2[:, 1:] >= d2[:, :-1]).all())
    # identical SETS wherever the k-th neighbour is separated from the (k+1)-th by more than fp32 rounding
    if val.shape[1] > k:
        clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-9
        same = (torch.sort(got, 1)[0] == torch.sort(ref, 1)[0]).all(1)
        assert bool(same[clear].all()) and float(clear.float().mean()) > 0.9


@pytest.mark.parametrize("n,d,k", [(2, 3, 1), (33, 7, 5), (129, 64, 8), (1000, 65, 24), (2500, 200, 15), (4099, 784, 15)])
def test_knn_kernel_matches_fp64_brute_force(n, d, k):
    from pymde_b200.preprocess import data_matrix as dm
    g = torch.Generator(device="cuda").manual_seed(n + d)
    X = torch.randn((n, d), generator=g, device="cuda")
    if d == 784:  # MNIST-like: clipped, many exact zeros
        X = torch.where(X < 0.3, torch.zeros_like(X), X.clamp(max=1.0)).contiguous()
    idx, d2 = dm.knn_device(X, k)
    _compare(X, k, idx, d2)


def test_knn_kernel_duplicates_and_far_offsets():
    """Duplicated rows (zero distances, exact ties) and data far from the origin (||x||^2 >> distances: the regime
    where the norm expansion loses digits and the exact re-rank has to restore them)."""
    from pymde_b200.preprocess import data_matrix as dm
    g = torch.Generator(device="cuda").manual_seed(7)
    base = torch.randn((700, 48), generator=g, device="cuda")
    X = torch.cat([base, base[:100]], 0) + 30.0
    k = 6
    idx, d2 = dm.knn_device(X, k)
    _compare(X, k, idx, d2)
    # every duplicated row finds its copy first, at distance exactly 0
    assert bool((d2[:100, 0] == 0).all()) and bool((idx[:100, 0].long() == torch.arange(700, 800, device="cuda")).all())


def test_k_nearest_neighbors_graph_uses_the_kernel_and_matches_gemm_path(monkeypatch):
    from pymde_b200 import preprocess
    rng = np.random.default_rng(3)
    X = rng.standard_normal((1500, 32)).astype(np.float32)
    g1 = preprocess.k_nearest_neighbors(X, k=7)
    monkeypatch.setenv("PYMDE_B200_KNN", "gemm")
    g2 = preprocess.k_nearest_neighbors(X, k=7)
    assert g1.n_items == g2.n_items == 1500
    e1 = np.asarray(g1.edges.cpu()); e2 = np.asarray(g2.edges.cpu())
    assert e1.shape == e2.shape and (e1 == e2).all()
    np.testing.assert_array_equal(np.asarray(g1.distances.cpu()), np.asarray(g2.distances.cpu()))


def test_knn_rejects_bad_arguments():
    import ctypes as C
    from pymde_b200 import _lib
    lib = _lib.load()
    assert lib.mde_knn_max_k() == 24
    X = torch.randn((10, 4), device="cuda")
    out_i = torch.empty((10, 25), dtype=torch.int32, device="cuda")
    out_d = torch.empty((10, 25), dtype=torch.float32, device="cuda")
    need = C.c_size_t(0)
    assert lib.mde_knn_ws_bytes(10, 4, C.byref(need)) == 0 and need.value > 0
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    assert lib.mde_knn(X.data_ptr(), 10, 4, 25, out_i.data_ptr(), out_d.data_ptr(), p, need.value, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn(X.data_ptr(), 10, 4, 9, out_i.data_ptr(), out_d.data_ptr(), p, need.value - 1, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn(X.data_ptr(), 10, 4, 10, out_i.data_ptr(), out_d.data_ptr(), p, need.value, None) == _lib.MDE_E_INVALID
