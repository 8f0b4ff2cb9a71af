"""Row f3, approximate: NN-descent k-nearest neighbours (`mde_knn_approx`, csrc/mde_knn_approx.cu).

Contract: k distinct rows per row, never the row itself, ascending by (squared distance, index), with the exact fp32
distances of the re-rank of `mde_knn` / `mde_knn_wide`; bit-identical results for the same (X, k, seed), whatever the
workspace held; recall against the exact search on low-intrinsic-dimension data; opt-in routing through
PYMDE_B200_KNN=approx."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_gpu_knn import _compare

pytestmark = pytest.mark.gpu


def _mixture(n, d, intrinsic, seed, clusters=50):
    """Gaussian mixture in `intrinsic` dimensions, embedded in d by a random orthonormal map, plus isotropic noise of
    1e-2 of the cluster spread."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = 4.0 * torch.randn((clusters, intrinsic), generator=g, device="cuda")
    lab = torch.randint(0, clusters, (n,), generator=g, device="cuda")
    Z = centres[lab] + torch.randn((n, intrinsic), generator=g, device="cuda")
    Q, _ = torch.linalg.qr(torch.randn((d, intrinsic), generator=g, device="cuda"))
    return (Z @ Q.T + 1e-2 * torch.randn((n, d), generator=g, device="cuda")).contiguous()


def _approx(X, k, seed=1, fill=None):
    from pymde_b200 import _lib
    lib = _lib.load()
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_approx_ws_bytes(n, d, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    if fill is not None:
        ws.fill_(fill)
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    _lib.check(lib.mde_knn_approx(X.data_ptr(), n, d, k, C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(), p,
                                  need.value, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return idx, d2


def _check_contract(X, k, idx, d2):
    n = X.shape[0]
    got = idx.long()
    assert int(got.min()) >= 0 and int(got.max()) < n
    assert not bool((got == torch.arange(n, device="cuda")[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())
    # ascending by (d2, index)
    asc = (d2[:, 1:] > d2[:, :-1]) | ((d2[:, 1:] == d2[:, :-1]) & (got[:, 1:] > got[:, :-1]))
    assert bool(asc.all())
    Xd = X.double()
    for s0 in range(0, n, 2048):
        gd = ((Xd[s0:s0 + 2048, None, :] - Xd[got[s0:s0 + 2048]]) ** 2).sum(-1)
        np.testing.assert_allclose(d2[s0:s0 + 2048].double().cpu().numpy(), gd.cpu().numpy(), rtol=2e-6, atol=1e-9)


@pytest.mark.parametrize("n,d,k", [(2, 3, 1), (33, 1, 5), (1000, 7, 24), (4099, 65, 64), (20000, 784, 15)])
def test_output_contract_on_awkward_shapes(n, d, k):
    g = torch.Generator(device="cuda").manual_seed(n + d)
    X = torch.randn((n, d), generator=g, device="cuda")  # isotropic: NN-descent's weak case, contract only
    idx, d2 = _approx(X, k)
    _check_contract(X, k, idx, d2)


@pytest.mark.parametrize("n,d,k", [(2, 3, 1), (20, 5, 7), (33, 40, 24), (30, 784, 15), (60, 16, 30), (97, 33, 64)])
def test_exact_when_the_lists_hold_every_row(n, d, k):
    """n - 1 <= 32 (k <= 24) or n - 1 <= 96 (k > 24): every list holds every other row, so the result is the exact
    search's, bit for bit (random data: no exact ties)."""
    from pymde_b200.preprocess import data_matrix as dm
    g = torch.Generator(device="cuda").manual_seed(3 * n + k)
    X = torch.randn((n, d), generator=g, device="cuda")
    idx, d2 = _approx(X, k)
    ri, rd = dm.knn_device(X, k)
    assert torch.equal(idx, ri)
    assert torch.equal(d2.view(torch.int32), rd.view(torch.int32))
    _compare(X, k, idx, d2)


def _recall_checks(idx, d2, ri, rd, floor=0.97):
    k = idx.shape[1]
    a = torch.sort(idx.long(), 1)[0]
    b = torch.sort(ri.long(), 1)[0]
    hits = (a[:, :, None] == b[:, None, :]).any(2).float().sum(1)
    recall = float(hits.mean()) / k
    assert recall >= floor, recall
    # an approximate list never beats the true j-th distance
    assert bool((d2 >= rd).all())
    # rows whose set is the exact set carry the exact search's bits
    same = (a == b).all(1)
    assert bool(torch.equal(d2[same].view(torch.int32), rd[same].view(torch.int32)))
    return recall


@pytest.fixture(scope="module")
def mixture():
    return _mixture(200000, 64, 8, seed=11)


@pytest.mark.parametrize("k", [15, 24, 50])
def test_recall_on_a_low_dimensional_mixture(mixture, k):
    from pymde_b200.preprocess import data_matrix as dm
    X = mixture
    idx, d2 = _approx(X, k, seed=5)
    ri, rd = dm.knn_device(X, k)  # mde_knn for k <= 24, mde_knn_wide for k = 50
    _check_contract(X, k, idx, d2)
    _recall_checks(idx, d2, ri, rd)


def test_determinism_seed_and_workspace(mixture):
    from pymde_b200.preprocess import data_matrix as dm
    X = mixture
    k = 15
    i1, d1 = _approx(X, k, seed=9, fill=0x00)
    i2, d2 = _approx(X, k, seed=9, fill=0xFF)
    i3, d3 = _approx(X, k, seed=9)
    assert torch.equal(i1, i2) and torch.equal(i1, i3)
    assert torch.equal(d1.view(torch.int32), d2.view(torch.int32)) and torch.equal(d1.view(torch.int32),
                                                                                    d3.view(torch.int32))
    # another seed: another run, the same quality
    i4, d4 = _approx(X, k, seed=12345)
    ri, rd = dm.knn_device(X, k)
    _recall_checks(i4, d4, ri, rd)


def test_k_nearest_neighbors_routes_to_the_approximate_search(monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import preprocess
    from pymde_b200.preprocess import data_matrix as dm
    Xn = _mixture(3000, 20, 4, seed=2).cpu().numpy()
    monkeypatch.setenv("PYMDE_B200_KNN", "approx")
    pm.seed(7)
    g1 = preprocess.k_nearest_neighbors(Xn, k=10)
    pm.seed(7)
    idx, d2 = dm.knn_approx_device(torch.from_numpy(Xn).cuda(), 10)
    g2 = dm._knn_graph(idx, d2, 3000, None, torch.device("cuda"))
    assert np.array_equal(np.asarray(g1.edges.cpu()), np.asarray(g2.edges.cpu()))
    np.testing.assert_array_equal(np.asarray(g1.distances.cpu()), np.asarray(g2.distances.cpu()))


def test_wide_k_routes_to_the_approximate_search(monkeypatch):
    import pymde_b200 as pm
    from pymde_b200 import _lib, preprocess
    from pymde_b200.preprocess import data_matrix as dm
    monkeypatch.setenv("PYMDE_B200_KNN", "approx")
    X = _mixture(1500, 16, 4, seed=5)
    pm.seed(4)
    g = preprocess.k_nearest_neighbors(X.cpu().numpy(), k=30)
    pm.seed(4)
    idx, d2 = dm.knn_approx_device(X, 30)
    ref = dm._knn_graph(idx, d2, 1500, None, torch.device("cuda"))
    assert np.array_equal(np.asarray(g.edges.cpu()), np.asarray(ref.edges.cpu()))
    with pytest.raises(_lib.MdeError):
        dm.knn_approx_device(X, 65)


def test_unset_variable_takes_the_exact_path(monkeypatch):
    from pymde_b200 import preprocess
    from pymde_b200.preprocess import data_matrix as dm
    monkeypatch.delenv("PYMDE_B200_KNN", raising=False)

    def refuse(*a, **kw):
        raise AssertionError("approximate search taken without PYMDE_B200_KNN=approx")
    monkeypatch.setattr(dm, "knn_approx_device", refuse)
    X = _mixture(1500, 16, 4, seed=4)
    g = preprocess.k_nearest_neighbors(X.cpu().numpy(), k=7)
    idx, d2 = dm.knn_device(X, 7)
    ref = dm._knn_graph(idx, d2, 1500, None, torch.device("cuda"))
    assert np.array_equal(np.asarray(g.edges.cpu()), np.asarray(ref.edges.cpu()))


def test_preserve_neighbors_is_reproducible_under_approx(monkeypatch):
    import pymde_b200 as pm
    monkeypatch.setenv("PYMDE_B200_KNN", "approx")
    Xn = _mixture(4000, 32, 6, seed=8).cpu().numpy()
    runs = []
    for _ in range(2):
        pm.seed(3)
        mde = pm.preserve_neighbors(Xn, embedding_dim=2, verbose=False)
        runs.append((mde.edges.cpu().numpy(), mde.distortion_function.weights.cpu().numpy()))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert np.array_equal(runs[0][1], runs[1][1])
    Y = mde.embed(max_iter=20)
    assert Y.shape == (4000, 2) and bool(torch.isfinite(Y).all())
