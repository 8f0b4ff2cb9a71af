"""The sparse exact k-nearest-neighbour searches on data far from the origin, against fp64.

`mde_knn_csr`, `mde_knn_csr_wide`, `mde_knn_csr_long` and `mde_knn_csr_rows` (csrc/mde_knn_sparse.cu) rank candidates
by ||x||^2 - 2 q.x with bf16 x 3 cross terms and do not centre the columns (that would densify the matrix).  A column
every row shares far from the origin -- one-hot categories next to a latitude and longitude, a year next to word
counts, a constant bias feature -- makes those scores rounding noise (tests/test_knn_csr_offset_cpu.py reproduces this
on the CPU).  The searches certify every row with a bound in the row's non-zeros and search the rows that fail
directly, so the result must be the exact one on every family below, and the ordinary families must rarely need the
direct search.

Reference: exact fp64 distances (candidates from the fp64 column-centred norm expansion of the dense matrix, then the
sum of squared differences; a row whose candidates reach an fp32 distance of +inf is measured against every row), the k
smallest by (fp32 distance, index).  Contract (that of tests/test_gpu_knn_sparse.py::_compare): indices in range, no
self neighbour, no repeat, distances within one ulp of the fp64 sum rounded once, ascending by (distance, index), the
reference's k smallest distances, and the reference's neighbour set on every row whose k-th and (k + 1)-th neighbours
are separated by more than fp32 rounding."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

N = 4000  # a multiple of neither 64 nor 128


# --- data families (seeded scipy CSR, float32) ------------------------------------------------------------------------

def _clustered(rng, n, d, nnz_row, n_centres):
    """Rows around sparse cluster centres: each row keeps its centre's support, with noisy values."""
    cols = np.stack([rng.choice(d, nnz_row, replace=False) for _ in range(n_centres)])
    vals = rng.standard_normal((n_centres, nnz_row)) * 4
    lab = rng.integers(0, n_centres, n)
    v = (vals[lab] + 0.1 * rng.standard_normal((n, nnz_row))).ravel()
    return sp.csr_matrix((v, (np.repeat(np.arange(n), nnz_row), cols[lab].ravel())), shape=(n, d))


def _zipf_counts(rng, n, d, per_row):
    """Column counts of documents whose terms follow a Zipf law (rank^-1.1)."""
    p = 1.0 / np.arange(1, d + 1) ** 1.1
    p /= p.sum()
    cols = rng.choice(d, size=(n, per_row), p=p)
    A = sp.csr_matrix((np.ones(n * per_row), (np.repeat(np.arange(n), per_row), cols.ravel())), shape=(n, d))
    A.sum_duplicates()
    return A


def family(name, n=N, seed=0):
    """A named n-row scipy CSR float32 matrix (seeded)."""
    rng = np.random.default_rng(seed)
    if name == "latlong_onehot":  # 20 one-hot categories next to the latitude and longitude of points in one city
        cat = sp.csr_matrix((np.ones(n), (np.arange(n), rng.integers(0, 20, n))), shape=(n, 20))
        ll = np.array([40.7, -74.0]) + 0.05 * rng.standard_normal((n, 2))
        A = sp.hstack([cat, sp.csr_matrix(ll)])
    elif name == "year_counts":  # a year column next to 1 %-dense term weights uniform in [0, 1), d = 3 001
        year = sp.csr_matrix((2000.0 + rng.integers(0, 20, n))[:, None])
        A = sp.hstack([year, sp.random(n, 3000, density=0.01, random_state=rng)])
    elif name == "far_shared":  # ten clusters at radius 1 000 on 16 shared columns, spread 1, plus sparse noise
        c = rng.standard_normal((10, 16))
        c *= 1000.0 / np.linalg.norm(c, axis=1, keepdims=True)
        dense = c[rng.integers(0, 10, n)] + rng.standard_normal((n, 16))
        noise = sp.random(n, 2000, density=0.01, random_state=rng, data_rvs=rng.standard_normal)
        A = sp.hstack([sp.csr_matrix(dense), noise])
    elif name == "bias_tfidf":  # L2-normalised TF-IDF of Zipf-column documents and a constant column of 100
        tf = _zipf_counts(rng, n, 3000, 40)
        df = np.bincount(tf.indices, minlength=3000)
        tf.data *= np.log(n / np.maximum(df, 1))[tf.indices] + 1.0
        tf = sp.diags(1.0 / np.sqrt(np.asarray(tf.multiply(tf).sum(1)).ravel())) @ tf
        A = sp.hstack([tf, sp.csr_matrix(np.full((n, 1), 100.0))])
    elif name == "dup_far":  # far_shared with its first n / 8 rows copied to the end: d^2 = 0 ties far from the origin
        base = family("far_shared", n - n // 8, seed)
        A = sp.vstack([base, base[: n // 8]])
    elif name == "huge_rows":  # ordinary rows and five rows near 1e20, whose fp32 squared norms overflow
        A = family("uniform", n, seed).tolil()
        for j, r in enumerate(rng.choice(n, 5, replace=False)):
            A.rows[r], A.data[r] = [10 * j], [1e20 * (1.0 + 0.1 * j)]
    elif name.startswith("far_groups_"):  # groups of g rows, each on its own column, next to a shared column of 300
        g = int(name.rsplit("_", 1)[1])
        lab = rng.permutation(np.arange(n) // g)
        own = sp.csr_matrix((np.full(n, 10.0), (np.arange(n), lab)), shape=(n, lab.max() + 1))
        dense = np.concatenate([np.full((n, 1), 300.0), 0.05 * rng.standard_normal((n, 4))], 1)
        A = sp.hstack([sp.csr_matrix(dense), own])
    elif name == "count_docs":  # near-duplicate integer count documents, values 500 .. 1 500
        cols = np.stack([rng.choice(3000, 40, replace=False) for _ in range(300)])
        vals = rng.integers(500, 1501, (300, 40))
        lab = rng.integers(0, 300, n)
        v = vals[lab] + rng.integers(-3, 4, (n, 40))
        A = sp.csr_matrix((v.ravel().astype(np.float64), (np.repeat(np.arange(n), 40), cols[lab].ravel())),
                          shape=(n, 3000))
    elif name == "uniform":  # 2 %-dense N(0, 1), d = 3 000
        A = sp.random(n, 3000, density=0.02, random_state=rng, data_rvs=rng.standard_normal)
    elif name == "clustered":
        A = _clustered(rng, n, 20000, 30, 273)
    elif name == "zipf_text":  # Zipf-column documents with continuous weights
        A = _zipf_counts(rng, n, 3000, 40)
        A.data = rng.random(A.nnz)
    elif name == "mnist_csr":  # MNIST-like clipped Gaussian, ~80 % zeros, as CSR
        X = rng.standard_normal((n, 784))
        A = sp.csr_matrix(np.where(X < 0.8416, 0.0, np.minimum(X, 1.0)))
    else:
        raise KeyError(name)
    A = sp.csr_matrix(A, dtype=np.float32)
    A.sum_duplicates()
    A.eliminate_zeros()
    return A


FAR = ["latlong_onehot", "year_counts", "far_shared", "bias_tfidf", "dup_far"]  # the certificate must fail there
ORDINARY = ["uniform", "clustered", "zipf_text", "mnist_csr"]  # continuous: the certificate must hold
TIE_HEAVY = ["dup_far", "count_docs"]  # exact ties at the k-th neighbour are common


# --- fp64 reference and the contract -----------------------------------------------------------------------------------

def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _exact(X, rows, cols):
    """fp64 sum (x_r - x_c)^2 of rows [r] against cols [r, m], in row chunks."""
    out = torch.empty(cols.shape, dtype=torch.float64, device=X.device)
    step = max(1, (1 << 27) // max(1, cols.shape[1] * X.shape[1]))
    for s0 in range(0, cols.shape[0], step):
        out[s0:s0 + step] = ((X[rows[s0:s0 + step]][:, None, :] - X[cols[s0:s0 + step]]) ** 2).sum(-1)
    return out


def _by_fp32_then_index(cand, exact):
    """Candidates ordered by (fp32 distance, index), with their fp64 distances."""
    cand, pos = torch.sort(cand, 1)
    exact = torch.gather(exact, 1, pos)
    _, pos = torch.sort(exact.float(), dim=1, stable=True)
    return torch.gather(cand, 1, pos), torch.gather(exact, 1, pos)


def reference(A, k, extra=24):
    """(fp64 distances [n, k + 1], indices [n, k]) of the k + 1 nearest rows by (fp32 distance, index)."""
    X = torch.tensor(A.toarray(), dtype=torch.float64, device="cuda")
    n = X.shape[0]
    sq = (X * X).sum(1)
    mu = X[sq < 1e30].mean(0)  # (rows near 1e20 would swamp the mean)
    Xc = X - mu
    sqc = (Xc * Xc).sum(1)
    kc = min(n - 1, k + extra)
    idx, val = [], []
    for s0 in range(0, n, 1024):
        Q = Xc[s0:s0 + 1024]
        r = torch.arange(s0, s0 + Q.shape[0], device="cuda")
        score = sqc[None, :] - 2.0 * Q @ Xc.T
        score[torch.arange(Q.shape[0]), r] = float("inf")
        cand = torch.topk(score, kc, dim=1, largest=False)[1]
        c, e = _by_fp32_then_index(cand, _exact(X, r, cand))
        idx.append(c); val.append(e)
    idx, val = torch.cat(idx), torch.cat(val)
    # a row whose kept candidates reach +inf in fp32 ties with every far row: measure it against all rows
    for r in torch.nonzero(~torch.isfinite(val[:, min(k, kc - 1)].float())).ravel().tolist():
        cand = torch.tensor([[c for c in range(n) if c != r]], device="cuda")
        c, e = _by_fp32_then_index(cand, _exact(X, torch.tensor([r], device="cuda"), cand))
        idx[r], val[r] = c[0, :kc], e[0, :kc]
    return val[:, :k + 1], idx[:, :k], X


def check(A, k, idx, d2, rows=None, tie_rare=True):
    """The contract on the query rows `rows` (default: all) of A."""
    val, ref, X = reference(A, k)
    n = A.shape[0]
    rows = torch.arange(n, device="cuda") if rows is None else rows
    val, ref = val[rows], ref[rows]
    got = idx.long()
    assert got.shape == (rows.numel(), k) and d2.shape == (rows.numel(), k)
    assert int(got.min()) >= 0 and int(got.max()) < n
    assert not bool((got == rows[:, None]).any())
    s = torch.sort(got, 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all())  # no repeats
    ex = _exact(X, rows, got).float().cpu().numpy()
    dg = d2.cpu().numpy()
    assert _ulps(dg, ex).max() <= 1  # the fp64 merge rounded once
    dd, ii, dp, ip = d2[:, 1:], idx[:, 1:], d2[:, :-1], idx[:, :-1]
    assert bool(((dd > dp) | ((dd == dp) & (ii > ip))).all())  # ascending by (distance, index)
    assert _ulps(dg, val[:, :k].float().cpu().numpy()).max() <= 1  # the k smallest distances
    if val.shape[1] > k:
        clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-30
        same = (s == torch.sort(ref, 1)[0]).all(1)
        assert bool(same[clear].all()), int((~same[clear]).sum())
        if tie_rare:
            assert float(clear.float().mean()) >= 0.9
        return clear, ref
    return None, ref


# --- the raw entries ---------------------------------------------------------------------------------------------------

def route_of(k):
    return "_long" if k > 64 else "_wide" if k > 24 else ""


def _ws(need, fill):
    ws = torch.full((need + 1024,), fill, dtype=torch.uint8, device="cuda")
    return ws, ws.data_ptr() + (-ws.data_ptr()) % 1024


def search(A, k, route=None, fill=0xA5):
    """(idx, d2, rows searched directly) of the full `_ex` entry of `route` (default: the one k selects) on a
    workspace filled with `fill`."""
    from pymde_b200 import _lib
    from pymde_b200.preprocess import data_matrix as dm
    lib = _lib.load()
    (ip, ix, v), (n, d) = dm._to_device_csr(A, torch.device("cuda"))
    nnz = int(ix.shape[0])
    name = "knn_csr" + (route_of(k) if route is None else route)
    need = C.c_size_t(0)
    _lib.check(getattr(lib, "mde_%s_ws_bytes" % name)(n, d, nnz, C.byref(need)))
    ws, p = _ws(need.value, fill)
    idx = torch.full((n, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((n, k), -7.0, dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    _lib.check(getattr(lib, "mde_%s_ex" % name)(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz, k,
                                                idx.data_ptr(), d2.data_ptr(), p, need.value, None, C.byref(fb)))
    torch.cuda.synchronize()
    assert 0 <= fb.value <= n
    return idx, d2, fb.value


def rows_search(A, k, rb, re, fill=0xA5):
    """(idx, d2, rows searched directly) of mde_knn_csr_rows_ex."""
    from pymde_b200 import _lib
    from pymde_b200.preprocess import data_matrix as dm
    lib = _lib.load()
    (ip, ix, v), (n, d) = dm._to_device_csr(A, torch.device("cuda"))
    nnz = int(ix.shape[0])
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_csr_rows_ws_bytes(n, d, nnz, re - rb, k, C.byref(need)))
    ws, p = _ws(need.value, fill)
    idx = torch.full((re - rb, k), -7, dtype=torch.int32, device="cuda")
    d2 = torch.full((re - rb, k), -7.0, dtype=torch.float32, device="cuda")
    fb = C.c_int(-1)
    _lib.check(lib.mde_knn_csr_rows_ex(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, d, nnz, rb, re, k,
                                       idx.data_ptr(), d2.data_ptr(), p, need.value, None, C.byref(fb)))
    torch.cuda.synchronize()
    assert 0 <= fb.value <= re - rb
    return idx, d2, fb.value


def _slices(n, rows, k):
    from pymde_b200 import _lib
    return _lib.load().mde_dbg_knn_csr_slices(n, rows, k)


# --- every route, every family -----------------------------------------------------------------------------------------

KS = [1, 15, 24, 25, 64, 65, 200, 256]


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", FAR + ["huge_rows"])
def test_far_families_on_every_route(name, k):
    A = family(name, n=3001, seed=k)
    idx, d2, fb = search(A, k)
    print(name, k, "rows searched directly:", fb)
    # (beyond k = 64 the k-th neighbour of latlong_onehot lies in another category, among near-ties)
    check(A, k, idx, d2, tie_rare=name not in TIE_HEAVY and k <= 64)
    if name in FAR:
        assert fb > 0.5 * A.shape[0]  # the scores cannot separate the neighbours: the certificate must fail
    if name == "dup_far":  # every copied row finds its copy first, at distance exactly 0
        m = A.shape[0] // 8
        assert bool((d2[:m, 0] == 0).all())
        assert bool((idx[:m, 0].long() == torch.arange(A.shape[0] - m, A.shape[0], device="cuda")).all())


@pytest.mark.parametrize("k", [15, 64, 200])
@pytest.mark.parametrize("name", ORDINARY + ["count_docs"])
def test_ordinary_families_certify_and_repeat_bit_for_bit(name, k):
    A = family(name)
    idx, d2, fb = search(A, k)
    print(name, k, "rows searched directly:", fb)
    check(A, k, idx, d2, tie_rare=name in ORDINARY)
    if name in ORDINARY:
        assert fb <= 0.01 * A.shape[0], fb
    i2, e2, fb2 = search(A, k, fill=0x00)  # another workspace fill: the same bits and the same count
    assert fb2 == fb and torch.equal(idx, i2) and torch.equal(d2, e2)


@pytest.mark.parametrize("k", [15, 64, 200])
def test_far_family_repeats_bit_for_bit(k):
    A = family("year_counts", n=3001)
    i1, e1, fb1 = search(A, k, fill=0xA5)
    i2, e2, fb2 = search(A, k, fill=0x3C)
    assert fb1 == fb2 > 0 and torch.equal(i1, i2) and torch.equal(e1, e2)


@pytest.mark.parametrize("route", ["", "_wide", "_long"])
@pytest.mark.parametrize("name", ["latlong_onehot", "far_shared", "dup_far"])
def test_smallest_n(name, route):
    """n = k + 2: every row's list holds every other row, so every row is certified without the direct search."""
    k = {"": 24, "_wide": 64, "_long": 256}[route]
    A = family(name, n=k + 2, seed=1)
    idx, d2, fb = search(A, k, route)
    check(A, k, idx, d2, tie_rare=False)
    assert fb == 0


@pytest.mark.parametrize("route", ["", "_wide", "_long"])
def test_lower_routes_agree_with_the_direct_search(route):
    """A k any route takes, on a far family: most rows searched directly, the same bits on every route."""
    A = family("year_counts", n=3001, seed=5)
    i0, d0, _ = search(A, 20, "")
    i1, d1, fb = search(A, 20, route)
    assert fb > 0 and torch.equal(i0, i1) and torch.equal(d0, d1)


def test_the_copy_in_the_last_row_is_found():
    """dup_far puts the copy of row m - 1 in row n - 1: a direct search that stops short of the last row misses it."""
    A = family("dup_far", n=3001, seed=2)
    n, m = A.shape[0], A.shape[0] // 8
    for k in (1, 15, 64, 200):
        idx, d2, fb = search(A, k)
        assert fb > 0
        assert int(idx[m - 1, 0]) == n - 1 and float(d2[m - 1, 0]) == 0.0
        assert int(idx[n - 1, 0]) == m - 1 and float(d2[n - 1, 0]) == 0.0


@pytest.mark.parametrize("g", [16, 40, 100])
def test_groups_of_k_rows_far_from_the_origin(g):
    """Groups of exactly k = g rows: the k - 1 others of a row's group lie near 0, every other row near 200, within the
    scores' error of one another.  The list keeps the group and a handful of those others at random, so the k-th
    neighbour is right only if the certificate compares the k-th re-ranked distance, not the (k - 1)-th, and fails."""
    A = family("far_groups_%d" % g, n=3001, seed=g)
    idx, d2, fb = search(A, g)
    check(A, g, idx, d2, tie_rare=False)
    assert fb > 0.5 * A.shape[0]


# --- the row search ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 15, 24, 25, 64, 65, 200])
@pytest.mark.parametrize("name", ["latlong_onehot", "year_counts", "dup_far", "huge_rows"])
def test_row_search_gives_the_full_search_on_far_families(name, k):
    """Ranges on and off tile boundaries, split into candidate slices (S > 1) up to k = 64, in one slice beyond: the
    full search's bits and the fp64 contract."""
    A = family(name, n=N, seed=3)
    n = A.shape[0]
    full_i, full_d, full_fb = search(A, k)
    seen = set()
    for rb, re in [(37, 41), (1000, 1300), (n - 500, n), (0, n)]:
        i, d2, fb = rows_search(A, k, rb, re)
        seen.add(_slices(n, re - rb, k))
        assert torch.equal(i, full_i[rb:re]) and torch.equal(d2, full_d[rb:re]), (rb, re)
        assert fb <= full_fb
        if (rb, re) == (0, n):
            assert fb == full_fb
        check(A, k, i, d2, rows=torch.arange(rb, re, device="cuda"), tie_rare=False)
    assert min(seen) > 1 if k <= 64 else seen == {1}, seen


@pytest.mark.parametrize("k", [15, 40])
def test_row_search_without_a_split_on_a_far_family(k):
    """Query ranges that fill the SMs on their own (S = 1) up to k = 64: the full search's bits and the contract."""
    A = family("latlong_onehot", n=17500, seed=4)
    n = A.shape[0]
    full_i, full_d, full_fb = search(A, k)
    for rb, re in [(0, n), (500, n)]:
        assert _slices(n, re - rb, k) == 1
        i, d2, fb = rows_search(A, k, rb, re)
        assert torch.equal(i, full_i[rb:re]) and torch.equal(d2, full_d[rb:re]), (rb, re)
        assert fb <= full_fb and fb > 0.5 * (re - rb)
    check(A, k, full_i, full_d, tie_rare=False)


# --- the Python entry points -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [15, 100])
@pytest.mark.parametrize("name", ["latlong_onehot", "year_counts"])
def test_graph_builders_on_offset_data(name, k):
    from pymde_b200 import preprocess
    from pymde_b200.preprocess import data_matrix as dm
    from pymde_b200.preprocess.graph import Graph
    A = family(name)
    idx, d2, n = dm._search(A, k, torch.device("cuda"))
    clear, ref = check(A, k, idx, d2, tie_rare=False)
    # the fp64 reference graph (on a row whose k-th and (k + 1)-th neighbours are within fp32 rounding, either is right)
    ref = torch.where(clear[:, None], ref, idx.long())
    e = torch.stack([torch.arange(N, device="cuda")[:, None].expand_as(ref).reshape(-1), ref.reshape(-1)], 1)
    want = Graph.from_edges(e.cpu(), None, n_items=N)
    g = preprocess.k_nearest_neighbors(A, k=k)
    np.testing.assert_array_equal(np.asarray(g.edges.cpu()), np.asarray(want.edges.cpu()))
    np.testing.assert_array_equal(np.asarray(g.weights.cpu()), np.asarray(want.weights.cpu()))
    build = dm.k_nearest_neighbors_device if k <= 64 else dm.k_nearest_neighbors_device_long
    gd = build(A, k)
    np.testing.assert_array_equal(gd.edges.cpu().numpy(), np.asarray(want.edges.cpu()))
    np.testing.assert_array_equal(gd.weights.cpu().numpy(), np.asarray(want.weights.cpu()))


@pytest.mark.parametrize("name", ["latlong_onehot", "year_counts"])
def test_embed_new_points_searches_the_new_rows_exactly(monkeypatch, name):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    data, new = family(name, n=3000, seed=7), family(name, n=300, seed=8)
    emb = torch.randn((3000, 2), generator=torch.Generator().manual_seed(0)).cuda()
    seen = {}
    original = dm.knn_rows_device

    def spy(X, k, row_begin, row_end):
        seen["args"] = (X, k, row_begin, row_end)
        seen["out"] = original(X, k, row_begin, row_end)
        return seen["out"]

    monkeypatch.setattr(dm, "knn_rows_device", spy)
    pm.seed(0)
    got = pm.embed_new_points(data, emb, new)
    assert got.shape == (300, 2) and bool(torch.isfinite(got).all())
    X, k, rb, re = seen["args"]
    assert sp.issparse(X) and (rb, re) == (3000, 3300)
    idx, d2 = seen["out"]
    check(sp.csr_matrix(X, dtype=np.float32), k, idx, d2, rows=torch.arange(rb, re, device="cuda"), tie_rare=False)
