"""CPU: the row-range k-nearest-neighbour search (`mde_knn_rows`, `mde_knn16_rows`, include/mde_b200.h) is exported,
additive (the ABI version is still 1) and rejects bad arguments before it touches a device; its candidate-slice rule
(mde_logic.h: knn_slices) fills the SMs only while the query tiles leave them idle; and steps 2-5 of
`pymde_b200.embed_new_points` (compaction, attractive and repulsive edges, initial iterate) agree with a numpy
restatement on CPU tensors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
NAMES = ("mde_knn_rows_ws_bytes", "mde_knn_rows", "mde_knn16_rows_ws_bytes", "mde_knn16_rows")
NUM_SMS = 132


def _ws(n, d, rows, k, half=False):
    need = C.c_size_t(0)
    fn = _lib.load().mde_knn16_rows_ws_bytes if half else _lib.load().mde_knn_rows_ws_bytes
    assert fn(n, d, rows, k, C.byref(need)) == 0
    return need.value


def _call(n, d, rb, re, k, half=False, dtype=_lib.DTYPE_FP16, X=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE,
          ws_bytes=1 << 40):
    lib = _lib.load()
    fb = C.c_int(-7)
    if half:
        code = lib.mde_knn16_rows(X, dtype, n, d, rb, re, k, out_i, out_d, ws, ws_bytes, None, C.byref(fb))
    else:
        code = lib.mde_knn_rows(X, n, d, rb, re, k, out_i, out_d, ws, ws_bytes, None, C.byref(fb))
    assert fb.value == -7  # nothing written on a refusal
    return code


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "16bit"])
def test_bad_ranges_and_k_are_rejected(half):
    n, d = 1000, 30
    for rb, re in [(-1, 5), (0, 0), (5, 5), (6, 5), (0, n + 1), (n, n + 1), (999, 1001)]:
        assert _call(n, d, rb, re, 5, half) == _lib.MDE_E_INVALID, (rb, re)
    for k in (0, -1, 65, 1000):
        assert _call(n, d, 0, 10, k, half) == _lib.MDE_E_INVALID, k
    assert _call(10, d, 0, 10, 10, half) == _lib.MDE_E_INVALID  # k > n - 1
    assert _call(1, d, 0, 1, 1, half) == _lib.MDE_E_INVALID
    assert _call(n, 0, 0, 10, 5, half) == _lib.MDE_E_INVALID
    for kw in ("X", "out_i", "out_d", "ws"):
        assert _call(n, d, 0, 10, 5, half, **{kw: None}) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("dtype", [0, 3, -1])
def test_unknown_dtype_codes_are_rejected(dtype):
    assert _call(1000, 30, 0, 10, 5, half=True, dtype=dtype) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "16bit"])
@pytest.mark.parametrize("k", [5, 40])
def test_workspace_too_small_or_misaligned_is_rejected(half, k):
    need = _ws(1000, 30, 300, k, half)
    assert need % 1024 == 0
    assert _call(1000, 30, 100, 400, k, half, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _call(1000, 30, 100, 400, k, half, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(1000, 30, 100, 400, k, half, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID


def test_workspace_query_rejects_bad_arguments():
    lib = _lib.load()
    need = C.c_size_t(0)
    for fn in (lib.mde_knn_rows_ws_bytes, lib.mde_knn16_rows_ws_bytes):
        assert fn(1000, 30, 10, 5, None) == _lib.MDE_E_INVALID
        for n, d, rows, k in [(1, 30, 1, 1), (1000, 0, 10, 5), (1000, 30, 0, 5), (1000, 30, 1001, 5),
                              (1000, 30, 10, 0), (1000, 30, 10, 65), (10, 30, 5, 10)]:
            assert fn(n, d, rows, k, C.byref(need)) == _lib.MDE_E_INVALID, (n, d, rows, k)


def _slices(n, rows, k):
    return _lib.load().mde_dbg_knn_slices(n, rows, k)


@pytest.mark.parametrize("k,tm,tn", [(15, 128, 128), (40, 64, 128)])
def test_slice_rule(k, tm, tn):
    for n in (130, 1000, 5000, 40000, 70000, 10 ** 6):
        c_tiles = -(-n // 128) * 128 // tn
        for rows in sorted({1, 37, 300, 1000, 3000, 10000, n // 2, n}):
            if rows > n:
                continue
            q_tiles = -(-rows // tm)
            s = _slices(n, rows, k)
            assert 1 <= s <= max(1, min(c_tiles, 16)), (n, rows, s)
            if q_tiles >= NUM_SMS:
                assert s == 1, (n, rows, s)  # the query tiles fill the SMs: no split
            else:
                assert q_tiles * s <= NUM_SMS  # one wave
                # as many slices as fit, up to one candidate tile each and 16
                assert s == max(1, min(NUM_SMS // q_tiles, c_tiles, 16)), (n, rows, s)
    # the full searches follow the same rule: split at n = 5 000, not at 70 000
    assert _slices(5000, 5000, 15) > 1 and _slices(70000, 70000, 15) == 1 and _slices(70000, 70000, 40) == 1
    assert _slices(1000, 2000, 15) == -1 and _slices(1000, 10, 65) == -1


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "16bit"])
def test_workspace_grows_with_the_slices(half):
    n, d = 200000, 64
    for k in (15, 40):
        s1, s2 = _slices(n, 1000, k), _slices(n, 20000, k)
        assert s1 > s2 == 1
        per_row1 = (_ws(n, d, 1000, k, half) - _ws(n, d, 1, k, half))
        assert _ws(n, d, 1000, k, half) > _ws(n, d, 1000 // s1 + 1, k, half)
        kk = 32 if k <= 24 else 96
        # two lists (indices, scores) of S KK entries per query row
        assert per_row1 >= 999 * s1 * kk * 8 - 4096
        assert _ws(n, d, 20000, k, half) >= _ws(n, d, 1000, k, half)


# --- steps 2-5 of embed_new_points on CPU tensors -------------------------------------------------------------------

def _lists_case(seed, n_old=40, n_new=12, k=5, holes=True):
    rng = np.random.default_rng(seed)
    n = n_old + n_new
    idx = np.empty((n_new, k), dtype=np.int64)
    for i in range(n_new):
        g = n_old + i
        cand = np.setdiff1d(np.arange(n), [g])
        # mostly old points, some new ones (mutual pairs likely among few new points)
        p = np.where(cand >= n_old, 4.0, 1.0)
        idx[i] = rng.choice(cand, k, replace=False, p=p / p.sum())
    if holes:
        idx[rng.random(idx.shape) < 0.15] = -1
        idx[0] = -1  # a new point without attractive edges
    for a, b in ((1, 2), (2, 1)):  # new points 1 and 2 list each other: a mutual pair
        idx[a][idx[a] == n_old + b] = -1
        idx[a, 0] = n_old + b
    return torch.from_numpy(idx)


def _restate(idx, n_old, rep_global):
    """numpy: items, local lists, attractive edge weights by directed-entry counts."""
    idx = idx.numpy()
    n_new = idx.shape[0]
    ends = np.concatenate([idx[idx >= 0], rep_global.reshape(-1)])
    items = np.concatenate([np.arange(n_old, n_old + n_new), np.unique(ends[(ends >= 0) & (ends < n_old)])])
    local = {int(g): i for i, g in enumerate(items)}
    weights = {}
    for i in range(n_new):
        for j in idx[i]:
            if j < 0:
                continue
            a, b = sorted((i, local[int(j)]))
            weights[(a, b)] = weights.get((a, b), 0) + 1
    return items, local, weights


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("fraction", [None, 1, 2.5])
def test_new_point_graph_restated(seed, fraction):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    from pymde_b200.preprocess.graph import Graph
    n_old = 40
    idx = _lists_case(seed, n_old=n_old)
    n_new = idx.shape[0]
    n = n_old + n_new
    pm.seed(seed)
    items, lists, edges, weights = recipes._new_points_graph(idx, n_old, fraction)
    pm.seed(seed)
    items2, lists2, edges2, weights2 = recipes._new_points_graph(idx, n_old, fraction)
    assert torch.equal(edges, edges2) and torch.equal(weights, weights2) and torch.equal(items, items2)
    att = weights > 0
    n_att = int(att.sum())
    assert bool(att[:n_att].all()) and not bool(att[n_att:].any())  # attractive edges first
    rep_local = edges[n_att:].numpy()
    rep_global = items.numpy()[rep_local]
    it, local, w = _restate(idx, n_old, rep_global)
    # compaction: new points first, then the referenced old points ascending
    np.testing.assert_array_equal(items.numpy(), it)
    assert list(items[:n_new]) == list(range(n_old, n))
    # local lists: relabelled new rows, -1 on old rows
    want = np.where(idx.numpy() >= 0, np.vectorize(lambda g: local.get(int(g), -1))(idx.numpy()), -1)
    np.testing.assert_array_equal(lists[:n_new].numpy(), want)
    assert bool((lists[n_new:] == -1).all())
    # attractive edges and weights: Graph.from_edges on the directed entries, and the counting rule
    e_att = edges[:n_att].numpy()
    got = {(int(a), int(b)): float(x) for (a, b), x in zip(e_att, weights[:n_att].numpy())}
    assert got == {kk: float(v) for kk, v in w.items()}
    rows = np.repeat(np.arange(n_new), idx.shape[1])
    ent = lists[:n_new].numpy().reshape(-1)
    g = Graph.from_edges(np.stack([rows[ent >= 0], ent[ent >= 0]], 1), None, n_items=len(it))
    np.testing.assert_array_equal(np.asarray(g.edges), e_att)
    np.testing.assert_array_equal(np.asarray(g.weights), weights[:n_att].numpy())
    assert set(w.values()) <= {1, 2} and 2 in w.values()  # mutual new-new pairs weigh 2
    # repulsive pairs: canonical, no self pair, no repeat, not attractive, touching a new point
    if fraction is None:
        assert rep_local.shape[0] == 0
        return
    assert bool((rep_local[:, 0] < rep_local[:, 1]).all())
    keys = rep_global.min(1) * n + rep_global.max(1)
    assert len(np.unique(keys)) == len(keys)
    att_g = {(min(a, b), max(a, b)) for a, b in items.numpy()[e_att]}
    assert not any((min(a, b), max(a, b)) in att_g for a, b in rep_global)
    assert bool((rep_global.max(1) >= n_old).all())
    available = n_new * (n - 1) - n_new * (n_new - 1) // 2 - n_att
    assert rep_local.shape[0] == min(int(fraction * n_att), available)
    assert bool((weights[n_att:] == -1).all())
    pm.seed(seed + 100)
    _, _, edges3, _ = recipes._new_points_graph(idx, n_old, fraction)
    assert not torch.equal(edges3, edges)  # the module RNG decides the draws


def test_repulsive_pairs_saturate_when_few_are_available():
    from pymde_b200 import recipes
    n_old = 3
    idx = torch.tensor([[0, 1, 4], [0, 3, 2], [3, 1, 2]])  # new points 3, 4, 5
    items, lists, edges, weights = recipes._new_points_graph(idx, n_old, 10)
    n_att = int((weights > 0).sum())
    n, n_new = 6, 3
    available = n_new * (n - 1) - n_new * (n_new - 1) // 2 - n_att
    assert edges.shape[0] - n_att == available  # every pair touching a new point is used


@pytest.mark.parametrize("seed", [0, 3])
def test_new_point_init_restated(seed):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    n_old, m = 40, 3
    idx = _lists_case(seed, n_old=n_old)
    n_new = idx.shape[0]
    rng = np.random.default_rng(seed)
    emb = torch.from_numpy(rng.standard_normal((n_old, m)).astype(np.float32))
    items, lists, edges, weights = recipes._new_points_graph(idx, n_old, 1)
    n_att = int((weights > 0).sum())
    X = recipes._new_points_init(items, lists, n_new, emb, edges[:n_att])
    assert X.dtype == torch.float32 and X.shape == (items.numel(), m)
    # anchored rows: exactly the embedding rows
    assert torch.equal(X[n_new:], emb[items[n_new:]])
    e = emb.numpy().astype(np.float64)
    want = np.concatenate([np.stack([e[o].mean(0) if len(o) else e.mean(0) for o in
                                     ([int(g) for g in idx[i].numpy() if 0 <= g < n_old] for i in range(n_new))]),
                           e[items[n_new:].numpy()]])
    ea = edges[:n_att].numpy()
    coincide = bool((np.abs(want[ea[:, 0]] - want[ea[:, 1]]).max(1) < 1e-6).any())
    # new points without fitted neighbours start at the same place: a joining edge has length 0, and 1e-4 randn
    # separates them
    np.testing.assert_allclose(X[:n_new].numpy(), want[:n_new], rtol=1e-5, atol=1e-3 if coincide else 1e-6)
    # coincident ends of an attractive edge: only the new rows move
    lists2 = torch.full_like(lists, -1)
    lists2[:n_new, 0] = n_new  # every new point's only neighbour is the first old item
    lists2[1, 1] = 0           # and new point 1 also joins new point 0: both start at the same place
    e2 = torch.tensor([[0, 1], [0, n_new]])
    pm.seed(seed)
    X2 = recipes._new_points_init(items, lists2, n_new, emb, e2)
    assert torch.equal(X2[n_new:], emb[items[n_new:]])
    assert not torch.equal(X2[0], X2[1])
    assert float((X2[:n_new] - emb[items[n_new]]).abs().max()) < 1e-2
