"""ELL pull records (pymde_b200/csrc/mde_ell.cu) built by the HOST builder the library also uses on the GPU box:
decode every record and check that (i) every edge appears exactly once from each end, (ii) the pull sums the kernel
forms from the records -- with its two pad conventions -- equal the oracle's value and gradient
(oracle restates pymde/average_distortion.py:36-80).  No device is involved."""
import ctypes as C

import numpy as np
import pytest

from oracle import mde_oracle as O
from pymde_b200 import _lib

PAIR, WMAX = 384, 8


def build(n, m, edges, w, push_pull, rb=0, max_cta=0):
    lib = _lib.load()
    src = np.ascontiguousarray(edges[:, 0], dtype=np.int32)
    dst = np.ascontiguousarray(edges[:, 1], dtype=np.int32)
    w = np.ascontiguousarray(w, dtype=np.float32)
    h = _lib.mde_ell_host_t()
    rc = lib.mde_ell_host_layout(n, len(src), m, src.ctypes.data, dst.ctypes.data, w.ctypes.data, int(push_pull), rb,
                                 max_cta, C.byref(h))
    if rc != 0:
        return rc, None
    out = dict(
        rec=np.ctypeslib.as_array(h.rec, shape=(h.rec_bytes,)).copy(),
        rec_off=np.ctypeslib.as_array(h.rec_off, shape=(h.nrec + 1,)).copy(),
        bkt_tile=np.ctypeslib.as_array(h.bkt_tile, shape=(h.nbkt,)).copy(),
        bkt_wt0=np.ctypeslib.as_array(h.bkt_wt0, shape=(h.nbkt + 1,)).copy(),
        cta_wt0=np.ctypeslib.as_array(h.cta_wt0, shape=(h.ncta + 1,)).copy(),
        cta_bkt0=np.ctypeslib.as_array(h.cta_bkt0, shape=(h.ncta,)).copy(),
        nrec=h.nrec, nslots=h.nslots, nentries=h.nentries, npadded=h.npadded, rb=h.tile_rows_log2, ncta=h.ncta)
    lib.mde_ell_host_free(C.byref(h))
    return 0, out


def decode(lay, n, m):
    """-> one tuple per lane-slot ROW of every record (a record holds K rows of 32 lane-slots):
    (tile, cls, W, own[32], cnt[32], dup[32], w[W,32], nbr[W,32] global rows)"""
    rec, off = lay["rec"], lay["rec_off"].astype(np.int64) * 16
    R = 1 << lay["rb"]
    out = []
    bkt = 0
    for t in range(lay["nrec"]):
        while t >= lay["bkt_wt0"][bkt + 1]:
            bkt += 1
        tile = int(lay["bkt_tile"][bkt])
        r = rec[off[t]:off[t + 1]]
        W, cls, K, ns = np.frombuffer(r[:16].tobytes(), dtype=np.int32)
        assert W % 2 == 0 and 2 <= W <= WMAX and 1 <= K <= {2: 4, 4: 2}.get(W, 1) and 32 * (K - 1) < ns <= 32 * K
        assert len(r) == 16 + K * (128 + (W // 2) * PAIR), "record size"
        assert len(r) <= 2064, "slot size of the kernel"
        oww = np.frombuffer(r[16:16 + 128 * K].tobytes(), dtype=np.uint32).reshape(K, 32)
        assert np.array_equal((oww >> 31).astype(bool).ravel(), np.arange(32 * K) >= ns)
        cols = r[16 + 128 * K:]
        for k in range(K):
            ow = oww[k]
            own = (ow & 0xFFFFFF).astype(np.int64)
            cnt = ((ow >> 24) & 0x7F).astype(np.int64)
            dup = (ow >> 31).astype(bool)
            assert np.all(cnt[~dup] >= 1) and np.all(cnt[dup] == 0) and cnt.max() <= W
            wv = np.zeros((W, 32), np.float32)
            nb = np.zeros((W, 32), np.int64)
            for c2 in range(W // 2):
                blk = cols[(k * (W // 2) + c2) * PAIR: (k * (W // 2) + c2 + 1) * PAIR]
                w2 = np.frombuffer(blk[:256].tobytes(), dtype=np.float32).reshape(32, 2)
                ix = np.frombuffer(blk[256:].tobytes(), dtype=np.uint16).reshape(32, 2).astype(np.int64)
                assert np.all(ix % (4 * m) == 0)
                wv[2 * c2], wv[2 * c2 + 1] = w2[:, 0], w2[:, 1]
                nb[2 * c2], nb[2 * c2 + 1] = tile * R + ix[:, 0] // (4 * m), tile * R + ix[:, 1] // (4 * m)
            assert nb.max() < n and own.max() < n
            out.append((tile, int(cls), int(W), own, cnt, dup, wv, nb))
    return out


def pull_sums(recs, X, coeff, masked):
    """What the kernel computes.  coeff(d2, w, cls) -> (f, g) per entry; masked: use the per-lane count (generic
    functions) instead of relying on w = 0 pads (weight functions)."""
    n, m = X.shape
    grad = np.zeros((n, m))
    loss = 0.0
    for tile, cls, W, own, cnt, dup, wv, nb in recs:
        xi = X[own]
        acc = np.zeros((32, m))
        for e in range(W):
            diff = xi - X[nb[e]]
            d2 = (diff * diff).sum(1)
            f, g = coeff(d2, wv[e].astype(np.float64), cls)
            if masked:
                live = e < cnt
                f = np.where(live, f, 0.0)
                g = np.where(live, g, 0.0)
            loss += f.sum()
            acc += g[:, None] * diff
        np.add.at(grad, own[~dup], acc[~dup])
    return 0.5 * loss, grad


def random_problem(rng, n, p, push_pull, local):
    if local:  # k-NN-like: neighbours inside a window
        i = rng.integers(0, n, p)
        j = (i + rng.integers(1, max(2, n // 20), p)) % n
    else:
        i = rng.integers(0, n, p)
        j = rng.integers(0, n, p)
    keep = i != j
    e = np.unique(np.sort(np.stack([i[keep], j[keep]], 1), axis=1), axis=0).astype(np.int64)
    if push_pull:
        w = np.where(rng.random(len(e)) < 0.5, 1.0, -1.0) * rng.uniform(0.5, 2.0, len(e))
    else:
        w = rng.uniform(0.2, 2.0, len(e))
    return e, w.astype(np.float32)


@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("push_pull", [False, True])
@pytest.mark.parametrize("n,p,rb,local", [(300, 2500, 8, False), (1000, 12000, 8, True), (64, 40, 0, False),
                                          (5000, 30000, 10, True), (40, 700, 8, False)])
def test_records_hold_every_edge_from_both_ends_and_reproduce_the_oracle(m, push_pull, n, p, rb, local):
    rng = np.random.default_rng(1000 * m + 7 * n + push_pull)
    edges, w = random_problem(rng, n, p, push_pull, local)
    rc, lay = build(n, m, edges, w, push_pull, rb)
    assert rc == 0
    recs = decode(lay, n, m)
    # (i) the multiset of real directed entries = both directions of every edge, class = sign of the weight
    got = []
    for tile, cls, W, own, cnt, dup, wv, nb in recs:
        for l in range(32):
            for e in range(int(cnt[l])):
                got.append((int(own[l]), int(nb[e, l]), float(wv[e, l]), cls))
            for e in range(int(cnt[l]), W):  # pads: zero weight, a real neighbour row
                assert wv[e, l] == 0.0
    want = []
    for (i, j), wk in zip(edges, w):
        c = int(push_pull and not (wk >= 0))
        want += [(int(i), int(j), float(wk), c), (int(j), int(i), float(wk), c)]
    assert sorted(got) == sorted(want)
    assert lay["nentries"] == 2 * len(edges) and lay["npadded"] == sum(32 * r[2] for r in recs)  # rows x W
    # tables
    assert lay["cta_wt0"][0] == 0 and lay["cta_wt0"][-1] == lay["nrec"] and np.all(np.diff(lay["cta_wt0"]) >= 0)
    assert np.all(np.diff(lay["bkt_wt0"]) > 0) and lay["bkt_wt0"][0] == 0 and lay["bkt_wt0"][-1] == lay["nrec"]
    assert np.all(np.diff(lay["bkt_tile"]) > 0)
    for c in range(lay["ncta"]):
        b = lay["cta_bkt0"][c]
        if lay["cta_wt0"][c] < lay["nrec"]:
            assert lay["bkt_wt0"][b] <= lay["cta_wt0"][c] < lay["bkt_wt0"][b + 1]
    # (ii) pull sums = oracle; weight function: quadratic penalty f = w d^2 (pads carry w = 0, no mask)
    X = rng.standard_normal((n, m))
    pt = len(edges)
    spec = O.FnSpec(O.P_QUADRATIC, w)
    v_ref, g_ref = O.average_distortion(X, edges, spec, True)
    loss, grad = pull_sums(recs, X, lambda d2, ww, cls: (ww * d2, 2.0 * ww / pt), masked=False)
    np.testing.assert_allclose(loss / pt, v_ref, rtol=1e-12)
    np.testing.assert_allclose(grad, g_ref, rtol=1e-10, atol=1e-12 * np.abs(g_ref).max())
    if not push_pull:
        # deviation function: quadratic loss f = (d - delta)^2 -- pads (delta = 0) must be masked by the lane count
        spec = O.FnSpec(O.L_QUADRATIC, w)
        v_ref, g_ref = O.average_distortion(X, edges, spec, True)

        def lq(d2, dev, cls):
            d = np.sqrt(d2)
            with np.errstate(all="ignore"):
                g = 2.0 * (d - dev) / pt / d
            return (d - dev) ** 2, np.where(np.isfinite(g), g, 1.0)
        loss, grad = pull_sums(recs, X, lq, masked=True)
        np.testing.assert_allclose(loss / pt, v_ref, rtol=1e-12)
        np.testing.assert_allclose(grad, g_ref, rtol=1e-10, atol=1e-12 * np.abs(g_ref).max())


def test_lane_slots_are_sorted_by_length_inside_a_class():
    rng = np.random.default_rng(5)
    n, m = 2000, 2
    edges, w = random_problem(rng, n, 30000, True, True)
    rc, lay = build(n, m, edges, w, True, 9)
    assert rc == 0
    recs = decode(lay, n, m)
    prev = None
    for tile, cls, W, own, cnt, dup, wv, nb in recs:
        real = cnt[~dup]
        if len(real) == 0:
            continue
        assert np.all(np.diff(real) <= 0), "longest lane-slots first"
        key = (tile, cls)
        if prev is not None and prev[0] == key:
            assert real[0] <= prev[1]
        prev = (key, real[-1])
    # padding overhead of the sorted packing stays small
    assert lay["npadded"] <= 1.35 * lay["nentries"]


def test_unsupported_shapes_are_refused():
    rng = np.random.default_rng(6)
    edges, w = random_problem(rng, 100, 300, False, False)
    assert build(100, 5, edges, w, False)[0] == _lib.MDE_E_UNSUPPORTED       # m > 4
    assert build(100, 2, edges, w, False, rb=14)[0] == _lib.MDE_E_UNSUPPORTED  # u16 byte offsets overflow
    big, wb = random_problem(rng, 9000, 2000, False, False)
    assert build(9000, 2, big, wb, False, rb=8)[0] == _lib.MDE_E_UNSUPPORTED  # more than 32 neighbour tiles


@pytest.mark.parametrize("pack", ["0", "1"])
def test_packing_switch_changes_the_records_not_the_sums(pack, monkeypatch):
    """MDE_B200_ELL_PACK=0 (one lane-slot per lane in every record, the A/B switch) holds the same entries."""
    monkeypatch.setenv("MDE_B200_ELL_PACK", pack)
    rng = np.random.default_rng(11)
    n, m = 1500, 2
    edges, w = random_problem(rng, n, 9000, True, False)
    rc, lay = build(n, m, edges, w, True, 8)
    assert rc == 0
    recs = decode(lay, n, m)
    X = rng.standard_normal((n, m))
    pt = len(edges)
    v_ref, g_ref = O.average_distortion(X, edges, O.FnSpec(O.P_QUADRATIC, w), True)
    loss, grad = pull_sums(recs, X, lambda d2, ww, cls: (ww * d2, 2.0 * ww / pt), masked=False)
    np.testing.assert_allclose(loss / pt, v_ref, rtol=1e-12)
    np.testing.assert_allclose(grad, g_ref, rtol=1e-10, atol=1e-12 * np.abs(g_ref).max())
    rec, off = lay["rec"], lay["rec_off"].astype(np.int64) * 16
    ks = {int(np.frombuffer(rec[o + 8:o + 12].tobytes(), dtype=np.int32)[0]) for o in off[:-1]}
    assert ks == {1} if pack == "0" else max(ks) > 1


def test_cta_ranges_are_cost_balanced_on_the_bench_workload():
    """The persistent grid gets contiguous record ranges of equal estimated cost (per record / per lane-slot row / per
    entry column instruction counts from the ncu source page, a tile load charged per bucket a range touches)."""
    import bench
    edges, w = bench.c2_edges(0)
    e = np.sort(edges, axis=1)
    rc, lay = build(bench.N_ITEMS, 2, e, w, True)
    assert rc == 0 and lay["ncta"] == 132          # one CTA per SM of an H100 SXM
    rec, off = lay["rec"], lay["rec_off"].astype(np.int64) * 16
    hdr = np.stack([np.frombuffer(rec[o:o + 16].tobytes(), dtype=np.int32) for o in off[:-1]])
    W, cls, K = hdr[:, 0], hdr[:, 1], hdr[:, 2]
    cost = 60 + K * (30 + W * np.where(cls == 1, 31, 23))
    cw, bw = lay["cta_wt0"], lay["bkt_wt0"]
    tot = []
    for c in range(lay["ncta"]):
        a, b = cw[c], cw[c + 1]
        tiles = 1 + int(np.sum((bw[1:-1] > a) & (bw[1:-1] < b)))
        tot.append(cost[a:b].sum() + 6000 * tiles if b > a else 0)
    tot = np.array(tot, dtype=np.float64)
    busy = tot[tot > 0]
    assert len(busy) >= 130                      # at most the tail CTAs stay empty
    assert busy.max() <= 1.12 * busy.mean(), (busy.max(), busy.mean())
    assert lay["npadded"] <= 1.15 * lay["nentries"]  # pads: 11 % at C2
