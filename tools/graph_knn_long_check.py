"""Graph k-nearest neighbours for 64 < k <= 256 on the device (`mde_graph_knn_long`, `mde_graph_knn_long_rows`).

  python tools/graph_knn_long_check.py [--reps 5] [--small]

  (a) the weighted geometric 8-NN graph of `graph_check.py` (n = 44 682, Euclidean weights of uniform points in the
      unit square) at k = 100 and 256 with `preserve_neighbors`' radius (3 times the 75th percentile of the edge
      lengths): `graph.k_nearest_neighbors_device_long` (the route the recipes take, CSR upload and graph assembly
      included) and the C call alone on a resident CSR; one run of the host row search (`graph.knn_rows_host` at
      k = 256: scipy's Dijkstra in the row chunks of the host `k_nearest_neighbors`, then the (length, index)
      selection); and whether the device lists equal the host lists, indices and fp32 lengths, bit for bit.
  (b) the same graph at k = 15 and 64: `mde_graph_knn_long` against `mde_graph_knn`, C calls alone on the same CSR
      and workspace, alternating call by call, and whether the lists are the same bits.
  (c) a 10^6-node weighted geometric 8-NN graph at k = 100: device only.
  (d) a unit-weight 10-community stochastic block model (10^5 nodes, about 6 edges per node inside its community and
      0.4 to uniform nodes) at k = 256 with the recipe radius (3 hops): the tie-heavy case, device time and the
      lists of 500 rows against the host row search.
  (e) `embed_new_points` with 1 000 new nodes next to the 10^6-node graph of (c) at n_neighbors = 100: the row search
      (`graph.knn_rows_device_long` on the union graph, upload included, as the recipe runs it) and the whole call,
      with a random fitted embedding (the fit is not part of the call).
Wall clock around calls that end in a device synchronise, after a warm-up call of the same shape; medians of --reps.
Prints the GPU's name, power limit and maximum SM clock, then one JSON object.  --small rehearses at small shapes."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()


def _sym(e, w, n):
    lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
    keep = lo != hi
    key, first = np.unique(lo[keep] * n + hi[keep], return_index=True)
    U = sp.coo_matrix((np.asarray(w, np.float32)[keep][first], (key // n, key % n)), shape=(n, n)).tocsr()
    return (U + U.T).tocsr()


def geometric(n, seed):
    from scipy.spatial import cKDTree
    pts = np.random.default_rng(seed).random((n, 2))
    _, idx = cKDTree(pts).query(pts, k=9)
    e = np.stack([np.repeat(np.arange(n), 8), idx[:, 1:].ravel()], 1)
    return _sym(e, np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1), n)


def sbm(n, seed, communities=10, d_in=6, d_out=0.4):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, communities, n)
    order = np.argsort(lab, kind="stable")
    start = np.searchsorted(lab[order], np.arange(communities))
    size = np.bincount(lab, minlength=communities)
    src = np.repeat(np.arange(n), d_in)
    c = lab[src]
    dst = order[start[c] + (rng.random(src.size) * size[c]).astype(np.int64)]
    e = np.concatenate([np.stack([src, dst], 1), rng.integers(0, n, (int(d_out * n), 2))])
    return _sym(e, np.ones(len(e)), n)


def split(A, n_old):
    from pymde_b200.preprocess import Graph
    U = sp.triu(A, k=1).tocoo()
    old = (U.row < n_old) & (U.col < n_old)
    e = np.stack([U.row, U.col], 1)
    return (Graph.from_edges(e[old], U.data[old], n_items=n_old),
            Graph.from_edges(e[~old], U.data[~old], n_items=A.shape[0]))


def radius(A):
    return float(3 * np.quantile(sp.triu(A).data, 0.75))


def _wall(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return round(float(np.median(ts)), 4)


class Resident:
    """The CSR of A on the device and one workspace for all n sources: the C searches alone."""

    def __init__(self, A):
        from pymde_b200 import _lib, util
        from pymde_b200.preprocess import graph as G
        self.lib, self.dev, self.n = _lib.load(), torch.device("cuda", 0), A.shape[0]
        self.indptr, self.indices, w = G._device_csr(A, self.dev)
        self.wptr = None if G._is_unweighted(A) else w.data_ptr()
        self.w = w
        self.ws = G._path_ws(self.lib.mde_graph_knn_ws_bytes, self.n, self.n, self.dev)
        self.stream = util.stream_ptr(self.dev)

    def run(self, k, md, long=True):
        from pymde_b200 import _lib
        idx = torch.empty((self.n, k), dtype=torch.int32, device=self.dev)
        ln = torch.empty((self.n, k), dtype=torch.float32, device=self.dev)
        fn = self.lib.mde_graph_knn_long if long else self.lib.mde_graph_knn
        _lib.check(fn(self.indptr.data_ptr(), self.indices.data_ptr(), self.wptr, self.n, k, md, idx.data_ptr(),
                      ln.data_ptr(), self.ws.data_ptr(), self.ws.numel(), self.stream))
        return idx, ln


def _equal(dev, host):
    i, l = dev
    hi, hl = host
    return bool(np.array_equal(i.cpu().numpy(), hi) and
                np.array_equal(l.cpu().numpy().view(np.int32), hl.astype(np.float32).view(np.int32)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    import pymde_b200 as pm
    from pymde_b200.preprocess import graph as G
    print(_gpu(), flush=True)
    n_a, n_c, n_d, n_new = (3000, 20000, 5000, 100) if a.small else (44682, 10 ** 6, 10 ** 5, 1000)
    out = {"gpu": _gpu()}

    A = geometric(n_a, 0)
    g, md = G.Graph(A), radius(A)
    t0 = time.perf_counter()
    host = G.knn_rows_host(g, 256, 0, n_a, max_distance=md)
    out["a_host_row_search_k256_s"] = round(time.perf_counter() - t0, 2)
    res = Resident(A)
    for k in (100, 256):
        out["a_k%d_builder_s" % k] = _wall(lambda: G.k_nearest_neighbors_device_long(g, k, max_distance=md), a.reps)
        out["a_k%d_call_s" % k] = _wall(lambda: res.run(k, md), a.reps)
        out["a_k%d_equals_host" % k] = _equal(res.run(k, md), (host[0][:, :k], host[1][:, :k]))
    print("(a)", json.dumps({k: v for k, v in out.items() if k.startswith("a_")}), flush=True)

    for k in (15, 64):
        res.run(k, md), res.run(k, md, long=False)
        ts = {"long": [], "short": []}
        for _ in range(a.reps):
            for tag in ts:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res.run(k, md, long=tag == "long")
                torch.cuda.synchronize()
                ts[tag].append(time.perf_counter() - t0)
        x, y = res.run(k, md), res.run(k, md, long=False)
        out["b_k%d" % k] = {"mde_graph_knn_long_s": round(float(np.median(ts["long"])), 4),
                            "mde_graph_knn_s": round(float(np.median(ts["short"])), 4),
                            "same_bits": bool(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]))}
        print("(b)", k, json.dumps(out["b_k%d" % k]), flush=True)
    del res
    torch.cuda.empty_cache()

    A = geometric(n_c, 2)
    g, md = G.Graph(A), radius(A)
    out["c_k100_builder_s"] = _wall(lambda: G.k_nearest_neighbors_device_long(g, 100, max_distance=md), a.reps)
    res = Resident(A)
    out["c_k100_call_s"] = _wall(lambda: res.run(100, md), a.reps)
    out["c_batch"] = int(res.ws.numel() // (int(res.lib.mde_graph_knn_ws_bytes(n_c, 64)) -
                                            int(res.lib.mde_graph_knn_ws_bytes(n_c, 32))) * 32)
    print("(c)", json.dumps({k: v for k, v in out.items() if k.startswith("c_")}), flush=True)
    del res
    torch.cuda.empty_cache()

    S = sbm(n_d, 3)
    md_s = radius(S)
    res = Resident(S)
    out["d_k256_call_s"] = _wall(lambda: res.run(256, md_s), a.reps)
    rows = np.random.default_rng(0).choice(n_d, 500, replace=False)
    idx, ln = res.run(256, md_s)
    sub = [G.knn_rows_host(S, 256, int(r), int(r) + 1, max_distance=md_s) for r in rows]
    pick = torch.as_tensor(rows, device=idx.device)
    out["d_k256_500_rows_equal_host"] = _equal((idx[pick], ln[pick]), (np.concatenate([s[0] for s in sub]),
                                                                        np.concatenate([s[1] for s in sub])))
    # per row, the entries of the 256-list at the 256-th length (the tied nodes the list could not all hold)
    out["d_mean_list_entries_at_kth_length"] = round(float(np.mean([(s[1][0] == s[1][0, -1]).sum() for s in sub])), 1)
    print("(d)", json.dumps({k: v for k, v in out.items() if k.startswith("d_")}), flush=True)
    del res
    torch.cuda.empty_cache()

    n_old = n_c - n_new
    data, new = split(A, n_old)
    emb = torch.randn((n_old, 2), device="cuda")
    from pymde_b200 import recipes
    union = recipes._union_graph(data, new)
    md_u = float(3 * torch.quantile(torch.cat([data.distances, new.distances]), 0.75))
    out["e_row_search_s"] = _wall(lambda: G.knn_rows_device_long(union, 100, n_old, n_c, max_distance=md_u), a.reps)

    def call():
        pm.seed(0)
        return pm.embed_new_points(data, emb, new, n_neighbors=100)

    out["e_embed_new_points_s"] = _wall(call, a.reps)
    print("(e)", json.dumps({k: v for k, v in out.items() if k.startswith("e_")}), flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
