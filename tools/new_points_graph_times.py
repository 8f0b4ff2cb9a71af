"""Cost of embedding new nodes next to a graph's embedding: the row-range graph search (`mde_graph_knn_rows`) and
`embed_new_points` on Graphs, against the full search and the reference workflow.

  python tools/new_points_graph_times.py [--reps 3] [--n-old 1000000] [--n-new 1000 10000] [--host-max 1000]
                                         [--graphs geometric,unweighted,sbm] [--base path/to/older/libmde_b200.so]
                                         [--reg-reps 7]

Graphs (seeded, n = n_old + n_new nodes; the last n_new are the new ones): the weighted geometric 8-NN graph of
`graph_check.py` (Euclidean weights of uniform points in the unit square), the same graph with unit weights, and a
10-community stochastic block model (about 6 edges per node inside its community and 0.4 to uniform nodes, unit
weights).  The fitted graph holds the edges between fitted nodes, the new graph every edge touching a new node.
k = 15, max_distance = the recipe's default (3 times the 75th percentile of the union's edge lengths).
Search: `graph.knn_rows_device` on rows [n_old, n) of the union (the CSR upload included, as the recipe runs it)
against `mde_graph_knn` on all n rows (the same upload), with the rows compared for equality; the host row search
(`graph.knn_rows_host`, scipy's Dijkstra) where n_new <= --host-max; peak device memory of each device search; and
the two C calls alone, with the CSR already on the device (`*_engine_s`, with the batch each workspace gives).
End to end: `embed_new_points` against the reference workflow, `preserve_neighbors` on the union graph with every
fitted node anchored, then `embed()`, each with its peak device memory.  The reference workflow runs with
init="random": its default spectral initialisation does not converge on the device for the 10^6-node geometric
graphs and is recomputed on the host, which would dominate the time, so its time here is a lower bound.  The fit
(`preserve_neighbors(fitted graph, init="random").embed()`) is not timed.
Regression (`--base`): `mde_graph_knn` of this build and of an older one on the two `graph_check.py` k-NN shapes
(44 682 and 10^6 nodes), alternating call by call, medians of --reg-reps, and whether the outputs are the same bits.
Wall clock around calls that end in a device synchronise, after a warm-up call of the same shape; medians of --reps
(one run of each reference workflow and host search).  Prints the GPU's name, power limit and maximum SM clock,
then one JSON object."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

K = 15


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()


def _sym(e, w, n):
    lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
    keep = lo != hi
    key, first = np.unique(lo[keep] * n + hi[keep], return_index=True)
    U = sp.coo_matrix((np.asarray(w, np.float32)[keep][first], (key // n, key % n)), shape=(n, n)).tocsr()
    return (U + U.T).tocsr()


def geometric(n, seed, weighted=True):
    from scipy.spatial import cKDTree
    pts = np.random.default_rng(seed).random((n, 2))
    _, idx = cKDTree(pts).query(pts, k=9)
    e = np.stack([np.repeat(np.arange(n), 8), idx[:, 1:].ravel()], 1)
    w = np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1) if weighted else np.ones(len(e))
    return _sym(e, w, n)


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


def _wall(fn, reps, warm=True):
    if warm:
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)


def full_search(lib, A, k, md, batch_rows=None):
    """(idx [n, k], len [n, k]) of `mde_graph_knn` through `lib`, with the CSR upload and the recipe's workspace."""
    from pymde_b200 import util
    from pymde_b200.preprocess import graph as G
    dev = torch.device("cuda", 0)
    n = A.shape[0]
    indptr, indices, w = G._device_csr(A, dev)
    wptr = None if G._is_unweighted(A) else w.data_ptr()
    ws = G._path_ws(lambda nn, b: lib.mde_graph_knn_ws_bytes(nn, b), n, batch_rows or n, dev)
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    ln = torch.empty((n, k), dtype=torch.float32, device=dev)
    code = lib.mde_graph_knn(indptr.data_ptr(), indices.data_ptr(), wptr, n, k, md, idx.data_ptr(), ln.data_ptr(),
                             ws.data_ptr(), ws.numel(), util.stream_ptr(dev))
    assert code == 0, code
    return idx, ln


def engine_only(lib, A, k, md, n_old, reps):
    """Seconds of the two C calls alone, the CSR already on the device and both workspaces allocated: what the
    search costs apart from the O(nnz) preparation and upload the two routes share."""
    from pymde_b200 import util
    from pymde_b200.preprocess import graph as G
    dev = torch.device("cuda", 0)
    n = A.shape[0]
    indptr, indices, w = G._device_csr(A, dev)
    wptr = None if G._is_unweighted(A) else w.data_ptr()
    out = {}
    for tag, s0, nsrc in (("rows", n_old, n - n_old), ("full", 0, n)):
        ws = G._path_ws(lib.mde_graph_knn_ws_bytes, n, nsrc, dev)
        idx = torch.empty((nsrc, k), dtype=torch.int32, device=dev)
        ln = torch.empty((nsrc, k), dtype=torch.float32, device=dev)
        if tag == "rows":
            call = lambda: lib.mde_graph_knn_rows(indptr.data_ptr(), indices.data_ptr(), wptr, n, s0, n, k, md,
                                                  idx.data_ptr(), ln.data_ptr(), ws.data_ptr(), ws.numel(),
                                                  util.stream_ptr(dev))
        else:
            call = lambda: lib.mde_graph_knn(indptr.data_ptr(), indices.data_ptr(), wptr, n, k, md, idx.data_ptr(),
                                             ln.data_ptr(), ws.data_ptr(), ws.numel(), util.stream_ptr(dev))
        out["%s_engine_s" % tag] = round(_wall(call, reps if tag == "rows" else 1), 4)
        out["%s_batch" % tag] = int(ws.numel() // max(1, int(lib.mde_graph_knn_ws_bytes(n, 64)) -
                                                      int(lib.mde_graph_knn_ws_bytes(n, 32))) * 32)
        del ws, idx, ln
        torch.cuda.empty_cache()
    return out


def _bind(lib):
    lib.mde_graph_knn_ws_bytes.restype = C.c_int64
    lib.mde_graph_knn_ws_bytes.argtypes = [C.c_int64, C.c_int]
    lib.mde_graph_knn.restype = C.c_int
    lib.mde_graph_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_double, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def regression(base_path, reps):
    """Median seconds of `mde_graph_knn` per library, alternating call by call, and whether the outputs agree."""
    from pymde_b200 import _lib
    libs = {"base": _bind(C.CDLL(os.path.abspath(base_path))), "this": _lib.load()}
    out = {}
    for name, A in (("geometric_44682", geometric(44682, 0)), ("geometric_1e6", geometric(10 ** 6, 2))):
        md = float(3 * np.quantile(sp.triu(A).data, 0.75))
        res = {t: [] for t in libs}
        outs = {}
        for t, lib in libs.items():
            outs[t] = full_search(lib, A, K, md)  # (warm-up)
        for _ in range(reps):
            for t, lib in libs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                full_search(lib, A, K, md)
                torch.cuda.synchronize()
                res[t].append(time.perf_counter() - t0)
        r = {t: round(float(np.median(v)), 4) for t, v in res.items()}
        r["same_bits"] = bool(torch.equal(outs["base"][0], outs["this"][0]) and
                              torch.equal(outs["base"][1], outs["this"][1]))
        print("regression", name, json.dumps(r), flush=True)
        out[name] = r
        del outs
        torch.cuda.empty_cache()
    return out


def run(graphs, n_old, n_news, host_max, reps):
    import pymde_b200 as pm
    from pymde_b200 import _lib, recipes
    from pymde_b200.preprocess import graph as G
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    out = {}
    for gname in graphs:
        n_max = n_old + max(n_news)
        A_max = {"geometric": lambda: geometric(n_max, 2), "unweighted": lambda: geometric(n_max, 2, False),
                 "sbm": lambda: sbm(n_max, 3)}[gname]()
        fitted = A_max[:n_old, :n_old].tocsr()
        data = G.Graph(fitted)
        pm.seed(0)
        emb = pm.preserve_neighbors(data, init="random").embed()  # (not timed)
        print("%s_%d fitted" % (gname, n_old), flush=True)
        for n_new in n_news:
            n = n_old + n_new
            A = A_max[:n, :n].tocsr()
            _, new = split(A, n_old)
            key = "%s_%d+%d" % (gname, n_old, n_new)
            union = recipes._union_graph(data, new)
            md = float(3 * torch.quantile(torch.cat([data.distances, new.distances]), 0.75))
            r = {"nnz": int(union.nnz), "max_distance": round(md, 6)}
            (rows_i, rows_l), r["rows_peak_gib"] = _peak(
                lambda: G.knn_rows_device(union, K, n_old, n, max_distance=md, device=dev))
            r["rows_s"] = round(_wall(lambda: G.knn_rows_device(union, K, n_old, n, max_distance=md, device=dev),
                                      reps, warm=False), 4)
            (full_i, full_l), r["full_peak_gib"] = _peak(lambda: full_search(lib, union, K, md))
            r["rows_equal_full"] = bool(torch.equal(rows_i, full_i[n_old:]) and torch.equal(rows_l, full_l[n_old:]))
            del full_i, full_l
            r["full_s"] = round(_wall(lambda: full_search(lib, union, K, md), 1, warm=False), 4)
            r["ratio"] = round(r["rows_s"] / r["full_s"], 4)
            r.update(engine_only(lib, union, K, md, n_old, reps))
            if n_new <= host_max:
                t0 = time.perf_counter()
                hi, hl = G.knn_rows_host(union, K, n_old, n, max_distance=md)
                r["host_rows_s"] = round(time.perf_counter() - t0, 3)
                r["host_equal_device"] = bool(np.array_equal(hi, rows_i.cpu().numpy()) and
                                              np.array_equal(hl, rows_l.cpu().numpy()))
            print(key, "search", json.dumps(r), flush=True)

            def ours():
                pm.seed(0)
                return pm.embed_new_points(data, emb, new)
            _, r["embed_new_points_peak_gib"] = _peak(ours)
            r["embed_new_points_s"] = round(_wall(ours, reps, warm=False), 3)

            def reference():
                pm.seed(0)
                anchored = pm.Anchored(torch.arange(n_old, device=dev), emb)
                return pm.preserve_neighbors(G.Graph(union), constraint=anchored, init="random").embed()
            t0 = time.perf_counter()
            _, r["reference_peak_gib"] = _peak(reference)
            r["reference_s"] = round(time.perf_counter() - t0, 3)
            print(key, json.dumps(r), flush=True)
            out[key] = r
            torch.cuda.empty_cache()
        del data, emb, A_max
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n-old", type=int, default=10 ** 6)
    ap.add_argument("--n-new", type=int, nargs="+", default=[1000, 10000])
    ap.add_argument("--host-max", type=int, default=1000)
    ap.add_argument("--graphs", default="geometric,unweighted,sbm")
    ap.add_argument("--base", default=None)
    ap.add_argument("--reg-reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool measures the GPU"
    print(_gpu(), flush=True)
    res = {"gpu": _gpu(), "reps": args.reps}
    if args.base:
        res["regression"] = regression(args.base, args.reg_reps)
    res["new_points"] = run(args.graphs.split(","), args.n_old, args.n_new, args.host_max, args.reps)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
