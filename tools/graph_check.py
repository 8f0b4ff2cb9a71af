"""Weighted shortest paths (mde_graph_sssp) and graph k-NN (mde_graph_knn) at recipe sizes: device time, host-path
time on the same shape, and a parity check against scipy's Dijkstra.  One JSON line per shape, each with the GPU
name and power limit read in the same run.

  (a) weighted geometric 8-NN graph, n = 44 682: shortest paths retaining 5e7 pairs (preserve_distances' default)
  (b) the same graph: k-NN, k = 15, max_distance = 3 x the 75th percentile of the edge weights (preserve_neighbors)
  (c) k-NN, k = 15, on a 1e6-node weighted geometric graph: device only (the host path is quadratic in n)

Device time: host clock around a call that ends in a synchronise, after a warm-up call, best of 3.  Host time: one
run of the host path (graph.shortest_paths / graph.k_nearest_neighbors) on this machine's CPU.

Usage: python tools/graph_check.py [--shapes abc] [--no-host-a]   (the host arm of (a) takes many minutes)"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, scipy.sparse as sp, scipy.sparse.csgraph as csgraph, torch
from pymde_b200 import _lib, util
from pymde_b200.preprocess import graph as G

dev = torch.device("cuda", 0)
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=10)
        out["power_limit_w"] = float(r.stdout.strip())
    except Exception:
        pass
    return out


def geometric(n, k, seed):
    from scipy.spatial import cKDTree
    pts = np.random.default_rng(seed).random((n, 2))
    _, idx = cKDTree(pts).query(pts, k=k + 1)
    e = np.unique(np.sort(np.stack([np.repeat(np.arange(n), k), idx[:, 1:].ravel()], 1), axis=1), axis=0)
    w = np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1).astype(np.float32)
    U = sp.coo_matrix((w, (e[:, 0], e[:, 1])), shape=(n, n)).tocsr()
    return G.Graph((U + U.T).tocsr())


def splitmix64(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def device_time(fn):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(3):
        t0 = time.perf_counter(); out = fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    return min(ts), out


def host_time(fn):
    t0 = time.perf_counter(); out = fn(); return time.perf_counter() - t0, out


def knn_raw(g, k, max_distance):
    """Per-row (index, length) arrays straight from mde_graph_knn."""
    lib = _lib.load()
    A = g.adjacency_matrix
    n = A.shape[0]
    indptr, indices, w = G._device_csr(A, dev)
    ws = G._path_ws(lib.mde_graph_knn_ws_bytes, n, n, dev)
    idx = torch.empty(n * k, dtype=torch.int32, device=dev)
    ln = torch.empty(n * k, dtype=torch.float32, device=dev)
    _lib.check(lib.mde_graph_knn(indptr.data_ptr(), indices.data_ptr(), w.data_ptr(), n, k, float(max_distance),
                                 idx.data_ptr(), ln.data_ptr(), ws.data_ptr(), ws.numel(), util.stream_ptr(dev)))
    return idx.view(n, k).cpu().numpy(), ln.view(n, k).cpu().numpy()


def knn_parity_rows(g, k, max_distance, rows):
    got_i, got_l = knn_raw(g, k, max_distance)
    D = csgraph.dijkstra(g.adjacency_matrix, directed=False, indices=rows, limit=max_distance)
    D[np.arange(len(rows)), rows] = np.inf
    order = np.argsort(D, axis=1, kind="stable")[:, :k]
    d = np.take_along_axis(D, order, 1)
    want_i = np.where(np.isfinite(d), order, -1)
    return bool(np.array_equal(got_i[rows], want_i) and np.array_equal(got_l[rows], d.astype(np.float32)))


def shape_a(g, host):
    n = g.n_items
    retain = 5e7 / (n * (n - 1) / 2)
    seed = 12345
    t, out = device_time(lambda: G.shortest_paths_device(g, retain_fraction=retain, device=dev, seed=seed))
    rec = {"shape": "a: shortest paths, retain 5e7 pairs", "n": n, "nnz": int(g.adjacency_matrix.nnz),
           "retain_fraction": retain, "pairs": out.n_edges, "device_s": t}
    # parity on 64 sources: the device's triples for s equal {v > s reachable, kept by the hash} with scipy's lengths
    rows = np.sort(np.random.default_rng(0).choice(n, 64, replace=False))
    D = csgraph.dijkstra(g.adjacency_matrix, directed=False, indices=rows)
    e, ln = out.edges.cpu().numpy(), out.distances.cpu().numpy()
    ok = True
    for r, s in enumerate(rows):
        v = np.arange(s + 1, n)
        d = D[r, s + 1:]
        keep = np.isfinite(d) & (splitmix64(np.uint64(seed) ^ (np.uint64(s) * np.uint64(n) + v.astype(np.uint64)))
                                 < np.uint64(int(retain * 2.0 ** 64)))
        sel = e[:, 0] == s
        ok &= bool(np.array_equal(e[sel, 1], v[keep]) and np.array_equal(ln[sel], d[keep].astype(np.float32)))
    rec["parity_rows_checked"] = 64
    rec["parity"] = ok
    if host:
        th, hg = host_time(lambda: G.shortest_paths(g, retain_fraction=retain))
        rec["host_s"] = th
        rec["host_pairs"] = hg.n_edges
        rec["host_note"] = "one run of graph.shortest_paths on this machine's CPU"
    else:
        rec["host_s"] = None
    return rec


def shape_b(g):
    n = g.n_items
    maxd = 3 * float(torch.quantile(g.distances, 0.75))
    t, out = device_time(lambda: G.k_nearest_neighbors_device(g, 15, max_distance=maxd, device=dev))
    th, host = host_time(lambda: G.k_nearest_neighbors(g, 15, max_distance=maxd))
    parity = bool(torch.equal(out.edges.cpu(), host.edges) and torch.equal(out.weights.cpu(), host.weights))
    return {"shape": "b: graph k-NN, k = 15", "n": n, "max_distance": maxd, "edges": out.n_edges, "device_s": t,
            "host_s": th, "host_note": "one run of graph.k_nearest_neighbors on this machine's CPU",
            "parity": parity, "parity_kind": "edges and weights equal to the host path"}


def shape_c():
    n = 1_000_000
    g = geometric(n, 8, 2)
    maxd = 3 * float(torch.quantile(g.distances, 0.75))
    t, out = device_time(lambda: G.k_nearest_neighbors_device(g, 15, max_distance=maxd, device=dev))
    rows = np.sort(np.random.default_rng(1).choice(n, 32, replace=False))
    return {"shape": "c: graph k-NN, k = 15", "n": n, "nnz": int(g.adjacency_matrix.nnz), "max_distance": maxd,
            "edges": out.n_edges, "device_s": t, "host_s": None,
            "host_note": "not run: the host path builds a dense chunk x n matrix per chunk (quadratic in n)",
            "parity": knn_parity_rows(g, 15, maxd, rows), "parity_rows_checked": 32}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="abc")
    ap.add_argument("--no-host-a", action="store_true")
    args = ap.parse_args()
    gpu = gpu_identity()
    g = geometric(44_682, 8, 0) if ("a" in args.shapes or "b" in args.shapes) else None
    for s in args.shapes:
        rec = {"a": lambda: shape_a(g, not args.no_host_a), "b": lambda: shape_b(g), "c": shape_c}[s]()
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
