"""mde_knn_approx (NN-descent) at 10^6 and 10^7 rows: wall time of the whole call (synchronised, best of `--reps`
after a warm-up on a small matrix), NN-descent iterations, peak device memory, recall@k on 4 096 sampled rows
against an fp64 brute force over all n rows (chunked GEMM), and at n <= 10^6 the exact mde_knn / mde_knn_wide on the
same matrix (the exact search is not run at 10^7: it scales as n^2 d).  At 10^7 it also times the host
`_knn_graph` (Graph.from_edges) on the result.  Data: a Gaussian mixture of `--intrinsic` dimensions embedded in d by
a random orthonormal map, plus noise of 1e-2 of the cluster spread; `--dtype fp16|bf16` casts it to that type, which
both searches read in place (mde_knn16_approx, mde_knn16*).  One JSON line per shape, with the GPU name, power limit
and max SM clock read in the same run.
Usage: python tools/knn_approx_check.py [--shapes 1e6x50x15,1e6x784x15,1e6x784x50,1e7x50x15,1e7x784x15] [--reps 3]
       [--dtype fp32|fp16|bf16]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pymde_b200 import _lib
from pymde_b200.preprocess import data_matrix as dm

dev = torch.device("cuda", 0)
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def gpu_identity():
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
        p, c = r.stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_clock_mhz"] = float(p), float(c)
    except Exception:
        pass
    return out


def mixture(n, d, intrinsic, seed, clusters=100, chunk=1 << 20, dtype=torch.float32):
    """Built in row chunks, so only X itself is n x d sized."""
    g = torch.Generator(device=dev).manual_seed(seed)
    centres = 4.0 * torch.randn((clusters, intrinsic), generator=g, device=dev)
    Q, _ = torch.linalg.qr(torch.randn((d, intrinsic), generator=g, device=dev))
    X = torch.empty((n, d), dtype=dtype, device=dev)
    for s0 in range(0, n, chunk):
        m = min(chunk, n - s0)
        lab = torch.randint(0, clusters, (m,), generator=g, device=dev)
        Z = centres[lab] + torch.randn((m, intrinsic), generator=g, device=dev)
        X[s0:s0 + m] = Z @ Q.T + 1e-2 * torch.randn((m, d), generator=g, device=dev)
    return X


def brute64(X, rows, k, chunk=1 << 17):
    """Indices of the k nearest rows (fp64 norm expansion over all n rows, in row chunks) of the sampled rows."""
    Q = X[rows].double()
    qn = (Q * Q).sum(1)
    best_v = torch.full((len(rows), k), float("inf"), dtype=torch.float64, device=dev)
    best_i = torch.zeros((len(rows), k), dtype=torch.int64, device=dev)
    for s0 in range(0, X.shape[0], chunk):
        Xc = X[s0:s0 + chunk].double()
        d2 = qn[:, None] + (Xc * Xc).sum(1)[None, :] - 2.0 * Q @ Xc.T
        self_col = rows - s0
        hit = (self_col >= 0) & (self_col < Xc.shape[0])
        d2[torch.nonzero(hit)[:, 0], self_col[hit]] = float("inf")
        v, i = torch.topk(d2, k, dim=1, largest=False)
        v = torch.cat([best_v, v], 1); i = torch.cat([best_i, i + s0], 1)
        best_v, pos = torch.topk(v, k, dim=1, largest=False)
        best_i = torch.gather(i, 1, pos)
        del d2, Xc
    return best_i


def approx(X, k, seed):
    lib = _lib.load()
    n, d = X.shape
    need = C.c_size_t(0)
    ws_bytes, _, args = dm._entries(lib, X, "_approx")
    _lib.check(ws_bytes(n, d, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    d2 = torch.empty((n, k), dtype=torch.float32, device=dev)
    it = C.c_int(0)
    search = getattr(lib, "mde_%s_approx_ex" % dm._SEARCH_DTYPES[X.dtype][0])
    _lib.check(search(*args, n, d, k, C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(),
                      ws.data_ptr() + (-ws.data_ptr()) % 1024, need.value, None, C.byref(it)))
    torch.cuda.synchronize()
    return idx, d2, need.value, it.value


def timed(fn, reps):
    ts = []
    out = None
    for _ in range(reps):
        del out
        torch.cuda.synchronize()
        t0 = time.perf_counter(); out = fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    return min(ts), ts, out


def run(n, d, k, reps, intrinsic, dtype, seed=0):
    lib = _lib.load()
    X = mixture(n, d, intrinsic, seed, dtype=DTYPES[dtype])
    torch.cuda.synchronize()
    rec = {"n": n, "d": d, "k": k, "dtype": dtype, "intrinsic_dim": intrinsic}
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    best, ts, (idx, d2, ws_bytes, iterations) = timed(lambda: approx(X, k, seed=1), reps)
    rec.update({"approx_s": best, "approx_all_s": ts, "iterations": iterations,
                "workspace_gb": ws_bytes / 1e9, "X_gb": X.numel() * X.element_size() / 1e9,
                "peak_device_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
                "peak_above_X_gb": (torch.cuda.max_memory_allocated(dev) - base) / 1e9})
    g = torch.Generator(device=dev).manual_seed(123)
    rows = torch.randperm(n, generator=g, device=dev)[:4096]
    ref = brute64(X, rows, k)
    got = idx[rows].long()
    hits = (torch.sort(got, 1)[0][:, :, None] == ref[:, None, :]).any(2).float().sum(1)
    rec["recall_4096"] = float(hits.mean()) / k
    rec["rows_all_found_4096"] = float((hits == k).float().mean())
    if n <= 10 ** 6:
        name = "mde_knn_s" if k <= lib.mde_knn_max_k() else "mde_knn_wide_s"
        torch.cuda.reset_peak_memory_stats(dev)
        ebest, ets, (ei, ed) = timed(lambda: dm.knn_device(X, k), min(reps, 2))
        rec["exact_peak_above_X_gb"] = (torch.cuda.max_memory_allocated(dev) - base) / 1e9
        rec.update({name: ebest, name.replace("_s", "_all_s"): ets, "speedup_vs_exact": ebest / best})
        same = (torch.sort(ei.long(), 1)[0] == torch.sort(idx.long(), 1)[0]).all(1)
        rec["rows_identical_to_exact"] = float(same.float().mean())
        rec["d2_ge_exact_everywhere"] = bool((d2 >= ed).all())
        rec["identical_rows_bit_identical_d2"] = bool(torch.equal(d2[same].view(torch.int32),
                                                                  ed[same].view(torch.int32)))
        del ei, ed
    else:
        rec["exact_search"] = "not run at this n"
        t0 = time.perf_counter()
        graph = dm._knn_graph(idx, d2, n, None, dev)
        rec["knn_graph_host_s"] = time.perf_counter() - t0
        rec["knn_graph_edges"] = int(graph.edges.shape[0])
        del graph
    rec.update(gpu_identity())
    print(json.dumps(rec), flush=True)
    del X, idx, d2
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1e6x50x15,1e6x784x15,1e6x784x50,1e7x50x15,1e7x784x15")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--intrinsic", type=int, default=16)
    ap.add_argument("--dtype", default="fp32", choices=sorted(DTYPES))
    a = ap.parse_args()
    # warm-up: module loads of both searches on a small matrix
    Xw = mixture(20000, 64, a.intrinsic, 99, dtype=DTYPES[a.dtype])
    for kw in (15, 50):
        approx(Xw, kw, 1); dm.knn_device(Xw, kw)
    del Xw
    for s in a.shapes.split(","):
        n, d, k = s.split("x")
        run(int(float(n)), int(d), int(k), a.reps, a.intrinsic, a.dtype)


if __name__ == "__main__":
    main()
