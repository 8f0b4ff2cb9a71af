"""Cost of embedding new points next to a sparse data matrix: the row-range sparse search (`mde_knn_csr_rows`) and
`embed_new_points` against the route before it (the full sparse search of the stacked matrix, sliced).

  python tools/new_points_sparse_times.py [--reps 3] [--n-old 100000 500000] [--max-full-n 100000]
                                          [--regression-only] [--base path/to/older/libmde_b200.so]

Data: seeded Zipf-column sparse blobs (ten topics; each row draws 24 columns from a global Zipf law and 24
from its topic's, values uniform in (0, 1]), d = 30 000, about 40 non-zeros per row.  n_old in --n-old, n_new in
{1 000, 10 000}, k in {15, 40, 100}.
Search: `knn_rows_device` on the new rows of the stacked matrix (new) against `knn_sparse_device` on all of it,
sliced (old), with the host stacking (`recipes._stacked_matrix`) and the upload (`_to_device_csr`) timed apart.
End to end: `embed_new_points` against the same call with the old route patched back in, at its default k (15),
under MDE_B200_DETERMINISTIC=1 with the same seed, so that the outputs can be compared bit for bit.  The old route is
only run where n_old <= --max-full-n (its n^2 search is what this removes).
Regression: the full `mde_knn_csr`, `mde_knn_csr_wide` and `mde_knn_csr_long` (k = 15, 40, 100) on 20 000 rows of the
same data, CUDA events around each call, median of --reg-reps after 2 warm-up calls; with `--base`, the same entries
of an older build of the library, alternating call by call, and whether the outputs agree.
Wall clock around calls that end in a device synchronise; every shape is warmed up before it is timed; medians of
--reps runs (one timed run of each full search).  Prints the GPU's name, power limit and maximum SM clock, then one
JSON object."""
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

D, PER_ROW, TOPICS = 30000, 48, 10  # 48 column draws per row: about 40 distinct


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()


def zipf_blobs(n, seed):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, D + 1) ** 1.1
    p /= p.sum()
    perms = np.stack([np.random.default_rng(1234 + t).permutation(D) for t in range(TOPICS)])  # a column order per topic
    topic = rng.integers(0, TOPICS, n)
    h = PER_ROW // 2
    glob = rng.choice(D, size=(n, h), p=p)
    local = perms[topic[:, None], rng.choice(D, size=(n, PER_ROW - h), p=p)]
    cols = np.concatenate([glob, local], 1).reshape(-1)
    rows = np.repeat(np.arange(n), PER_ROW)
    vals = (1.0 - rng.random(n * PER_ROW)).astype(np.float32)
    A = sp.csr_matrix((vals, (rows, cols)), shape=(n, D))
    A.sum_duplicates()
    return A


def _wall(fn, reps, warm=True):
    if warm:
        fn()  # warm-up of this shape
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def _full_entry(lib, k):
    name = "mde_knn_csr" if k <= 24 else "mde_knn_csr_wide" if k <= 64 else "mde_knn_csr_long"
    ws_fn, fn = getattr(lib, name + "_ws_bytes"), getattr(lib, name)
    ws_fn.argtypes = [C.c_int64, C.c_int, C.c_int64, C.POINTER(C.c_size_t)]
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_void_p,
                   C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    return name, ws_fn, fn


def regression(libs, reps):
    """Median ms of each full sparse search per library, alternating call by call; and whether the outputs agree."""
    from pymde_b200.preprocess import data_matrix as dm
    n = 20000
    (ip, ix, v), _ = dm._to_device_csr(zipf_blobs(n, 7), torch.device("cuda"))
    nnz = int(ix.shape[0])
    out = {}
    for k in (15, 40, 100):
        res, calls = {}, {}
        for tag, lib in libs.items():
            name, ws_fn, fn = _full_entry(lib, k)
            need = C.c_size_t(0)
            assert ws_fn(n, D, nnz, C.byref(need)) == 0
            ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
            p = ws.data_ptr() + (-ws.data_ptr()) % 1024
            idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
            d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
            calls[tag] = (fn, p, need.value, idx, d2, ws)
            res[tag] = []
        stream = torch.cuda.current_stream().cuda_stream

        def run(tag):
            fn, p, nb, idx, d2, _ = calls[tag]
            assert fn(ip.data_ptr(), ix.data_ptr(), v.data_ptr(), n, D, nnz, k, idx.data_ptr(), d2.data_ptr(), p, nb,
                      stream) == 0
        for _ in range(2):
            for tag in libs:
                run(tag)
        torch.cuda.synchronize()
        for _ in range(reps):
            for tag in libs:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                run(tag)
                b.record()
                b.synchronize()
                res[tag].append(a.elapsed_time(b))
        key = "%s_n%d_k%d" % (name, n, k)
        out[key] = {tag: round(float(np.median(t)), 3) for tag, t in res.items()}
        tags = list(libs)
        if len(tags) == 2:
            i0, d0 = calls[tags[0]][3], calls[tags[0]][4]
            i1, d1 = calls[tags[1]][3], calls[tags[1]][4]
            out[key]["same_bits"] = bool(torch.equal(i0, i1) and torch.equal(d0, d1))
        print(key, json.dumps(out[key]), flush=True)
        del calls
    return out


def search_and_end_to_end(n_olds, max_full_n, reps):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    from pymde_b200.preprocess import data_matrix as dm
    dev = torch.device("cuda")
    original = dm.knn_sparse_rows_device

    def full_then_slice(csr, shape, k, row_begin, row_end):  # the route before the row search
        idx, d2 = dm.knn_sparse_device(csr, shape, k)
        return idx[row_begin:row_end].contiguous(), d2[row_begin:row_end].contiguous()

    os.environ["MDE_B200_DETERMINISTIC"] = "1"
    out = {}
    for n_old in n_olds:
        data = zipf_blobs(n_old, 1)
        os.environ["PYMDE_B200_KNN_SPARSE"] = "approx"  # the fit is not timed: NN-descent keeps it affordable
        pm.seed(0)
        emb = pm.preserve_neighbors(data, embedding_dim=2).embed()
        del os.environ["PYMDE_B200_KNN_SPARSE"]
        full_too = n_old <= max_full_n
        for n_new in (1000, 10000):
            new = zipf_blobs(n_new, 2)
            key = "%dx%d+%d" % (n_old, D, n_new)
            r = {"nnz_per_row": round((data.nnz + new.nnz) / (n_old + n_new), 1)}
            r["host_stack_s"] = round(_wall(lambda: recipes._stacked_matrix(data, new, dev), reps), 4)
            S = recipes._stacked_matrix(data, new, dev)
            n = S.shape[0]
            r["upload_csr_s"] = round(_wall(lambda: dm._to_device_csr(S, dev), reps), 4)
            csr, shape = dm._to_device_csr(S, dev)
            for k in (15, 40, 100):
                rows_i, rows_d = dm.knn_sparse_rows_device(csr, shape, k, n_old, n)
                r["k%d_search_rows_s" % k] = round(_wall(lambda: dm.knn_sparse_rows_device(csr, shape, k, n_old, n),
                                                         reps, warm=False), 4)
                if full_too:
                    full_i, full_d = dm.knn_sparse_device(csr, shape, k)  # (also the warm-up)
                    r["k%d_rows_equal_full" % k] = bool(torch.equal(rows_i, full_i[n_old:]) and
                                                        torch.equal(rows_d, full_d[n_old:]))
                    del full_i, full_d
                    r["k%d_search_full_s" % k] = round(_wall(lambda: dm.knn_sparse_device(csr, shape, k), 1,
                                                             warm=False), 4)
                    r["k%d_ratio" % k] = round(r["k%d_search_rows_s" % k] / r["k%d_search_full_s" % k], 4)
                print(key, "k", k, json.dumps({kk: vv for kk, vv in r.items() if kk.startswith("k%d_" % k)}),
                      flush=True)
            del csr
            pm.seed(0)
            got = pm.embed_new_points(data, emb, new)

            def embed_new():
                pm.seed(0)
                return pm.embed_new_points(data, emb, new)
            r["embed_new_points_s"] = round(_wall(embed_new, reps), 3)
            if full_too:
                dm.knn_sparse_rows_device = full_then_slice
                try:
                    pm.seed(0)
                    want = pm.embed_new_points(data, emb, new)
                    r["embed_equal_old_route"] = bool(torch.equal(got, want))
                    r["embed_old_route_s"] = round(_wall(embed_new, 1, warm=False), 3)
                finally:
                    dm.knn_sparse_rows_device = original
            print(key, json.dumps(r), flush=True)
            out[key] = r
            torch.cuda.empty_cache()
        del data, emb
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reg-reps", type=int, default=5)
    ap.add_argument("--n-old", type=int, nargs="+", default=[100000, 500000])
    ap.add_argument("--max-full-n", type=int, default=100000)
    ap.add_argument("--regression-only", action="store_true")
    ap.add_argument("--base", default=None, help="an older libmde_b200.so to time the full searches against")
    args = ap.parse_args()
    gpu = _gpu()
    print(gpu, flush=True)
    from pymde_b200 import _lib
    libs = {"this": _lib.load()}
    if args.base:
        libs["base"] = C.CDLL(os.path.abspath(args.base))
    result = {"gpu": gpu, "regression_full_search_ms": regression(libs, args.reg_reps)}
    if not args.regression_only:
        result["new_points"] = search_and_end_to_end(args.n_old, args.max_full_n, args.reps)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
