"""Cost of embedding new points: the row-range exact search and `embed_new_points` against what the reference
workflow pays (a full search of the stacked matrix; `preserve_neighbors` on it with the fitted rows anchored).

  python tools/new_points_times.py [--reps 3] [--regression-only] [--base path/to/older/libmde_b200.so]

Search: n_old = 70 000 x 784 (ten Gaussian blobs) and 10^6 x 64, n_new = 1 000 and 10 000 rows from the same
distribution, k = 15; `knn_rows_device` on the new rows of the stacked matrix against `knn_device` on all of it.
End to end: `embed_new_points` against the reference workflow, wall clock around calls that end in a device
synchronise, on the same workloads (the fitted embedding is `preserve_neighbors(data).embed()`, not timed).
Regression: the full search alone (`mde_knn` at k = 15, `mde_knn_wide` at k = 40) at n = 5 000 and 70 000 (d = 784),
CUDA events around each call, median of 20 after 3 warm-up calls; with `--base`, the same entries of an older build
of the library, alternating call by call.  Every shape is warmed up before it is timed; medians of --reps runs.
Prints the GPU's name, power limit and maximum SM clock, then one JSON object."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()


def _blobs(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((10, d), generator=torch.Generator(device="cuda").manual_seed(99), device="cuda") * 2.0
    lab = torch.randint(0, 10, (n,), generator=g, device="cuda")
    return (c[lab] + torch.randn((n, d), generator=g, device="cuda")).contiguous()


def _wall(fn, reps):
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
    name = "mde_knn" if k <= 24 else "mde_knn_wide"
    ws_fn, fn = getattr(lib, name + "_ws_bytes"), getattr(lib, name)
    ws_fn.argtypes = [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]
    fn.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    return ws_fn, fn


def regression(libs, reps=20):
    """Median ms of the full search per library, alternating call by call; and whether the outputs agree."""
    out = {}
    for n in (5000, 70000):
        X = _blobs(n, 784, 7)
        for k in (15, 40):
            res, outs = {}, {}
            calls = {}
            for tag, lib in libs.items():
                ws_fn, fn = _full_entry(lib, k)
                need = C.c_size_t(0)
                assert ws_fn(n, 784, C.byref(need)) == 0
                ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
                p = ws.data_ptr() + (-ws.data_ptr()) % 1024
                idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
                d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
                calls[tag] = (fn, p, need.value, idx, d2, ws)
                res[tag] = []
            stream = torch.cuda.current_stream().cuda_stream

            def run(tag):
                fn, p, nb, idx, d2, _ = calls[tag]
                assert fn(X.data_ptr(), n, 784, k, idx.data_ptr(), d2.data_ptr(), p, nb, stream) == 0
            for _ in range(3):
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
            key = "n%d_k%d" % (n, k)
            out[key] = {tag: round(float(np.median(v)), 3) for tag, v in res.items()}
            tags = list(libs)
            if len(tags) == 2:
                i0, d0 = calls[tags[0]][3], calls[tags[0]][4]
                i1, d1 = calls[tags[1]][3], calls[tags[1]][4]
                out[key]["same_bits"] = bool(torch.equal(i0, i1) and torch.equal(d0, d1))
            del calls
    return out


def search_and_end_to_end(reps):
    import pymde_b200 as pm
    from pymde_b200.preprocess import data_matrix as dm
    out = {}
    for n_old, d in ((70000, 784), (10 ** 6, 64)):
        data = _blobs(n_old, d, 1)
        pm.seed(0)
        emb = pm.preserve_neighbors(data).embed()
        for n_new in (1000, 10000):
            new = _blobs(n_new, d, 2)
            X = torch.cat([data, new]).contiguous()
            n = X.shape[0]
            key = "%dx%d+%d" % (n_old, d, n_new)
            r = {}
            rows_i, rows_d = dm.knn_rows_device(X, 15, n_old, n)
            full_i, full_d = dm.knn_device(X, 15)
            r["rows_equal_full"] = bool(torch.equal(rows_i, full_i[n_old:]) and torch.equal(rows_d, full_d[n_old:]))
            del full_i, full_d
            r["search_rows_s"] = round(_wall(lambda: dm.knn_rows_device(X, 15, n_old, n), reps), 4)
            r["search_full_s"] = round(_wall(lambda: dm.knn_device(X, 15), reps), 4)
            r["embed_new_points_s"] = round(_wall(lambda: pm.embed_new_points(data, emb, new), reps), 3)
            anchors = torch.arange(n_old, device="cuda")
            r["reference_workflow_s"] = round(_wall(
                lambda: pm.preserve_neighbors(X, constraint=pm.Anchored(anchors, emb)).embed(), reps), 3)
            print(key, json.dumps(r), flush=True)
            out[key] = r
            del X, new
        del data, emb
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--regression-only", action="store_true")
    ap.add_argument("--base", default=None, help="an older libmde_b200.so to time the full search against")
    args = ap.parse_args()
    gpu = _gpu()
    print(gpu, flush=True)
    from pymde_b200 import _lib
    libs = {"this": _lib.load()}
    if args.base:
        libs["base"] = C.CDLL(os.path.abspath(args.base))
    result = {"gpu": gpu, "regression_full_search_ms": regression(libs)}
    print(json.dumps(result["regression_full_search_ms"]), flush=True)
    if not args.regression_only:
        result["new_points"] = search_and_end_to_end(args.reps)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
