"""The long row-range exact search (`mde_knn_long_rows`, `mde_knn16_long_rows`, `mde_knn8_long_rows`) against the GEMM
rows it replaces in `embed_new_points` at 64 < n_neighbors <= 256, and the full long searches against an older build.

  python tools/new_points_long_times.py [--reps 3] [--base path/to/older/libmde_b200.so] [--small] [--skip-large]

Row search: the new rows n_old .. n - 1 of a stacked matrix of ten Gaussian blobs (1 000 and 10 000 new rows) at
10^6 x 64 fp32 (k = 100, 256), 70 000 x 784 fp32 and uint8 (k = 100) and 2 10^6 x 1 024 uint8 (k = 100):
`data_matrix.knn_rows_device_long` against `data_matrix.knn_rows_device` (the GEMM rows: an fp32 copy, an fp64 centred
copy, fp64 score chunks), wall clock around calls that end in a device synchronise, median of --reps after a warm-up
call, peak device memory above the resident data of each call, and how the two lists compare: rows with the same
index lists, rows with the same distance bits.
End to end: `embed_new_points` at n_neighbors = 100 with 1 000 new rows, with the long row search and with the GEMM
rows forced, next to 70 000 x 784 uint8 and 10^6 x 64 fp32 (the fitted embedding is two columns of the data, not timed).
Regression: the full `mde_knn_long_ex` / `mde_knn16_long_ex` / `mde_knn8_long_ex` at k = 100 on 70 000 x 784 (and
20 000 x 784 at k = 256), CUDA events around each call, median of 9 after 2 warm-up calls; with --base the same
entries of an older build, alternating call by call, and whether the two give the same bits and fallback counts.
Prints the GPU's name, power limit and maximum SM clock, then one JSON object.  --small rehearses at 1/50 of every n
(the timings then say nothing); --skip-large leaves out the 2 10^6 x 1 024 shape."""
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


def _blobs(n, d, seed, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((10, d), generator=torch.Generator(device="cuda").manual_seed(99), device="cuda") * 2.0
    out = torch.empty((n, d), dtype=dtype, device="cuda")
    for s0 in range(0, n, 1 << 18):  # in chunks: a 2 10^6 x 1 024 uint8 matrix never exists in fp32
        m = min(n, s0 + (1 << 18)) - s0
        lab = torch.randint(0, 10, (m,), generator=g, device="cuda")
        x = c[lab] + torch.randn((m, d), generator=g, device="cuda")
        out[s0:s0 + m] = torch.clamp(torch.round(x * 16.0 + 128.0), 0, 255).to(dtype) if dtype == torch.uint8 else x
    return out


def _timed(fn, reps):
    """(median wall seconds, peak bytes allocated above what was allocated before, last result)."""
    res = fn()  # warm-up of this shape
    del res
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
        if _ < reps - 1:
            del res
    return float(np.median(ts)), torch.cuda.max_memory_allocated() - base, res


def _compare(a, b):
    """Rows whose index lists are identical, and rows whose distances are identical bit for bit (the GEMM rows sum
    the squared differences in torch's order, so on fp32 input their distances may differ in the last bits)."""
    same = (a[0].long() == b[0].long()).all(1)
    dist = (a[1] == b[1]).all(1)
    return {"rows_same_indices": int(same.sum()), "rows_same_distance_bits": int(dist.sum())}


def row_searches(reps, scale, large):
    from pymde_b200.preprocess import data_matrix as dm
    shapes = [(10 ** 6, 64, torch.float32, (100, 256)), (70000, 784, torch.float32, (100,)),
              (70000, 784, torch.uint8, (100,))]
    if large:
        shapes.append((2 * 10 ** 6, 1024, torch.uint8, (100,)))
    out = {}
    for n_old, d, dtype, ks in shapes:
        n_old = max(1000, n_old // scale)
        for n_new in (1000, 10000):
            n_new = max(100, n_new // scale)
            X = torch.cat([_blobs(n_old, d, 1, dtype), _blobs(n_new, d, 2, dtype)]).contiguous()
            n = X.shape[0]
            for k in ks:
                key = "%dx%d_%s+%d_k%d" % (n_old, d, str(dtype).split(".")[-1], n_new, k)
                r = {}
                t, m, a = _timed(lambda: dm.knn_rows_device_long(X, k, n_old, n), reps)
                r["long_rows_s"], r["long_rows_peak_mb"] = round(t, 4), round(m / 2 ** 20, 1)
                del a
                t, m, b = _timed(lambda: dm.knn_rows_device(X, k, n_old, n), reps)
                r["gemm_rows_s"], r["gemm_rows_peak_mb"] = round(t, 4), round(m / 2 ** 20, 1)
                a = dm.knn_rows_device_long(X, k, n_old, n)
                r.update(_compare(a, b))
                del a, b
                torch.cuda.empty_cache()
                print(key, json.dumps(r), flush=True)
                out[key] = r
            del X
            torch.cuda.empty_cache()
    return out


def end_to_end(reps, scale):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    from pymde_b200.preprocess import data_matrix as dm
    out = {}
    default = recipes._dense_new_lists
    routes = {"long_rows": lambda X, k, a, b: dm.knn_rows_device_long(X, k, a, b),
              "gemm_rows": lambda X, k, a, b: dm.knn_rows_device(X, k, a, b)}
    for n_old, d, dtype in ((70000, 784, torch.uint8), (10 ** 6, 64, torch.float32)):
        n_old = max(1000, n_old // scale)
        data = _blobs(n_old, d, 1, dtype)
        new = _blobs(max(100, 1000 // scale), d, 2, dtype)
        emb = data[:, :2].float().contiguous()
        key = "%dx%d_%s+%d" % (n_old, d, str(dtype).split(".")[-1], new.shape[0])
        r = {}
        for name, route in routes.items():
            recipes._dense_new_lists = route
            try:
                pm.seed(0)
                r["embed_new_points_%s_s" % name] = round(
                    _timed(lambda: pm.embed_new_points(data, emb, new, n_neighbors=100), reps)[0], 3)
            finally:
                recipes._dense_new_lists = default
        print(key, json.dumps(r), flush=True)
        out[key] = r
        del data, new, emb
        torch.cuda.empty_cache()
    return out


def _long_entry(lib, dtype):
    prefix = {torch.float32: "mde_knn", torch.float16: "mde_knn16", torch.uint8: "mde_knn8"}[dtype]
    ws_fn, fn = getattr(lib, prefix + "_long_ws_bytes"), getattr(lib, prefix + "_long_ex")
    ws_fn.argtypes = [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]
    lead = [C.c_void_p] if dtype == torch.float32 else [C.c_void_p, C.c_int]
    fn.argtypes = lead + [C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                          C.POINTER(C.c_int)]
    return ws_fn, fn


def regression(libs, scale, reps=9):
    from pymde_b200 import _lib
    out = {}
    codes = {torch.float16: _lib.DTYPE_FP16, torch.uint8: _lib.DTYPE_U8}
    for n, k in ((70000, 100), (20000, 256)):
        n = max(1000, n // scale)
        for dtype in (torch.float32, torch.float16, torch.uint8):
            X = _blobs(n, 784, 7, torch.uint8 if dtype == torch.uint8 else torch.float32).to(dtype).contiguous()
            lead = (X.data_ptr(),) if dtype == torch.float32 else (X.data_ptr(), codes[dtype])
            calls, res = {}, {}
            for tag, lib in libs.items():
                ws_fn, fn = _long_entry(lib, dtype)
                need = C.c_size_t(0)
                assert ws_fn(n, 784, C.byref(need)) == 0
                ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
                p = ws.data_ptr() + (-ws.data_ptr()) % 1024
                idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
                d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
                calls[tag] = (fn, p, need.value, idx, d2, ws, C.c_int(-1))
                res[tag] = []
            stream = torch.cuda.current_stream().cuda_stream

            def run(tag):
                fn, p, nb, idx, d2, _, fb = calls[tag]
                assert fn(*lead, n, 784, k, idx.data_ptr(), d2.data_ptr(), p, nb, stream, C.byref(fb)) == 0
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
            key = "%dx784_%s_k%d" % (n, str(dtype).split(".")[-1], k)
            out[key] = {tag: round(float(np.median(v)), 3) for tag, v in res.items()}
            out[key]["fallback_rows"] = {tag: calls[tag][6].value for tag in libs}
            tags = list(libs)
            if len(tags) == 2:
                c0, c1 = calls[tags[0]], calls[tags[1]]
                out[key]["same_bits"] = bool(torch.equal(c0[3], c1[3]) and torch.equal(c0[4], c1[4]))
            print(key, json.dumps(out[key]), flush=True)
            del calls, X
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--base", default=None, help="an older libmde_b200.so to time the full long searches against")
    ap.add_argument("--small", action="store_true", help="rehearse at 1/50 of every n")
    ap.add_argument("--skip-large", action="store_true", help="leave out 2 10^6 x 1 024 uint8")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the timings need a GPU"
    scale = 50 if args.small else 1
    gpu = _gpu()
    print(gpu, flush=True)
    from pymde_b200 import _lib
    libs = {"this": _lib.load()}
    if args.base:
        libs["base"] = C.CDLL(os.path.abspath(args.base))
    result = {"gpu": gpu}
    result["regression_full_long_ms"] = regression(libs, scale)
    result["row_search"] = row_searches(args.reps, scale, not args.skip_large)
    result["embed_new_points"] = end_to_end(args.reps, scale)
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
