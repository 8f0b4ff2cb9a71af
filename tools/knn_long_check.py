"""Exact k-NN for 64 < k <= 256 (mde_knn_long, mde_knn_csr_long) at realistic sizes, in one run: synchronised wall
time of the whole call (preparation included), peak device memory, and parity on sampled rows against an fp64 brute
force.  Synthetic data only; one JSON line per measurement, each with the GPU name, power limit and max SM clock read
in the same run.

  dense   70 000 x 784 MNIST-like at k = 65, 128, 256: mde_knn_long against the chunked GEMM + top-k path it
          replaces, and against mde_knn_wide at k = 64 (best of 3 after a warm-up)
  (b)     the same matrix as CSR (DESIGN section 11.1) at k = 65 and 256 (best of 3 after a warm-up)
  (a)     text-like 3e5 x 1e5 (120 GB dense) at k = 100, one run

`--dtype fp16|bf16` casts the dense matrix to that type, which mde_knn16_long (and mde_knn16_wide at k = 64) read in
place; the GEMM path and the parity check work on its fp32 upcast.  Dense lines also carry the peak device memory of
the search above the input.

Usage: python tools/knn_long_check.py [--parts dense,b,a] [--rows 4096] [--dtype fp32|fp16|bf16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pymde_b200 import _lib  # noqa: E402
from pymde_b200.preprocess import data_matrix as dm  # noqa: E402
from tools.knn_sparse_check import host_brute, mnist_like, text_like, timed  # noqa: E402

dev = torch.device("cuda", 0)
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
        p, c = r.stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_clock_mhz"] = float(p), float(c)
    except Exception:
        pass
    return out


def emit(line):
    line.update(gpu_identity())
    print(json.dumps(line), flush=True)


def gemm_topk(X, k):
    """The path the long search replaces: `_search` with PYMDE_B200_KNN=gemm."""
    os.environ["PYMDE_B200_KNN"] = "gemm"
    try:
        return dm._search(X, k, dev)[:2]
    finally:
        del os.environ["PYMDE_B200_KNN"]


def dense_parity(X, idx, d2, rows):
    """Against an fp64 brute force on the sampled rows: identical neighbour sets where the k-th neighbour is clear of
    the (k+1)-th by more than fp32 rounding, and the largest relative gap between the returned distances and the k
    smallest exact ones."""
    k = idx.shape[1]
    Xd = X.double()
    out = {"rows": len(rows), "same_sets": 0, "clear_rows": 0, "max_rel_d2": 0.0}
    for s0 in range(0, len(rows), 256):
        r = torch.as_tensor(rows[s0:s0 + 256], device=dev)
        q = Xd[r]
        D = (q * q).sum(1)[:, None] + (Xd * Xd).sum(1)[None, :] - 2.0 * q @ Xd.T
        D[torch.arange(len(r), device=dev), r] = float("inf")
        cand = torch.topk(D, k + 9, dim=1, largest=False)[1]
        ex = ((q[:, None, :] - Xd[cand]) ** 2).sum(-1)
        val, pos = torch.sort(ex, 1)
        ref = torch.gather(cand, 1, pos)[:, :k]
        clear = (val[:, k] - val[:, k - 1]) > 4e-6 * val[:, k].abs() + 1e-9
        got = idx[r].long()
        same = (torch.sort(got, 1)[0] == torch.sort(ref, 1)[0]).all(1)
        gd = ((q[:, None, :] - Xd[got]) ** 2).sum(-1)
        out["same_sets"] += int(same.sum())
        out["clear_rows"] += int(clear.sum())
        out["same_sets_of_clear_rows"] = out.get("same_sets_of_clear_rows", 0) + int((same & clear).sum())
        rel = ((gd - val[:, :k]).abs() / val[:, :k].clamp(min=1e-30)).max()
        out["max_rel_d2"] = max(out["max_rel_d2"], float(rel))
    return out


def peak_above(fn):
    """Peak device memory allocated by fn() above what was allocated before it, in bytes."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    out = fn()
    torch.cuda.synchronize()
    del out
    return torch.cuda.max_memory_allocated(dev) - base


def run_dense(n_rows, dtype):
    Xn = mnist_like()
    X = torch.from_numpy(Xn).to(dev).to(DTYPES[dtype])
    rows = np.random.default_rng(1).choice(X.shape[0], n_rows, replace=False)
    w = torch.from_numpy(mnist_like(4096, seed=3)).to(dev).to(DTYPES[dtype])
    for k in (64, 65, 256):  # warm-up: module loads and the GEMM path's algorithm choice
        dm.knn_device(w, k)
        gemm_topk(w, k)
    res = {}
    t = timed(lambda: res.__setitem__("w", dm.knn_device(X, 64)))
    emit({"part": "dense", "n": 70000, "d": 784, "k": 64, "dtype": dtype, "kernel": "mde_knn_wide",
          "search_s": round(t, 4), "timing": "best of 3 after a warm-up",
          "peak_above_input_bytes": peak_above(lambda: dm.knn_device(X, 64))})
    del res["w"]
    for k in (65, 128, 256):
        t_long = timed(lambda: res.__setitem__("long", dm.knn_device(X, k)))
        t_gemm = timed(lambda: res.__setitem__("gemm", gemm_topk(X, k)))
        del res["gemm"]
        idx, d2 = res.pop("long")
        line = {"part": "dense", "n": 70000, "d": 784, "k": k, "dtype": dtype, "kernel": "mde_knn_long",
                "search_s": round(t_long, 4), "gemm_topk_s": round(t_gemm, 4), "timing": "best of 3 after a warm-up",
                "peak_above_input_bytes": peak_above(lambda: dm.knn_device(X, k))}
        line.update({"parity_" + a: b for a, b in dense_parity(X.float(), idx, d2, rows).items()})
        emit(line)
        del idx, d2
    torch.cuda.empty_cache()


def run_sparse(name, A, ks, reps, n_rows):
    n, d = A.shape
    csr, shape = dm._to_device_csr(A, dev)
    rows = np.random.default_rng(1).choice(n, n_rows, replace=False)
    bi, bd = host_brute(A, rows, max(ks))
    for k in ks:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        res = {}

        def go():
            res["out"] = dm.knn_sparse_device(csr, shape, k)
        if reps > 1:
            t = timed(go, reps)
        else:
            t0 = time.perf_counter()
            go()
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated(dev)
        idx, d2 = (x.cpu().numpy() for x in res.pop("out"))
        ulp = np.abs(d2[rows].view(np.int32).astype(np.int64) - bd[:, :k].view(np.int32).astype(np.int64))
        emit({"part": name, "n": n, "d": d, "nnz": int(A.nnz), "k": k, "kernel": "mde_knn_csr_long",
              "search_s": round(t, 4),
              "timing": "best of %d after a warm-up" % reps if reps > 1 else "single run after a warm-up",
              "peak_device_bytes": int(peak), "peak_above_input_bytes": int(peak - base),
              "dense_bytes": int(n) * int(d) * 4, "parity_rows": n_rows,
              "parity_rows_identical": float((idx[rows] == bi[:, :k]).all(1).mean()),
              "parity_max_ulp": int(ulp.max())})
    del csr
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="dense,b,a")
    ap.add_argument("--rows", type=int, default=4096, help="rows sampled for the dense parity check")
    ap.add_argument("--dtype", default="fp32", choices=sorted(DTYPES), help="element type of the dense matrix")
    a = ap.parse_args()
    torch.cuda.init()
    assert _lib.load().mde_knn_long_max_k() == 256
    parts = a.parts.split(",")
    w = text_like(20_000, seed=5)
    cw, sw = dm._to_device_csr(w, dev)
    dm.knn_sparse_device(cw, sw, 100)  # warm-up of the sparse search
    del cw
    if "dense" in parts:
        run_dense(a.rows, a.dtype)
    if "b" in parts:
        run_sparse("b_mnist_like_csr", sp.csr_matrix(mnist_like()), [65, 256], 3, 256)
    if "a" in parts:
        run_sparse("a_text_like", text_like(300_000), [100], 1, 256)


if __name__ == "__main__":
    main()
