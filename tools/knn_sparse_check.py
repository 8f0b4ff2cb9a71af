"""Exact k-NN of sparse data matrices (mde_knn_csr) at realistic sizes: device time, peak device memory, the fraction
of K blocks the tile kernel visits, and parity on 256 sampled rows against a host fp64 brute force.  Synthetic data
only; one JSON line per shape, each with the GPU name and power limit read in the same run.

  (a) text-like: 3e5 x 1e5, Zipf feature frequencies, ~100 non-zeros per row around 1 000 cluster centres
      (120 GB dense: does not fit on the GPU); the host brute-force time is extrapolated from the sampled rows
  (b) MNIST-like: 70 000 x 784 clipped Gaussian, ~80 % zeros, stored as CSR, timed against the dense mde_knn
  (c) (a)'s kind with 1e6 rows, run once

--approx measures the approximate search (mde_knn_approx_csr, NN-descent) instead, on (a) and (c) at every k of
--k: call time (one run after a warm-up on a small matrix), iterations, peak device memory, recall@k on
--recall-rows (4 096) sampled rows against the host fp64 brute force, and on (a) the exact mde_knn_csr / mde_knn_csr_wide on the same matrix.

Usage: python tools/knn_sparse_check.py [--shapes abc] [--k 15] [--approx --k 15,50]
"""
import ctypes as C
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

dev = torch.device("cuda", 0)


def gpu_identity():
    out = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=10)
        out["power_limit_w"] = float(r.stdout.strip())
    except Exception:
        pass
    return out


def text_like(n, d=100_000, centres=1000, seed=0):
    """Rows around cluster centres; centre supports and background terms drawn from a Zipf law over the features
    (the frequent features in random positions), positive tf-idf-like values."""
    rng = np.random.default_rng(seed)
    zipf = 1.0 / np.arange(1, d + 1) ** 1.1
    zipf /= zipf.sum()
    pos = rng.permutation(d)
    sup = pos[rng.choice(d, (centres, 220), p=zipf)]
    w = rng.lognormal(0.0, 0.5, (centres, 220)).astype(np.float32)
    parts = []
    for s0 in range(0, n, 100_000):
        m = min(100_000, n - s0)
        lab = rng.integers(0, centres, m)
        keep = rng.random((m, 220)) < 0.6
        bg = pos[rng.choice(d, (m, 10), p=zipf)]
        r = np.concatenate([np.repeat(np.arange(m), 220)[keep.ravel()], np.repeat(np.arange(m), 10)])
        c = np.concatenate([sup[lab].ravel()[keep.ravel()], bg.ravel()])
        v = np.concatenate([(w[lab] * rng.lognormal(0.0, 0.3, (m, 220)).astype(np.float32)).ravel()[keep.ravel()],
                            np.full(m * 10, 0.5, np.float32)])
        parts.append(sp.csr_matrix((v, (r, c)), shape=(m, d), dtype=np.float32))
    A = sp.vstack(parts).tocsr()
    A.sum_duplicates()
    return A


def mnist_like(n=70_000, d=784, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    X = np.where(X < 0.8416, 0.0, np.minimum(X, 1.0)).astype(np.float32)  # P(X < 0.8416) = 0.8
    return X


def visited_fraction(A):
    """Share of (tile pair, K block) combinations the tile kernel visits: the features reordered by descending
    document frequency (stable), blocks of 64, tiles of 128 rows; every CTA sweeps every candidate tile."""
    n, d = A.shape
    cnt = np.bincount(A.indices, minlength=d)
    order = np.argsort(-cnt, kind="stable")
    perm = np.empty(d, np.int64)
    perm[order] = np.arange(d)
    rows = np.repeat(np.arange(n), np.diff(A.indptr))
    tb = np.unique((rows // 128) * ((d + 63) // 64) + perm[A.indices] // 64)
    per_block = np.bincount(tb % ((d + 63) // 64), minlength=(d + 63) // 64).astype(np.float64)
    tiles = (n + 127) // 128
    return float((per_block ** 2).sum() / (tiles * tiles * ((d + 63) // 64)))


def host_brute(A, rows, k):
    """fp64 brute force for the sampled rows: candidates from Q X^T (scipy sparse), exact re-rank of k + 9."""
    X = A.astype(np.float64).tocsr()
    sq = np.asarray(X.multiply(X).sum(1)).ravel()
    out_i, out_d = [], []
    for s0 in range(0, len(rows), 32):
        r = rows[s0:s0 + 32]
        S = (X[r] @ X.T).toarray()
        d2 = sq[r, None] + sq[None, :] - 2.0 * S
        d2[np.arange(len(r)), r] = np.inf
        cand = np.argpartition(d2, k + 9, axis=1)[:, :k + 9]
        for j, q in enumerate(r):
            c = np.sort(cand[j])
            diff = X[c] - X[np.full(len(c), q)]
            ex = np.asarray(diff.multiply(diff).sum(1)).ravel().astype(np.float32)
            o = np.lexsort((c, ex))[:k]
            out_i.append(c[o]); out_d.append(ex[o])
    return np.array(out_i), np.array(out_d)


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def run_sparse(name, A, k, reps, host_extrapolate, extra=None):
    n, d = A.shape
    csr, shape = dm._to_device_csr(A, dev)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    res = {}

    def go():
        res["out"] = dm.knn_sparse_device(csr, shape, k)
    t = timed(go, reps) if reps > 1 else None
    if t is None:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        go()
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(dev)
    idx, d2 = (x.cpu().numpy() for x in res["out"])
    rows = np.random.default_rng(1).choice(n, 256, replace=False)
    t0 = time.perf_counter()
    bi, bd = host_brute(A, rows, k)
    t_host = time.perf_counter() - t0
    same_rows = float((idx[rows] == bi).all(1).mean())
    ulp = np.abs(d2[rows].view(np.int32).astype(np.int64) - bd.view(np.int32).astype(np.int64))
    line = {"shape": name, "n": n, "d": d, "nnz": int(A.nnz), "k": k, "search_s": round(t, 4),
            "timing": "best of %d after a warm-up" % reps if reps > 1 else "single run",
            "peak_device_bytes": int(peak), "dense_bytes": int(n) * int(d) * 4,
            "visited_block_fraction": visited_fraction(A),
            "parity_rows_identical": same_rows, "parity_max_ulp": int(ulp.max())}
    if host_extrapolate:
        line["host_brute_s_extrapolated"] = round(t_host * n / len(rows), 1)
    if extra:
        line.update(extra(res["out"]))
    line.update(gpu_identity())
    print(json.dumps(line), flush=True)


def approx_call(csr, shape, k, seed=1):
    """mde_knn_approx_csr_ex: (idx, d2, iterations)."""
    lib = _lib.load()
    indptr, indices, values = csr
    n, d = shape
    nnz = int(indices.shape[0])
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_approx_csr_ws_bytes(n, d, nnz, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    d2 = torch.empty((n, k), dtype=torch.float32, device=dev)
    it = C.c_int(0)
    _lib.check(lib.mde_knn_approx_csr_ex(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), n, d, nnz, k,
                                         C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(),
                                         ws.data_ptr() + (-ws.data_ptr()) % 1024, need.value, None, C.byref(it)))
    torch.cuda.synchronize()
    return idx, d2, it.value


def recall(idx, ref):
    return float(np.mean([len(np.intersect1d(a, b)) for a, b in zip(idx, ref)])) / ref.shape[1]


def run_approx(name, A, ks, with_exact, n_rows=4096):
    """One JSON line per k; the host brute force runs once, at the largest k (its first k columns are the k-NN)."""
    n, d = A.shape
    csr, shape = dm._to_device_csr(A, dev)
    rows = np.random.default_rng(1).choice(n, n_rows, replace=False)
    t0 = time.perf_counter()
    bi, _ = host_brute(A, rows, max(ks))
    t_host = time.perf_counter() - t0
    for k in ks:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        t0 = time.perf_counter()
        idx, d2, it = approx_call(csr, shape, k)
        t = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated(dev)
        got = idx.cpu().numpy()
        line = {"shape": name, "n": n, "d": d, "nnz": int(A.nnz), "k": k, "approx_s": round(t, 3),
                "timing": "single run after a warm-up", "iterations": it, "peak_device_bytes": int(peak),
                "peak_above_input_bytes": int(peak - base), "recall_rows": n_rows,
                "recall": round(recall(got[rows], bi[:, :k]), 5), "host_brute_s": round(t_host, 1)}
        if with_exact:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ei, ed = dm.knn_sparse_device(csr, shape, k)
            torch.cuda.synchronize()
            line["exact_s"] = round(time.perf_counter() - t0, 3)
            line["exact_kernel"] = "mde_knn_csr" if k <= _lib.load().mde_knn_max_k() else "mde_knn_csr_wide"
            line["exact_recall"] = round(recall(ei.cpu().numpy()[rows], bi[:, :k]), 5)
            same = (torch.sort(ei.long(), 1)[0] == torch.sort(idx.long(), 1)[0]).all(1)
            line["rows_identical_to_exact"] = float(same.float().mean())
            line["identical_rows_bit_identical_d2"] = bool(torch.equal(d2[same].view(torch.int32),
                                                                       ed[same].view(torch.int32)))
            del ei, ed
        line.update(gpu_identity())
        print(json.dumps(line), flush=True)
        del idx, d2
    del csr
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="abc")
    ap.add_argument("--k", default="15", help="one k, or a comma-separated list with --approx")
    ap.add_argument("--rows-c", type=int, default=1_000_000)
    ap.add_argument("--reps-a", type=int, default=3)
    ap.add_argument("--approx", action="store_true")
    ap.add_argument("--recall-rows", type=int, default=4096, help="rows sampled for recall (--approx)")
    a = ap.parse_args()
    torch.cuda.init()
    if a.approx:
        ks = [int(k) for k in a.k.split(",")]
        w = text_like(20_000, seed=5)
        for k in ks:  # warm-up: module loads of both searches
            cw, sw = dm._to_device_csr(w, dev)
            approx_call(cw, sw, k)
            dm.knn_sparse_device(cw, sw, k)
        if "a" in a.shapes:
            run_approx("a_text_like", text_like(300_000), ks, True, a.recall_rows)
        if "c" in a.shapes:
            run_approx("c_text_like_1e6", text_like(a.rows_c, seed=2), ks, False, a.recall_rows)
        return
    a.k = int(a.k)
    if "a" in a.shapes:
        run_sparse("a_text_like", text_like(300_000), a.k, a.reps_a, True)
    if "b" in a.shapes:
        Xn = mnist_like()
        A = sp.csr_matrix(Xn)

        def dense_cmp(out):
            X = torch.from_numpy(Xn).to(dev)
            r = {}

            def go():
                r["out"] = dm.knn_device(X, a.k)
            t = timed(go)
            si, sd = out
            di, dd = r["out"]
            return {"dense_mde_knn_s": round(t, 4),
                    "rows_identical_to_dense": float((si == di).all(1).float().mean()),
                    "dense_sparse_max_rel_d2": float(((sd - dd).abs() / dd.clamp(min=1e-30)).max())}
        run_sparse("b_mnist_like", A, a.k, 3, False, dense_cmp)
    if "c" in a.shapes:
        run_sparse("c_text_like_1e6", text_like(a.rows_c, seed=2), a.k, 1, True)


if __name__ == "__main__":
    main()
