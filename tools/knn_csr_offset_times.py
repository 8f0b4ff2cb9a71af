"""Cost of the certificate and the direct search of the exact sparse k-nearest-neighbour searches (DESIGN 11.1).

  python tools/knn_csr_offset_times.py [--base path/to/older/libmde_b200.so] [--reps 5] [--text-rows 100000]
                                       [--worst-text-rows 20000]

Ordinary data, against --base (an older build, alternating call by call, CUDA events, median and spread of --reps after
two warm-up calls each), with whether the outputs are bit-identical and the share of rows certified:
  (a) text-like CSR of tools/knn_sparse_check.py at --text-rows rows, (b) its MNIST-like 70 000 x 784 as CSR;
  k = 15, 64, 256 (mde_knn_csr, mde_knn_csr_wide, mde_knn_csr_long).
Offset data (this build only: an older build returns wrong neighbours there), one timed call after a warm-up:
  latlong_onehot and year_counts of tests/test_gpu_knn_csr_offset.py at 70 000 rows, k = 15;
  the worst case, where no row certifies: (b) with a constant column of 1 000, k = 15, 64, 256;
  (a) at --worst-text-rows rows with a constant column of 100, k = 15.
Prints the GPU's name and power limit, then one JSON line per case."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

ARGS = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_size_t, C.c_void_p]


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def _entry(lib, k, ex):
    name = "mde_knn_csr" + ("_long" if k > 64 else "_wide" if k > 24 else "")
    ws_fn = getattr(lib, name + "_ws_bytes")
    ws_fn.argtypes = [C.c_int64, C.c_int, C.c_int64, C.POINTER(C.c_size_t)]
    fn = getattr(lib, name + ("_ex" if ex else ""))
    fn.argtypes = ARGS + ([C.POINTER(C.c_int)] if ex else [])
    return name, ws_fn, fn


class Call:
    """One library's search of one matrix at one k, with its own workspace and outputs."""

    def __init__(self, lib, csr, shape, k, ex):
        (self.ip, self.ix, self.v), (self.n, self.d) = csr, shape
        self.nnz, self.k, self.ex = int(self.ix.shape[0]), k, ex
        self.name, ws_fn, self.fn = _entry(lib, k, ex)
        need = C.c_size_t(0)
        assert ws_fn(self.n, self.d, self.nnz, C.byref(need)) == 0
        self.need = need.value
        self.ws = torch.empty(self.need + 1024, dtype=torch.uint8, device="cuda")
        self.p = self.ws.data_ptr() + (-self.ws.data_ptr()) % 1024
        self.idx = torch.empty((self.n, k), dtype=torch.int32, device="cuda")
        self.d2 = torch.empty((self.n, k), dtype=torch.float32, device="cuda")
        self.fb = C.c_int(-1)

    def __call__(self, count=False):
        args = [self.ip.data_ptr(), self.ix.data_ptr(), self.v.data_ptr(), self.n, self.d, self.nnz, self.k,
                self.idx.data_ptr(), self.d2.data_ptr(), self.p, self.need, torch.cuda.current_stream().cuda_stream]
        if self.ex:
            args.append(C.byref(self.fb) if count else None)
        assert self.fn(*args) == 0


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def ordinary(case, A, libs, reps):
    from pymde_b200.preprocess import data_matrix as dm
    csr, shape = dm._to_device_csr(A, torch.device("cuda"))
    for k in (15, 64, 256):
        calls = {tag: Call(lib, csr, shape, k, tag == "new") for tag, lib in libs.items()}
        for _ in range(2):
            for c in calls.values():
                c()
        ts = {tag: [] for tag in calls}
        for _ in range(reps):
            for tag, c in calls.items():
                ts[tag] += _time(c, 1)
        calls["new"](count=True)
        line = {"case": case, "n": shape[0], "d": shape[1], "nnz": int(A.nnz), "k": k, "entry": calls["new"].name,
                "certified_fraction": round(1.0 - calls["new"].fb.value / shape[0], 6)}
        for tag, t in ts.items():
            line[tag + "_ms"] = {"median": round(float(np.median(t)), 2), "min": round(min(t), 2),
                                 "max": round(max(t), 2)}
        if "base" in calls:
            line["same_bits"] = bool(torch.equal(calls["new"].idx, calls["base"].idx) and
                                     torch.equal(calls["new"].d2, calls["base"].d2))
        print(json.dumps(line), flush=True)
        del calls
        torch.cuda.empty_cache()


def offset(case, A, lib, ks):
    from pymde_b200.preprocess import data_matrix as dm
    csr, shape = dm._to_device_csr(A, torch.device("cuda"))
    for k in ks:
        c = Call(lib, csr, shape, k, True)
        c(count=True)  # warm-up
        t = _time(lambda: c(count=True), 1)[0]
        print(json.dumps({"case": case, "n": shape[0], "d": shape[1], "nnz": int(A.nnz), "k": k, "entry": c.name,
                          "rows_searched_directly": c.fb.value, "ms": round(t, 1), "timing": "one call after a warm-up"}),
              flush=True)
        del c
        torch.cuda.empty_cache()


def with_column(A, value):
    return sp.hstack([A, sp.csr_matrix(np.full((A.shape[0], 1), value, np.float32))]).tocsr()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="an older libmde_b200.so to time the ordinary cases against")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--text-rows", type=int, default=100_000)
    ap.add_argument("--worst-text-rows", type=int, default=20_000)
    a = ap.parse_args()
    from knn_sparse_check import mnist_like, text_like
    from pymde_b200 import _lib
    from tests.test_gpu_knn_csr_offset import family
    torch.cuda.init()
    print("gpu:", _gpu(), flush=True)
    libs = {"new": _lib.load()}
    if a.base:
        libs["base"] = C.CDLL(os.path.abspath(a.base))
    text = text_like(a.text_rows)
    mnist = sp.csr_matrix(mnist_like())
    ordinary("b_mnist_like", mnist, libs, a.reps)
    ordinary("a_text_like", text, libs, a.reps)
    for name in ("latlong_onehot", "year_counts"):
        offset(name, family(name, n=70_000), libs["new"], (15,))
    offset("worst_b_mnist_like_plus_1000", with_column(mnist, 1000.0), libs["new"], (15, 64, 256))
    offset("a_text_like_plus_100", with_column(text_like(a.worst_text_rows, seed=3), 100.0), libs["new"], (15,))


if __name__ == "__main__":
    main()
