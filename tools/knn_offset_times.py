"""Cost of centring and certifying the dense exact k-nearest-neighbour searches (csrc/mde_knn.cu), on one GPU.

  python tools/knn_offset_times.py [--base path/to/older/libmde_b200.so] [--out result.json]

Times `mde_knn`, `mde_knn_wide` and `mde_knn_long` at 70 000 x 784 (MNIST-shaped: clipped Gaussian values, many exact
zeros), k = 15, 64 and 256, and `mde_knn16` / `mde_knn16_wide` on its fp16 and bf16 copies, with CUDA events around each call (median of 5 after a warm-up call), alternating with the
same entries of `--base` when given.  The GEMM path at k = 100 and 256 against its fp32 / top-k form before
centring (median of 2 after a warm-up).  Then the worst case -- far-apart clusters, where no row certifies and every
row is searched directly -- at 70 000 x 64 and 70 000 x 784, and the fraction of rows certified on the MNIST-shaped
data for fp32, fp16 and bf16 input.  Prints one JSON object, with the GPU's name and power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

ENTRIES = {15: "mde_knn", 64: "mde_knn_wide", 256: "mde_knn_long"}


def _declare(lib):
    for name in ENTRIES.values():
        getattr(lib, name + "_ws_bytes").argtypes = [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]
        getattr(lib, name).argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_size_t, C.c_void_p]
        name16 = name.replace("mde_knn", "mde_knn16")
        getattr(lib, name16 + "_ws_bytes").argtypes = [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]
        getattr(lib, name16).argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]
    return lib


def _call(lib, name, X, k, fb=None):
    """One search; returns its time in ms (CUDA events) and the outputs."""
    n, d = X.shape
    half = X.dtype != torch.float32
    need = C.c_size_t(0)
    assert getattr(lib, "%s_ws_bytes" % name.replace("mde_knn", "mde_knn16" if half else "mde_knn"))(
        n, d, C.byref(need)) == 0
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device="cuda")
    p = ws.data_ptr() + (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((n, k), dtype=torch.float32, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn = name.replace("mde_knn", "mde_knn16") if half else name
    args = (X.data_ptr(), 1 if X.dtype == torch.float16 else 2) if half else (X.data_ptr(),)
    if fb is None:
        rc = getattr(lib, fn)(*args, n, d, k, idx.data_ptr(), d2.data_ptr(), p, need.value, None)
    else:
        rc = getattr(lib, fn + "_ex")(*args, n, d, k, idx.data_ptr(), d2.data_ptr(), p, need.value, None, C.byref(fb))
    e1.record()
    torch.cuda.synchronize()
    assert rc == 0, rc
    return e0.elapsed_time(e1), idx, d2


def _old_gemm(X, k):
    """The GEMM path before centring, for the timing comparison: fp32 norm expansion and top-k, no re-rank."""
    n = X.shape[0]
    sq = (X * X).sum(1)
    rows = max(256, min(n, int(2 ** 27 // max(n, 1))))
    out = []
    for s0 in range(0, n, rows):
        Q = X[s0:s0 + rows]
        d2 = (sq[s0:s0 + rows, None] + sq[None, :] - 2.0 * (Q @ X.T)).clamp_(min=0)
        d2[torch.arange(Q.shape[0], device=X.device), torch.arange(s0, s0 + Q.shape[0], device=X.device)] = float("inf")
        out.append(torch.topk(d2, k, dim=1, largest=False))
    return out


def mnist_shaped(n=70_000, d=784, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn((n, d), generator=g, device="cuda")
    return torch.where(X < 0.3, torch.zeros_like(X), X.clamp(max=1.0)).contiguous()


def far_clusters(n, d, seed=0):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((10, d))
    c *= 1000.0 / np.linalg.norm(c, axis=1, keepdims=True)
    X = c[rng.integers(0, 10, n)] + rng.standard_normal((n, d))
    return torch.from_numpy(X.astype(np.float32)).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="an older libmde_b200.so to time against")
    ap.add_argument("--out")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from pymde_b200 import _lib
    cur = _lib.load()
    libs = {"new": cur}
    if a.base:
        libs["base"] = _declare(C.CDLL(os.path.abspath(a.base)))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu, "shape": [70_000, 784], "times_ms": {}, "worst_case_ms": {}, "certified_fraction": {}}
    X = mnist_shaped()
    runs = [(k, name, torch.float32) for k, name in ENTRIES.items()]
    runs += [(k, ENTRIES[k], dt) for dt in (torch.float16, torch.bfloat16) for k in (15, 64)]
    for k, name, dt in runs:
        Y = X.to(dt)
        tag = name if dt == torch.float32 else name.replace("mde_knn", "mde_knn16") + "_" + str(dt).split(".")[1]
        ts = {key: [] for key in libs}
        for key, lib in libs.items():
            _call(lib, name, Y, k)  # warm-up
        for _ in range(a.reps):
            for key, lib in libs.items():
                ts[key].append(_call(lib, name, Y, k)[0])
        if "base" in libs:  # the same result as the older library
            _, i0, d0 = _call(libs["base"], name, Y, k)
            _, i1, d1 = _call(cur, name, Y, k)
            out.setdefault("rows_differing_from_base", {})[tag] = int(((i0 != i1) | (d0 != d1)).any(1).sum())
        out["times_ms"][tag] = {key: float(np.median(v)) for key, v in ts.items()}
    # the GEMM path (the default for dense 64 < k <= 256) against its fp32 / top-k form before centring
    from pymde_b200.preprocess import data_matrix as dm
    for k in (100, 256):
        ts = {"new": [], "base": []}
        for rep in range(3):
            for key, fn in (("new", lambda: dm._gemm_search(X, k)), ("base", lambda: _old_gemm(X, k))):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                if rep:  # (the first round warms up)
                    ts[key].append(e0.elapsed_time(e1))
        out["times_ms"]["gemm_path_k%d" % k] = {key: float(np.median(v)) for key, v in ts.items()}
        if k == 256:
            out["times_ms"]["gemm_path_k%d" % k]["mde_knn_long"] = out["times_ms"]["mde_knn_long"]["new"]
    for d in (64, 784):
        F = far_clusters(70_000, d)
        fb = C.c_int(-1)
        _call(cur, "mde_knn", F, 15, fb)
        t = [_call(cur, "mde_knn", F, 15, fb)[0] for _ in range(2)]
        out["worst_case_ms"]["70000x%d_k15" % d] = {"ms": float(np.median(t)), "rows_searched_directly": fb.value}
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        Y = X.to(dtype)
        for k, name in ENTRIES.items():
            fb = C.c_int(-1)
            _call(cur, name, Y, k, fb)
            out["certified_fraction"]["%s_k%d" % (str(dtype).split(".")[1], k)] = 1.0 - fb.value / X.shape[0]
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
