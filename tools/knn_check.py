"""mde_knn (wgmma cross terms + running top-32 + exact re-rank; mde_knn_wide and its top-96 for 24 < k <= 64) against
an fp64 brute force, and timed against the library-GEMM + torch.topk path it replaces.  At k <= 24 the full run also
times mde_knn_wide on the same matrix.  `--dtype fp16|bf16` casts every matrix to that type and searches it in place
(mde_knn16*); the brute force and the GEMM path work on its fp32 upcast.  One JSON line per shape, with the GPU name,
power limit and max SM clock read in the same run, and in the full run the peak device memory of the search.
Usage: python tools/knn_check.py [small|full] [k] [--dtype fp32|fp16|bf16]   (k: the neighbours of the full run,
default 15)"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pymde_b200.preprocess import data_matrix as dm

dev = torch.device("cuda", 0)


def brute64(X, rows, k):
    """k smallest fp64 squared distances (and indices) of the given rows."""
    Xd = X.double()
    Q = Xd[rows]
    d2 = (Q * Q).sum(1)[:, None] + (Xd * Xd).sum(1)[None, :] - 2.0 * Q @ Xd.T
    d2[torch.arange(len(rows), device=X.device), rows] = float("inf")
    val, idx = torch.topk(d2, k, dim=1, largest=False)
    return val, idx


def gemm_path(X, k, rows=8192):
    sq = (X * X).sum(1)
    out = []
    for s0 in range(0, X.shape[0], rows):
        Q = X[s0:s0 + rows]
        d2 = (sq[s0:s0 + rows, None] + sq[None, :] - 2.0 * (Q @ X.T)).clamp_(min=0)
        d2[torch.arange(Q.shape[0], device=X.device), torch.arange(s0, s0 + Q.shape[0], device=X.device)] = float("inf")
        out.append(torch.topk(d2, k, dim=1, largest=False)[1])
    return torch.cat(out)


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


def wide_only(X, k):
    """mde_knn_wide (mde_knn16_wide for 16-bit X) at any k <= 64 (knn_device takes it only above 24)."""
    import ctypes as C
    from pymde_b200 import _lib
    lib = _lib.load()
    n, d = X.shape
    ws_bytes, search, args = dm._entries(lib, X, "_wide")
    need = C.c_size_t(0)
    _lib.check(ws_bytes(n, d, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=X.device)
    idx = torch.empty((n, k), dtype=torch.int32, device=X.device)
    d2 = torch.empty((n, k), dtype=torch.float32, device=X.device)
    _lib.check(search(*args, n, d, k, idx.data_ptr(), d2.data_ptr(), ws.data_ptr() + (-ws.data_ptr()) % 1024,
                      need.value, None))
    torch.cuda.synchronize()
    return idx, d2


def check(n, d, k, seed, clustered, time_it=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    if clustered:  # MNIST-like: non-negative, many exact zeros, cluster structure
        centers = torch.rand((10, d), generator=g, device=dev)
        lab = torch.randint(0, 10, (n,), generator=g, device=dev)
        X = (centers[lab] + 0.35 * torch.randn((n, d), generator=g, device=dev)).clamp_(0, 1)
        X = torch.where(X < 0.3, torch.zeros_like(X), X).contiguous()
    else:
        X = torch.randn((n, d), generator=g, device=dev)
    X = X.to(DTYPE)
    Xs, X = X, X.float()  # Xs: the matrix searched; X: its fp32 values, for the checks and the GEMM path
    idx, d2 = dm.knn_device(Xs, k)
    torch.cuda.synchronize()
    rows = torch.arange(n, device=dev) if n <= 8192 else torch.randperm(n, generator=g, device=dev)[:4096]
    val, ref = brute64(X, rows, k)
    got = idx[rows].long()
    # exact fp64 distances of what we returned, in the returned order
    gd = ((X[rows].double()[:, None, :] - X[got].double()) ** 2).sum(-1)
    ok_sorted = bool((gd[:, 1:] >= gd[:, :-1] - 1e-6 * gd[:, 1:].abs() - 1e-9).all())
    rel = ((gd - val).abs() / val.clamp_min(1e-12)).max().item()
    same = (torch.sort(got, 1)[0] == torch.sort(ref, 1)[0]).all(1).float().mean().item()
    d2rel = ((d2[rows].double() - gd).abs() / gd.clamp_min(1e-12)).max().item()
    rec = {"n": n, "d": d, "k": k, "dtype": DTYPE_NAME, "clustered": clustered, "rows_checked": int(len(rows)),
           "kth_distance_max_rel_err_vs_fp64": rel, "rows_with_identical_sets": same, "ascending": ok_sorted,
           "returned_d2_max_rel_err": d2rel, "self_in_list": bool((got == rows[:, None]).any())}
    if time_it:
        arms = [("kernel_ms", lambda: dm.knn_device(Xs, k)), ("gemm_topk_ms", lambda: gemm_path(X, k))]
        if k <= 24:
            arms.append(("wide_kernel_ms", lambda: wide_only(Xs, k)))
            wi, wd = wide_only(Xs, k)
            rec["wide_d2_identical"] = bool(torch.equal(wd, d2))
        for name, fn in arms:
            fn(); torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
            rec[name] = min(ts)
        del idx, d2
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        out = dm.knn_device(Xs, k)
        torch.cuda.synchronize()
        rec["kernel_peak_above_input_bytes"] = torch.cuda.max_memory_allocated(dev) - base
        rec["input_bytes"] = Xs.numel() * Xs.element_size()
        del out
        flops = (3 if DTYPE == torch.float32 else 1) * 2.0 * n * n * ((d + 63) // 64 * 64)
        rec["tensor_tflops_at_kernel_ms"] = flops / (rec["kernel_ms"] * 1e-3) / 1e12
        rec.update(gpu_identity())
    print(json.dumps(rec), flush=True)
    return rec


argv = sys.argv[1:]
DTYPE_NAME = "fp32"
if "--dtype" in argv:
    i = argv.index("--dtype")
    DTYPE_NAME = argv[i + 1]
    del argv[i:i + 2]
DTYPE = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}[DTYPE_NAME]
mode = argv[0] if len(argv) > 0 else "small"
k_full = int(argv[1]) if len(argv) > 1 else 15
check(1000, 64, 5, 0, False)
check(3000, 100, 15, 1, False)
check(5000, 784, 15, 2, True)
check(5000, 784, 40, 2, True)
if mode == "full":
    check(70000, 784, k_full, 3, True, time_it=True)
