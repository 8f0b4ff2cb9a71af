"""The 8-bit k-nearest-neighbour route (uint8 / int8 read in place, `mde_knn8*`) against the fp32 route it replaces
(the parent's handling of such a matrix: an fp32 copy X.float() searched by `mde_knn*`), on one GPU.

  python tools/knn8_times.py [--out result.json] [--small]

Shapes: 70 000 x 784 uint8 at k = 15 (MNIST pixels), 10^6 x 128 int8 at k = 15 (quantised embeddings), and
2 * 10^6 x 1024 uint8 at k = 15 under PYMDE_B200_KNN=approx (NN-descent).  For each shape the two routes alternate in
one process: the whole neighbour search `data_matrix._search` on the CUDA 8-bit matrix, and the same call on its fp32
upcast with the upcast inside the timed call.  Wall time of the call ended by a device synchronise, best of 3 after a
warm-up call of each, and the peak device memory allocated during one call beyond what was allocated before it.  The
two results must be the same bits.  For the exact shapes the _ex entries also report how many rows the certificate
sent to the direct search.  Prints one JSON object with the card's name, power limit and max SM clock, read in the same
run.  `--small` runs every shape at 1/20 of its rows (a rehearsal)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

dev = torch.device("cuda", 0)


def gpu_identity():
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": None, "max_sm_clock_mhz": None}
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    p, c = r.stdout.strip().split(",")
    out["power_limit_w"], out["max_sm_clock_mhz"] = float(p), float(c)
    return out


def pixels(n, d, seed):
    """MNIST-like uint8: ten cluster templates, Gaussian noise, values below 60 set to 0."""
    g = torch.Generator(device=dev).manual_seed(seed)
    centers = torch.rand((10, d), generator=g, device=dev) * 255
    lab = torch.randint(0, 10, (n,), generator=g, device=dev)
    X = centers[lab]
    X += 40 * torch.randn((n, d), generator=g, device=dev)
    X[X < 60] = 0
    return X.clamp_(0, 255).to(torch.uint8)


def quantised(n, d, seed):
    """int8-quantised embedding vectors: unit Gaussian clusters scaled by 127 / 4 and rounded."""
    g = torch.Generator(device=dev).manual_seed(seed)
    centers = torch.randn((64, d), generator=g, device=dev)
    lab = torch.randint(0, 64, (n,), generator=g, device=dev)
    X = centers[lab]
    X += 0.5 * torch.randn((n, d), generator=g, device=dev)
    return (X * (127 / 4)).round_().clamp_(-128, 127).to(torch.int8)


def call(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def fallback_rows(X, k):
    """Rows the certificate sent to the direct search: (8-bit route, fp32 route on X.float())."""
    from pymde_b200 import _lib
    from pymde_b200.preprocess import data_matrix as dm
    lib = _lib.load()
    out = []
    for Y in (X, X.float()):
        ws_bytes, _, args = dm._entries(lib, Y)
        n, d = Y.shape
        need = C.c_size_t(0)
        _lib.check(ws_bytes(n, d, C.byref(need)))
        ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
        idx = torch.empty((n, k), dtype=torch.int32, device=dev)
        d2 = torch.empty((n, k), dtype=torch.float32, device=dev)
        fb = C.c_int(-1)
        search = getattr(lib, "mde_%s_ex" % dm._SEARCH_DTYPES[Y.dtype][0])
        _lib.check(search(*args, n, d, k, idx.data_ptr(), d2.data_ptr(), ws.data_ptr() + (-ws.data_ptr()) % 1024,
                          need.value, torch.cuda.current_stream().cuda_stream, C.byref(fb)))
        del ws, idx, d2
        out.append(fb.value)
    return out


def measure(name, X, k, mode, reps=3):
    from pymde_b200 import seed
    from pymde_b200.preprocess import data_matrix as dm
    if mode == "approx":
        os.environ["PYMDE_B200_KNN"] = "approx"
    else:
        os.environ.pop("PYMDE_B200_KNN", None)

    def run8():
        seed(0)
        return dm._search(X, k, dev)[:2]

    def run32():
        seed(0)
        return dm._search(X.float(), k, dev)[:2]

    res = {"shape": name, "n": X.shape[0], "d": X.shape[1], "dtype": str(X.dtype).replace("torch.", ""), "k": k,
           "mode": mode}
    (i8, d8), _, _ = call(run8)  # warm-up of each route
    (i32, d32), _, _ = call(run32)
    assert torch.equal(i8, i32) and torch.equal(d8, d32), name
    del i32, d32
    t8, t32, m8, m32 = [], [], 0, 0
    for _ in range(reps):
        (i, d), t, m = call(run8)
        assert torch.equal(i, i8) and torch.equal(d, d8)
        del i, d
        t8.append(t); m8 = max(m8, m)
        (i, d), t, m = call(run32)
        assert torch.equal(i, i8) and torch.equal(d, d8)
        del i, d
        t32.append(t); m32 = max(m32, m)
    res.update({"same_bits": True, "t8_s": round(min(t8), 4), "t32_s": round(min(t32), 4),
                "t8_all_s": [round(t, 4) for t in t8], "t32_all_s": [round(t, 4) for t in t32],
                "speedup": round(min(t32) / min(t8), 3), "peak8_bytes": m8, "peak32_bytes": m32,
                "x_bytes": X.numel()})
    if mode != "approx":
        res["fallback_rows_8"], res["fallback_rows_32"] = fallback_rows(X, k)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    s = 20 if a.small else 1
    out = gpu_identity()
    out["results"] = []
    for name, make, n, d, mode in [("mnist_pixels_u8", pixels, 70_000, 784, "kernel"),
                                   ("embeddings_s8", quantised, 1_000_000, 128, "kernel"),
                                   ("wide_u8_approx", pixels, 2_000_000, 1024, "approx")]:
        X = make(n // s, d, 1)
        r = measure(name, X, 15, mode)
        print(json.dumps(r), file=sys.stderr, flush=True)
        out["results"].append(r)
        del X
        torch.cuda.empty_cache()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
