"""CPU: the C ABI of the 8-bit dense k-nearest-neighbour searches (`mde_knn8`, `mde_knn8_wide`, `mde_knn8_long`,
`mde_knn8_approx(_ex)`, `mde_knn8_rows`, `mde_knn8_max_d`, include/mde_b200.h) is exported, additive (the ABI version is
still 1), rejects bad arguments before it touches a device, keeps one 1-byte operand in its workspace, and its kernels
keep everything in registers; d_max and the certificate's gamma (csrc/mde_knn.cu, cert_bound) are derived again here
in exact integer and fp64 arithmetic."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "pymde_b200", "csrc")
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
EXACT = ("knn8", "knn8_wide", "knn8_long")
NAMES = tuple("mde_%s%s" % (e, s) for e in EXACT for s in ("", "_ex", "_ws_bytes")) + (
    "mde_knn8_approx_ws_bytes", "mde_knn8_approx", "mde_knn8_approx_ex", "mde_knn8_rows_ws_bytes", "mde_knn8_rows",
    "mde_knn8_max_d")
MAX_K = {"knn8": 24, "knn8_wide": 64, "knn8_long": 256, "knn8_approx": 64, "knn8_rows": 64}
DTYPES = (_lib.DTYPE_U8, _lib.DTYPE_S8)
ENTRIES = EXACT + tuple(e + "_ex" for e in EXACT) + ("knn8_approx", "knn8_approx_ex", "knn8_rows")


def _ws(entry, n, d, k=None):
    need = C.c_size_t(0)
    fn = getattr(_lib.load(), "mde_%s_ws_bytes" % entry)
    if entry == "knn8_rows":
        assert fn(n, d, n, k, C.byref(need)) == 0
    else:
        assert (fn(n, d, C.byref(need)) if k is None else fn(n, d, k, C.byref(need))) == 0
    return need.value


def _call(entry, n, d, k, dtype=_lib.DTYPE_U8, X=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE, ws_bytes=1 << 40):
    lib = _lib.load()
    if entry == "knn8_approx":
        return lib.mde_knn8_approx(X, dtype, n, d, k, C.c_uint64(1), out_i, out_d, ws, ws_bytes, None)
    if entry == "knn8_approx_ex":
        it = C.c_int(-7)
        code = lib.mde_knn8_approx_ex(X, dtype, n, d, k, C.c_uint64(1), out_i, out_d, ws, ws_bytes, None,
                                      C.byref(it))
        assert it.value == -7  # nothing written on a refusal
        return code
    fb = C.c_int(-7)
    if entry == "knn8_rows":
        code = lib.mde_knn8_rows(X, dtype, n, d, 0, max(n, 1), k, out_i, out_d, ws, ws_bytes, None, C.byref(fb))
    elif entry.endswith("_ex"):
        code = getattr(lib, "mde_" + entry)(X, dtype, n, d, k, out_i, out_d, ws, ws_bytes, None, C.byref(fb))
    else:
        return getattr(lib, "mde_" + entry)(X, dtype, n, d, k, out_i, out_d, ws, ws_bytes, None)
    assert fb.value == -7
    return code


def _max_k(entry):
    return MAX_K[entry.replace("_ex", "")]


def _base(entry):
    return entry.replace("_ex", "")


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header
    assert "#define MDE_DTYPE_U8 %d" % _lib.DTYPE_U8 in header
    assert "#define MDE_DTYPE_S8 %d" % _lib.DTYPE_S8 in header
    # the 16-bit codes are unchanged
    assert "#define MDE_DTYPE_FP16 1" in header and "#define MDE_DTYPE_BF16 2" in header


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", [0, 1, 2, 5, -1, 1 << 20])
def test_unknown_dtype_codes_are_rejected(entry, dtype):
    # every other argument is valid: only the code stops the call before its first CUDA call
    assert _call(entry, 300, 16, 5, dtype=dtype) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("dtype", [0, 1, 2, 5, -1, 1 << 20])
def test_max_d_rejects_unknown_codes(dtype):
    assert _lib.load().mde_knn8_max_d(dtype) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_null_pointers_are_rejected(entry, dtype):
    for kw in ("X", "out_i", "out_d", "ws"):
        assert _call(entry, 300, 16, 5, dtype=dtype, **{kw: None}) == _lib.MDE_E_INVALID
    lib = _lib.load()
    for e in EXACT:
        assert getattr(lib, "mde_%s_ws_bytes" % e)(300, 16, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn8_approx_ws_bytes(300, 16, 5, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn8_rows_ws_bytes(300, 16, 10, 5, None) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_bad_shapes_are_rejected(entry, dtype):
    top = _max_k(entry)
    for n, d, k in [(300, 4, 0), (300, 4, -1), (300, 4, top + 1), (10, 4, 10), (top + 1, 4, top + 1), (1, 4, 1),
                    (300, 0, 5), (0, 4, 1), (-5, 4, 1)]:
        assert _call(entry, n, d, k, dtype=dtype) == _lib.MDE_E_INVALID, (n, d, k)
    lib = _lib.load()
    need = C.c_size_t(0)
    for n, d in [(1, 4), (300, 0), (-3, 4)]:
        for e in EXACT:
            assert getattr(lib, "mde_%s_ws_bytes" % e)(n, d, C.byref(need)) == _lib.MDE_E_INVALID
        assert lib.mde_knn8_approx_ws_bytes(n, d, 5, C.byref(need)) == _lib.MDE_E_INVALID
    assert lib.mde_knn8_approx_ws_bytes(300, 4, 65, C.byref(need)) == _lib.MDE_E_INVALID
    assert lib.mde_knn8_rows_ws_bytes(300, 4, 10, 65, C.byref(need)) == _lib.MDE_E_INVALID
    # a row range outside [0, n)
    for lo, hi in [(-1, 10), (10, 10), (20, 10), (0, 301)]:
        assert lib.mde_knn8_rows(FAKE, dtype, 300, 4, lo, hi, 5, FAKE, FAKE, FAKE, 1 << 40, None,
                                 None) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_workspace_too_small_or_misaligned_is_rejected(entry, dtype):
    k = min(20, _max_k(entry))
    need = _ws(_base(entry), 1000, 30, k if "approx" in entry or "rows" in entry else None)
    assert _call(entry, 1000, 30, k, dtype=dtype, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _call(entry, 1000, 30, k, dtype=dtype, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(entry, 1000, 30, k, dtype=dtype, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(entry, 1100, 30, k, dtype=dtype, ws_bytes=need) == _lib.MDE_E_INVALID  # a larger problem


def _max_d_exact(dtype):
    """The largest d for which every accumulator, norm and score of the tiles is exact in int32 and every score stays
    below INT_MAX (the key of padded rows and empty slots), from the extreme values of the type in Python integers."""
    lo, hi = (0, 255) if dtype == _lib.DTYPE_U8 else (-128, 127)
    int_max = 2 ** 31 - 1

    def fits(d):
        dot = [d * a * b for a in (lo, hi) for b in (lo, hi)]          # <q, y> at the corners of the cube
        norm_max = d * max(lo * lo, hi * hi)
        two_dot = [2 * x for x in dot]
        # the score ||y||^2 - 2 <q, y>: its largest value takes the largest norm with the most negative product,
        # which the corner y = the value of larger magnitude, q = the other sign, attains
        score_max = max(d * y * y - 2 * d * q * y for q in (lo, hi) for y in (lo, hi))
        score_min = min(d * y * y - 2 * d * q * y for q in (lo, hi) for y in (lo, hi))
        return (all(-2 ** 31 <= x <= int_max for x in dot + two_dot) and norm_max <= int_max
                and score_max < int_max and score_min >= -2 ** 31)

    d = 1
    while fits(d * 2):
        d *= 2
    step = d
    while step:
        if fits(d + step):
            d += step
        step //= 2
    assert fits(d) and not fits(d + 1)
    return d


@pytest.mark.parametrize("dtype", DTYPES)
def test_max_d_is_the_int32_limit(dtype):
    lib = _lib.load()
    d_max = lib.mde_knn8_max_d(dtype)
    assert d_max == _max_d_exact(dtype)
    assert d_max == {_lib.DTYPE_U8: 16512, _lib.DTYPE_S8: 43919}[dtype]
    # one column more is refused by every exact entry, before any CUDA call; d_max itself passes the checks (the
    # fake workspace is too small, which is the next check)
    for entry in EXACT + tuple(e + "_ex" for e in EXACT) + ("knn8_rows",):
        assert _call(entry, 300, d_max + 1, 5, dtype=dtype) == _lib.MDE_E_UNSUPPORTED, entry
        assert _call(entry, 300, d_max, 5, dtype=dtype, ws_bytes=1) == _lib.MDE_E_INVALID, entry


def _gamma(d):
    """The certificate's relative error bound of the re-rank's fp32 sum of d exact squared differences: 0 while every
    partial sum is an integer below 2^24, else L u / (1 - L u) with L = ceil(d / 32) + 5 roundings on a path, plus
    2^-50 for the fp64 product (1 - gamma) D."""
    if d * 255 * 255 <= 2 ** 24:
        return 0.0
    u = 2.0 ** -24
    L = (d + 31) // 32 + 5
    return L * u / (1 - L * u) + 2.0 ** -50


@pytest.mark.parametrize("d", [1, 100, 128, 257, 258, 259, 784, 1024, 16512, 43919])
def test_certificate_gamma_is_the_derived_bound(d):
    assert _lib.load().mde_dbg_knn8_gamma(d) == _gamma(d)


def _rerank_f32(q, y):
    """The re-rank's fp32 arithmetic on exact integer rows: lane-strided fmaf chains, then a 5-level butterfly."""
    d = q.shape[0]
    lanes = np.zeros(32, np.float32)
    for j in range(d):
        t = np.float32(float(q[j]) - float(y[j]))
        lanes[j % 32] = np.float32(np.float64(t) * np.float64(t) + np.float64(lanes[j % 32]))  # one rounding
    o = 16
    while o:
        lanes = (lanes + lanes[np.arange(32) ^ o]).astype(np.float32)
        o >>= 1
    return float(lanes[0])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", [258, 259, 784, 3000])
def test_gamma_bounds_the_rerank_error(dtype, d):
    """r(y) >= (1 - gamma) D(y) on rows whose sums round the most: every difference at its largest magnitude (and
    random ones), so the partial sums sit where fp32 rounding is coarsest."""
    rng = np.random.default_rng(d)
    lo, hi = (0, 255) if dtype == _lib.DTYPE_U8 else (-128, 127)
    g = _gamma(d)
    worst = 0.0
    for trial in range(12):
        if trial < 4:
            q = np.full(d, lo, np.int64)
            y = np.full(d, hi, np.int64)
            y[rng.random(d) < 0.25 * trial] = lo + 1
        else:
            q = rng.integers(lo, hi + 1, d)
            y = rng.integers(lo, hi + 1, d)
        D = int(((q - y) ** 2).sum())
        r = _rerank_f32(q, y)
        if d * 255 * 255 <= 2 ** 24:
            assert r == D
        assert r >= (1 - g) * D, (r, D, g)
        worst = max(worst, (D - r) / D if D else 0.0)
    assert worst <= g


@pytest.mark.parametrize("n,d", [(2, 1), (129, 7), (3001, 65), (70000, 784), (10 ** 6, 1024)])
def test_workspace_has_no_lo_operand_and_one_byte_per_element(n, d):
    n_pad, k_pad16, k_pad8 = -(-n // 128) * 128, -(-d // 64) * 64, -(-d // 128) * 128
    for e8, e16 in zip(EXACT, ("knn16", "knn16_wide", "knn16_long")):
        w8, w16 = _ws(e8, n, d), _ws(e16, n, d)
        assert w8 % 1024 == 0
        assert w8 >= n_pad * k_pad8  # the one 8-bit operand
        # the 16-bit layout less its 2-byte operand and the column mean's sums, plus the 1-byte operand
        assert w8 <= w16 - 2 * n_pad * k_pad16 + n_pad * k_pad8 + 1024, (e8, w8, w16)
    # NN-descent keeps no copy of X at all: the same workspace as the fp32 search
    for k in (1, 24, 25, 64):
        if k <= n - 1:
            assert _ws("knn8_approx", n, d, k) == _ws("knn_approx", n, d, k)


def test_rows_workspace_matches_the_full_search():
    """A rows search of all n rows needs what the full search of the same list size needs."""
    for n, d in [(300, 16), (70000, 784)]:
        assert _ws("knn8_rows", n, d, 20) == _ws("knn8", n, d)
        assert _ws("knn8_rows", n, d, 40) == _ws("knn8_wide", n, d)


def test_the_fp32_workspace_of_a_large_uint8_search():
    """10^7 x 1024: the fp32 route needs over 80 GB of scratch beyond the fp32 copy; the 8-bit route about 12.8 GB."""
    n, d = 10 ** 7, 1024
    w8 = _ws("knn8", n, d)
    w32 = _ws("knn", n, d)
    assert w8 < 13 * 10 ** 9
    assert w32 + 4 * n * d > 80 * 10 ** 9


def _tool(name):
    for c in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
        if c and os.path.exists(c):
            return c
    return None


def test_8_bit_kernels_do_not_spill():
    nvcc = _tool("nvcc")
    if nvcc is None:
        pytest.skip("needs nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        procs = [subprocess.Popen([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas",
                                  "-v", "-c", os.path.join(CSRC, src), "-o", os.path.join(tmp, src + ".o")],
                                 stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
                 for src in ("mde_knn.cu", "mde_knn_approx.cu")]
        logs = []
        for p in procs:
            _, err = p.communicate()
            assert p.returncode == 0, err[-2000:]
            logs.append(err)
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores",
                       "\n".join(logs))
    # the 8-bit instantiations: uint8_t (h) / int8_t (a) as the first template argument, and the integer certificate
    eight = [(fn, int(frame), int(spill)) for fn, frame, spill in found
             if re.search(r"kernelI[ha](E|Li)", fn) or re.search(r"nnd_\w+_kernelILi\d+E[ha]E", fn)
             or "knn_certify_kernelIiE" in fn]
    names = " ".join(fn for fn, _, _ in eight)
    for kernel in ("knn_prep_kernel", "knn_tile_kernel", "knn_wide_tile_kernel", "knn_rerank_kernel",
                   "knn_wide_rerank_kernel", "knn_long_rerank_kernel", "knn_certify_kernel", "knn_direct_kernel",
                   "knn_merge_rerank_kernel", "nnd_join_kernel"):
        assert kernel in names, kernel
    # prep, narrow tiles, wide and long tiles, three re-ranks, merge, direct (x2 types); join x2 list sizes (x2 types)
    assert len(eight) >= 2 * (1 + 1 + 2 + 3 + 1 + 1) + 2 * 2, len(eight)
    for fn, frame, spill in eight:
        assert frame == 0 and spill == 0, (fn, frame, spill)
