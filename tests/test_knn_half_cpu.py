"""CPU: the C ABI of the 16-bit dense k-nearest-neighbour searches (`mde_knn16`, `mde_knn16_wide`, `mde_knn16_long`,
`mde_knn16_approx(_ex)`, include/mde_b200.h) is exported, additive (the ABI version is still 1), rejects bad arguments
before it touches a device, needs no lo operand in its workspace, and its kernels keep everything in registers."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "pymde_b200", "csrc")
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
EXACT = ("knn16", "knn16_wide", "knn16_long")
NAMES = tuple("mde_%s%s" % (e, s) for e in EXACT for s in ("", "_ws_bytes")) + (
    "mde_knn16_approx_ws_bytes", "mde_knn16_approx", "mde_knn16_approx_ex")
MAX_K = {"knn16": 24, "knn16_wide": 64, "knn16_long": 256, "knn16_approx": 64}
DTYPES = (_lib.DTYPE_FP16, _lib.DTYPE_BF16)


def _ws(entry, n, d, k=None):
    need = C.c_size_t(0)
    fn = getattr(_lib.load(), "mde_%s_ws_bytes" % entry)
    assert (fn(n, d, C.byref(need)) if k is None else fn(n, d, k, C.byref(need))) == 0
    return need.value


def _call(entry, n, d, k, dtype=_lib.DTYPE_FP16, X=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE, ws_bytes=1 << 40):
    lib = _lib.load()
    if entry == "knn16_approx":
        return lib.mde_knn16_approx(X, dtype, n, d, k, C.c_uint64(1), out_i, out_d, ws, ws_bytes, None)
    if entry == "knn16_approx_ex":
        it = C.c_int(-7)
        code = lib.mde_knn16_approx_ex(X, dtype, n, d, k, C.c_uint64(1), out_i, out_d, ws, ws_bytes, None,
                                       C.byref(it))
        assert it.value == -7  # nothing written on a refusal
        return code
    return getattr(lib, "mde_" + entry)(X, dtype, n, d, k, out_i, out_d, ws, ws_bytes, None)


ENTRIES = EXACT + ("knn16_approx", "knn16_approx_ex")


def _max_k(entry):
    return MAX_K[entry.replace("_ex", "")]


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header
    assert "#define MDE_DTYPE_FP16 %d" % _lib.DTYPE_FP16 in header
    assert "#define MDE_DTYPE_BF16 %d" % _lib.DTYPE_BF16 in header
    # the fp32 entries keep their bounds, which the 16-bit entries share
    assert lib.mde_knn_max_k() == 24 and lib.mde_knn_wide_max_k() == 64 and lib.mde_knn_long_max_k() == 256
    assert lib.mde_knn_approx_max_k() == 64


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", [0, 3, -1, 1 << 20])
def test_unknown_dtype_codes_are_rejected(entry, dtype):
    # every other argument is valid: only the code stops the call before its first CUDA call
    assert _call(entry, 300, 16, 5, dtype=dtype) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_null_pointers_are_rejected(entry, dtype):
    for kw in ("X", "out_i", "out_d", "ws"):
        assert _call(entry, 300, 16, 5, dtype=dtype, **{kw: None}) == _lib.MDE_E_INVALID
    lib = _lib.load()
    for e in EXACT:
        assert getattr(lib, "mde_%s_ws_bytes" % e)(300, 16, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn16_approx_ws_bytes(300, 16, 5, None) == _lib.MDE_E_INVALID


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
        assert lib.mde_knn16_approx_ws_bytes(n, d, 5, C.byref(need)) == _lib.MDE_E_INVALID
    assert lib.mde_knn16_approx_ws_bytes(300, 4, 65, C.byref(need)) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_workspace_too_small_or_misaligned_is_rejected(entry, dtype):
    k = min(20, _max_k(entry))
    base = entry.replace("_ex", "")
    need = _ws(base, 1000, 30, k if "approx" in entry else None)
    assert _call(entry, 1000, 30, k, dtype=dtype, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _call(entry, 1000, 30, k, dtype=dtype, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(entry, 1000, 30, k, dtype=dtype, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(entry, 1100, 30, k, dtype=dtype, ws_bytes=need) == _lib.MDE_E_INVALID  # a larger problem


@pytest.mark.parametrize("n,d", [(2, 1), (129, 7), (3001, 65), (70000, 784), (10 ** 6, 1024)])
def test_workspace_has_no_lo_operand(n, d):
    n_pad, k_pad = -(-n // 128) * 128, -(-d // 64) * 64
    for e16, e32 in zip(EXACT, ("knn", "knn_wide", "knn_long")):
        w16, w32 = _ws(e16, n, d), _ws(e32, n, d)
        assert w16 % 1024 == 0
        assert w16 <= w32 - 2 * n_pad * k_pad, (e16, w16, w32)
        assert w16 >= 2 * n_pad * k_pad  # the one operand is still there
    # NN-descent keeps no copy of X at all: the same workspace as the fp32 search
    for k in (1, 24, 25, 64):
        if k <= n - 1:
            assert _ws("knn16_approx", n, d, k) == _ws("knn_approx", n, d, k)


def _tool(name):
    for c in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
        if c and os.path.exists(c):
            return c
    return None


def test_16_bit_kernels_do_not_spill():
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
    # the 16-bit instantiations: __half / __nv_bfloat16 in the mangled name
    half = [(fn, int(frame), int(spill)) for fn, frame, spill in found if "6__half" in fn or "13__nv_bfloat16" in fn]
    names = " ".join(fn for fn, _, _ in half)
    for kernel in ("knn_prep_kernel", "knn_tile_kernel", "knn_wide_tile_kernel", "knn_rerank_kernel",
                   "knn_wide_rerank_kernel", "knn_long_rerank_kernel", "nnd_init_kernel", "nnd_join_kernel"):
        assert kernel in names, kernel
    # prep, narrow tiles, wide and long tiles, three re-ranks (x2 types); init x2 and join x2 list sizes (x2 types)
    assert len(half) >= 2 * (1 + 1 + 2 + 3) + 2 * (2 + 2), len(half)
    for fn, frame, spill in half:
        assert frame == 0 and spill == 0, (fn, frame, spill)
