"""CPU: the long row-range k-nearest-neighbour searches (`mde_knn_long_rows`, `mde_knn16_long_rows`,
`mde_knn8_long_rows`, include/mde_b200.h) are exported, additive (the ABI version is still 1) and reject bad arguments
before they touch a device; their candidate-slice rule (mde_dbg_knn_long_slices) fills the SMs only while the query
tiles leave them idle, with tiles of 64 query and 64 candidate rows; their workspace grows with the slices; and
`data_matrix.knn_rows_device_long` checks its arguments before it touches a device."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
NAMES = ("mde_knn_long_rows_ws_bytes", "mde_knn_long_rows", "mde_knn16_long_rows_ws_bytes", "mde_knn16_long_rows",
         "mde_knn8_long_rows_ws_bytes", "mde_knn8_long_rows")
NUM_SMS = 132
KINDS = ["fp32", "16bit", "8bit"]
CODE = {"16bit": _lib.DTYPE_FP16, "8bit": _lib.DTYPE_U8}


def _ws_fn(kind):
    lib = _lib.load()
    return {"fp32": lib.mde_knn_long_rows_ws_bytes, "16bit": lib.mde_knn16_long_rows_ws_bytes,
            "8bit": lib.mde_knn8_long_rows_ws_bytes}[kind]


def _ws(n, d, rows, k, kind="fp32"):
    need = C.c_size_t(0)
    assert _ws_fn(kind)(n, d, rows, k, C.byref(need)) == 0
    return need.value


def _call(n, d, rb, re, k, kind="fp32", dtype=None, X=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE, ws_bytes=1 << 40):
    lib = _lib.load()
    fb = C.c_int(-7)
    if kind == "fp32":
        code = lib.mde_knn_long_rows(X, n, d, rb, re, k, out_i, out_d, ws, ws_bytes, None, C.byref(fb))
    else:
        fn = lib.mde_knn16_long_rows if kind == "16bit" else lib.mde_knn8_long_rows
        code = fn(X, CODE[kind] if dtype is None else dtype, n, d, rb, re, k, out_i, out_d, ws, ws_bytes, None,
                  C.byref(fb))
    assert fb.value == -7  # nothing written on a refusal
    return code


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header
    assert "mde_dbg_knn_long_slices" in _lib.SIGNATURES  # declared in the header, unlike the older debug entries
    assert "int mde_dbg_knn_long_slices(" in header


@pytest.mark.parametrize("kind", KINDS)
def test_bad_ranges_and_k_are_rejected(kind):
    n, d = 1000, 30
    for rb, re in [(-1, 5), (0, 0), (5, 5), (6, 5), (0, n + 1), (n, n + 1), (999, 1001)]:
        assert _call(n, d, rb, re, 100, kind) == _lib.MDE_E_INVALID, (rb, re)
    for k in (0, -1, 257, 1000):
        assert _call(n, d, 0, 10, k, kind) == _lib.MDE_E_INVALID, k
    assert _call(100, d, 0, 10, 100, kind) == _lib.MDE_E_INVALID  # k > n - 1
    assert _call(1, d, 0, 1, 1, kind) == _lib.MDE_E_INVALID
    assert _call(n, 0, 0, 10, 100, kind) == _lib.MDE_E_INVALID
    for kw in ("X", "out_i", "out_d", "ws"):
        assert _call(n, d, 0, 10, 100, kind, **{kw: None}) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("kind,dtype", [("16bit", 0), ("16bit", 3), ("16bit", -1), ("8bit", 0), ("8bit", 1),
                                        ("8bit", 5)])
def test_unknown_dtype_codes_are_rejected(kind, dtype):
    assert _call(1000, 30, 0, 10, 100, kind, dtype=dtype) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("dtype", [_lib.DTYPE_U8, _lib.DTYPE_S8])
def test_8bit_wider_than_d_max_is_unsupported(dtype):
    d_max = _lib.load().mde_knn8_max_d(dtype)
    assert _call(1000, d_max + 1, 0, 10, 100, "8bit", dtype=dtype) == _lib.MDE_E_UNSUPPORTED
    assert _call(1000, d_max, 0, 10, 100, "8bit", dtype=dtype, ws_bytes=0) == _lib.MDE_E_INVALID  # (d_max passes)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("k", [1, 100, 256])
def test_workspace_too_small_or_misaligned_is_rejected(kind, k):
    need = _ws(1000, 30, 300, k, kind)
    assert need % 1024 == 0
    assert _call(1000, 30, 100, 400, k, kind, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _call(1000, 30, 100, 400, k, kind, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(1000, 30, 100, 400, k, kind, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("kind", KINDS)
def test_workspace_query_rejects_bad_arguments(kind):
    fn = _ws_fn(kind)
    need = C.c_size_t(0)
    assert fn(1000, 30, 10, 100, None) == _lib.MDE_E_INVALID
    for n, d, rows, k in [(1, 30, 1, 1), (1000, 0, 10, 100), (1000, 30, 0, 100), (1000, 30, 1001, 100),
                          (1000, 30, 10, 0), (1000, 30, 10, 257), (100, 30, 5, 100)]:
        assert fn(n, d, rows, k, C.byref(need)) == _lib.MDE_E_INVALID, (n, d, rows, k)


def _slices(n, rows, k=100):
    return _lib.load().mde_dbg_knn_long_slices(n, rows, k)


def test_slice_rule():
    for n in (130, 1000, 5000, 40000, 70000, 10 ** 6, 2 * 10 ** 6):
        c_tiles = -(-n // 128) * 128 // 64
        for rows in sorted({1, 37, 64, 65, 300, 1000, 3000, 8448, 8449, 10000, n // 2, n}):
            if rows > n or rows < 1:
                continue
            q_tiles = -(-rows // 64)
            s = _slices(n, rows)
            assert s == max(1, min(NUM_SMS // q_tiles, c_tiles, 16)), (n, rows, s)
            if q_tiles >= NUM_SMS:
                assert s == 1, (n, rows, s)  # the query tiles fill the SMs: no split
            else:
                assert q_tiles * s <= NUM_SMS  # one wave
    # 1 000 new rows are 16 query tiles: 8 slices fill 128 of the 132 SMs
    assert _slices(10 ** 6, 1000) == 8 and _slices(10 ** 6, 64) == 16 and _slices(10 ** 6, 10000) == 1
    assert _slices(130, 1) == 4  # at most one candidate tile per slice
    for k in (1, 65, 256):
        assert _slices(5000, 100, k) == _slices(5000, 100)  # S does not depend on k
    assert _slices(1000, 2000) == -1 and _slices(1000, 0) == -1 and _slices(1, 1) == -1
    assert _slices(1000, 10, 0) == -1 and _slices(1000, 10, 257) == -1
    # the short searches keep their own rule, and the existing debug entry still refuses k > 64
    assert _lib.load().mde_dbg_knn_slices(1000, 10, 65) == -1


@pytest.mark.parametrize("kind", KINDS)
def test_workspace_grows_with_the_slices(kind):
    n, d = 200000, 64
    s1, s2 = _slices(n, 1000), _slices(n, 20000)
    assert s1 > s2 == 1
    for k in (65, 256):
        assert _ws(n, d, 1000, k, kind) == _ws(n, d, 1000, 100, kind)  # (k does not size it)
    per_row = _ws(n, d, 1000, 100, kind) - _ws(n, d, 1, 100, kind)
    # two lists (indices, scores) of S 288 entries and one merged list of 288 per query row
    assert per_row >= 999 * (s1 + 1) * 288 * 8 - 8192
    assert _ws(n, d, 1000, 100, kind) > _ws(n, d, 1000 // s1 + 1, 100, kind)
    # monotone in rows and in n
    prev = 0
    for rows in (1, 10, 64, 65, 500, 1000, 8448, 8449, 20000, n):
        w = _ws(n, d, rows, 100, kind)
        assert w >= prev, rows
        prev = w
    prev = 0
    for nn in (1000, 1001, 5000, 70000, n):
        w = _ws(nn, d, 1000, 100, kind)
        assert w >= prev, nn
        prev = w


def test_operand_bytes_by_element_type():
    # the fp32 search keeps a bf16 hi and lo operand, a 16-bit one its own, an 8-bit one one byte per element
    n, d, rows = 200000, 256, 1000
    w32, w16, w8 = (_ws(n, d, rows, 100, kind) for kind in KINDS)
    n_pad = -(-n // 128) * 128
    assert w32 - w16 >= 2 * n_pad * d - 4096
    assert w16 > w8
    assert w8 < n * d * 4  # smaller than an fp32 copy of X


def test_wrapper_argument_errors():
    from pymde_b200.preprocess import data_matrix as dm
    X = np.zeros((300, 8), dtype=np.float32)
    for k in (0, -1, 257, 1000):
        with pytest.raises(ValueError):
            dm.knn_rows_device_long(X, k, 0, 10)
    with pytest.raises(ValueError):
        dm.knn_rows_device_long(X[:50], 100, 0, 10)  # k > n - 1
    for rb, re in [(-1, 5), (0, 0), (5, 5), (6, 5), (0, 301), (300, 301)]:
        with pytest.raises(ValueError):
            dm.knn_rows_device_long(X, 100, rb, re)
        with pytest.raises(ValueError):
            dm.knn_rows_device_long(sp.csr_matrix(X), 100, rb, re)
