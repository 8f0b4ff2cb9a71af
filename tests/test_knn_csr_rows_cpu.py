"""CPU: the row-range sparse k-nearest-neighbour search (`mde_knn_csr_rows`, include/mde_b200.h) is exported, additive
(the ABI version is still 1) and refuses bad arguments before it touches a device; its candidate-slice rule
(mde_logic.h: knn_slices, with the narrow, wide and long CSR tile shapes) fills the SMs only while the query tiles
leave them idle; and its workspace, host arithmetic alone, grows with n and holds the larger split."""
import ctypes as C
import os

import numpy as np
import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
NAMES = ("mde_knn_csr_rows_ws_bytes", "mde_knn_csr_rows")
NUM_SMS = 132


def _ws(n, d, nnz, rows, k):
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_csr_rows_ws_bytes(n, d, nnz, rows, k, C.byref(need)) == 0
    return need.value


class _Out:
    """Host buffers prefilled with -7 in place of the outputs: a refusal must leave them as they are."""

    def __init__(self, rows=64, k=8):
        self.i = np.full(rows * k, -7, dtype=np.int32)
        self.d = np.full(rows * k, -7.0, dtype=np.float32)

    def untouched(self):
        return bool((self.i == -7).all() and (self.d == -7.0).all())


_HOST = object()  # the default outputs: the host buffers of _Out


def _call(n, d, nnz, rb, re, k, indptr=FAKE, indices=FAKE, values=FAKE, out_i=_HOST, out_d=_HOST, ws=FAKE,
          ws_bytes=1 << 40):
    out = _Out()
    oi = out.i.ctypes.data if out_i is _HOST else out_i
    od = out.d.ctypes.data if out_d is _HOST else out_d
    code = _lib.load().mde_knn_csr_rows(indptr, indices, values, n, d, nnz, rb, re, k, oi, od, ws, ws_bytes, None)
    assert out.untouched()
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
    assert "mde_dbg_knn_csr_slices" in _lib.DEBUG_SIGNATURES
    assert lib.mde_dbg_knn_csr_slices is not None


def test_bad_ranges_and_k_are_rejected():
    n, d, nnz = 1000, 30, 500
    for rb, re in [(-1, 5), (0, 0), (5, 5), (6, 5), (0, n + 1), (n, n + 1), (999, 1001)]:
        assert _call(n, d, nnz, rb, re, 5) == _lib.MDE_E_INVALID, (rb, re)
    for k in (0, -1, 257, 1000):
        assert _call(n, d, nnz, 0, 10, k) == _lib.MDE_E_INVALID, k
    assert _call(10, d, nnz, 0, 10, 10) == _lib.MDE_E_INVALID  # k > n - 1
    assert _call(1, d, nnz, 0, 1, 1) == _lib.MDE_E_INVALID
    assert _call(n, 0, nnz, 0, 10, 5) == _lib.MDE_E_INVALID
    assert _call(n, d, -1, 0, 10, 5) == _lib.MDE_E_INVALID


def test_null_pointers_are_rejected():
    n, d, nnz = 1000, 30, 500
    for kw in ("indptr", "indices", "values", "out_i", "out_d", "ws"):
        assert _call(n, d, nnz, 0, 10, 5, **{kw: None}) == _lib.MDE_E_INVALID, kw
    # with no non-zeros the index and value arrays are not read: the call goes on to the workspace check
    assert _call(n, d, 0, 0, 10, 5, indices=None, values=None, ws_bytes=0) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("k", [5, 40, 100, 256])
def test_workspace_too_small_or_misaligned_is_rejected(k):
    n, d, nnz = 1000, 30, 500
    need = _ws(n, d, nnz, 300, k)
    assert need % 1024 == 0
    assert _call(n, d, nnz, 100, 400, k, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _call(n, d, nnz, 100, 400, k, ws_bytes=0) == _lib.MDE_E_INVALID
    assert _call(n, d, nnz, 100, 400, k, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _call(n, d, nnz, 100, 400, k, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID


def test_workspace_query_rejects_bad_arguments_and_writes_nothing():
    lib = _lib.load()
    assert lib.mde_knn_csr_rows_ws_bytes(1000, 30, 500, 10, 5, None) == _lib.MDE_E_INVALID
    for n, d, nnz, rows, k in [(1, 30, 5, 1, 1), (1000, 0, 5, 10, 5), (1000, 30, -1, 10, 5), (1000, 30, 5, 0, 5),
                               (1000, 30, 5, 1001, 5), (1000, 30, 5, 10, 0), (1000, 30, 5, 10, 257),
                               (10, 30, 5, 5, 10)]:
        need = C.c_size_t(12345)
        assert lib.mde_knn_csr_rows_ws_bytes(n, d, nnz, rows, k, C.byref(need)) == _lib.MDE_E_INVALID
        assert need.value == 12345, (n, d, nnz, rows, k)


def _slices(n, rows, k):
    return _lib.load().mde_dbg_knn_csr_slices(n, rows, k)


@pytest.mark.parametrize("k,tm,tn", [(1, 128, 128), (15, 128, 128), (24, 128, 128), (25, 64, 128), (64, 64, 128)])
def test_slice_rule(k, tm, tn):
    for n in (130, 1000, 5000, 40000, 100000, 500000, 10 ** 6):
        c_tiles = -(-n // 128) * 128 // tn
        for rows in sorted({1, 37, 300, 1000, 3000, 10000, n // 2, n}):
            if rows > n:
                continue
            q_tiles = -(-rows // tm)
            s = _slices(n, rows, k)
            assert 1 <= s <= 16 and s <= max(1, c_tiles), (n, rows, s)
            if q_tiles >= NUM_SMS:
                assert s == 1, (n, rows, s)  # the query tiles fill the SMs: no split
            else:
                assert q_tiles * s <= NUM_SMS, (n, rows, s)  # one wave
                assert s == max(1, min(NUM_SMS // q_tiles, c_tiles, 16)), (n, rows, s)
    # 1 000 new rows next to 10^5 rows split; as many rows as fill the SMs do not
    assert _slices(101000, 1000, k) > 1
    assert _slices(10 ** 6, NUM_SMS * tm, k) == 1


@pytest.mark.parametrize("k", [65, 100, 256])
def test_the_long_search_keeps_one_slice(k):
    for n in (300, 5000, 10 ** 6):
        for rows in (1, 37, 1000, n):
            if rows <= n:
                assert _slices(n, rows, k) == 1, (n, rows, k)


def test_slice_query_rejects_bad_arguments():
    for n, rows, k in [(1, 1, 1), (1000, 0, 5), (1000, 1001, 5), (1000, 10, 0), (1000, 10, 257)]:
        assert _slices(n, rows, k) == -1, (n, rows, k)


@pytest.mark.parametrize("k", [15, 40, 100])
def test_workspace_grows_with_n(k):
    d, per_row = 30000, 40
    for rows in (1, 1000, 10000):
        sizes = [_ws(n, d, n * per_row, rows, k) for n in (rows + k + 1, 20000, 100000, 101000, 500000, 510000)
                 if n >= rows]
        assert all(b >= a for a, b in zip(sizes, sizes[1:])), (rows, sizes)
    # and with the non-zeros at a fixed n
    assert _ws(100000, d, 5 * 10 ** 6, 1000, k) > _ws(100000, d, 4 * 10 ** 6, 1000, k)


@pytest.mark.parametrize("k", [15, 40])
def test_workspace_holds_the_larger_split(k):
    n, d, nnz = 200000, 30000, 200000 * 40
    kk = 32 if k <= 24 else 96
    s1, s2 = _slices(n, 1000, k), _slices(n, 20000, k)
    assert s1 > s2 == 1
    # two lists (indices, scores) of S KK entries per query row, and the KK the merge selects
    lists1 = _ws(n, d, nnz, 1000, k) - _ws(n, d, nnz, 1, k)
    assert lists1 >= 999 * s1 * kk * 8 - 4096
    assert _ws(n, d, nnz, 1000, k) > _ws(n, d, nnz, 1000 // s1 + 1, k)
    # a workspace sized for more rows fits every search of fewer
    for rows in (1, 10, 100, 1000, 5000, 20000):
        assert _ws(n, d, nnz, 20000, k) >= _ws(n, d, nnz, rows, k), rows
