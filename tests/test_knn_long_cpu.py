"""CPU: the C ABI of the long k-nearest-neighbour searches (`mde_knn_long`, `mde_knn_csr_long`) and of the long
neighbour-graph builder (`mde_knn_graph_long_*`, include/mde_b200.h) is exported, additive (the ABI version is still
1), and rejects bad arguments before it touches a device."""
import ctypes as C
import os

import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
SEARCH = ("mde_knn_long_max_k", "mde_knn_long_ws_bytes", "mde_knn_long", "mde_knn_csr_long_ws_bytes",
          "mde_knn_csr_long")
GRAPH = ("mde_knn_graph_long_max_k", "mde_knn_graph_long_ws_bytes", "mde_knn_graph_long_count",
         "mde_knn_graph_long_emit")


def _dense_ws(n, d):
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_long_ws_bytes(n, d, C.byref(need)) == 0
    return need.value


def _graph_ws(n, k):
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_graph_long_ws_bytes(n, k, C.byref(need)) == 0
    return need.value


def _dense(n, d, k, X=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE, ws_bytes=1 << 40):
    return _lib.load().mde_knn_long(X, n, d, k, out_i, out_d, ws, ws_bytes, None)


def _csr(n, d, nnz, k, indptr=FAKE, indices=FAKE, values=FAKE, out_i=FAKE, out_d=FAKE, ws=FAKE, ws_bytes=1 << 40):
    return _lib.load().mde_knn_csr_long(indptr, indices, values, n, d, nnz, k, out_i, out_d, ws, ws_bytes, None)


def _count(n, k, idx=FAKE, ws=FAKE, ws_bytes=1 << 40, out=True):
    p = C.c_int64(-7)
    code = _lib.load().mde_knn_graph_long_count(idx, n, k, ws, ws_bytes, C.byref(p) if out else None, None)
    assert p.value == -7  # nothing written on a refusal
    return code


def _emit(n, k, ws=FAKE, ws_bytes=1 << 40, edges=FAKE, weights=FAKE):
    return _lib.load().mde_knn_graph_long_emit(n, k, ws, ws_bytes, edges, weights, None)


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in SEARCH + GRAPH:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header
    assert lib.mde_knn_long_max_k() == lib.mde_knn_graph_long_max_k() == 256
    # the wide and narrow entries keep their bounds
    assert lib.mde_knn_max_k() == 24 and lib.mde_knn_wide_max_k() == 64 and lib.mde_knn_graph_max_k() == 64


def test_dense_search_workspace_grows_with_n_and_d():
    lib = _lib.load()
    base = _dense_ws(10000, 100)
    assert base % 1024 == 0
    assert _dense_ws(20000, 100) > base and _dense_ws(10000, 200) > base
    # 288 candidates per row against the wide search's 96: 1536 more bytes per row
    wide = C.c_size_t(0)
    assert lib.mde_knn_wide_ws_bytes(10000, 100, C.byref(wide)) == 0
    assert base - wide.value >= 1536 * 10000 - 4096
    # (the CSR workspace includes CUB's sort scratch, a device query: tests/test_gpu_knn_long.py checks it)


def test_graph_workspace_grows_with_n_and_k():
    base = _graph_ws(10000, 100)
    assert base % 1024 == 0
    assert _graph_ws(20000, 100) > base and _graph_ws(10000, 256) > _graph_ws(10000, 128) > base
    assert _graph_ws(1, 1) > 0
    # the same layout as the k <= 64 builder where both apply
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_graph_ws_bytes(10000, 64, C.byref(need)) == 0
    assert need.value == _graph_ws(10000, 64)


@pytest.mark.parametrize("n,d,k", [(300, 4, 0), (300, 4, -1), (300, 4, 257), (100, 4, 100), (257, 4, 257),
                                   (1, 4, 1), (300, 0, 65)])
def test_bad_search_shapes_are_rejected(n, d, k):
    lib = _lib.load()
    assert _dense(n, d, k) == _lib.MDE_E_INVALID
    assert _csr(n, d, 10, k) == _lib.MDE_E_INVALID
    if n < 2 or d < 1:
        need = C.c_size_t(0)
        assert lib.mde_knn_long_ws_bytes(n, d, C.byref(need)) == _lib.MDE_E_INVALID
        assert lib.mde_knn_csr_long_ws_bytes(n, d, 10, C.byref(need)) == _lib.MDE_E_INVALID
    assert _csr(300, 4, -1, 65) == _lib.MDE_E_INVALID


def test_search_null_pointers_are_rejected():
    lib = _lib.load()
    assert lib.mde_knn_long_ws_bytes(300, 4, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn_csr_long_ws_bytes(300, 4, 10, None) == _lib.MDE_E_INVALID
    for kw in ("X", "out_i", "out_d", "ws"):
        assert _dense(300, 4, 100, **{kw: None}) == _lib.MDE_E_INVALID
    for kw in ("indptr", "indices", "values", "out_i", "out_d", "ws"):
        assert _csr(300, 4, 10, 100, **{kw: None}) == _lib.MDE_E_INVALID


def test_search_workspace_too_small_or_misaligned_is_rejected():
    need = _dense_ws(1000, 30)
    assert _dense(1000, 30, 100, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _dense(1000, 30, 100, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _dense(1000, 30, 100, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _dense(1100, 30, 100, ws_bytes=need) == _lib.MDE_E_INVALID  # a larger problem


@pytest.mark.parametrize("n,k", [(10, 0), (10, -1), (10, 257), (0, 5), (-3, 5)])
def test_bad_graph_shapes_are_rejected(n, k):
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_graph_long_ws_bytes(n, k, C.byref(need)) == _lib.MDE_E_INVALID
    assert _count(n, k) == _lib.MDE_E_INVALID
    assert _emit(n, k) == _lib.MDE_E_INVALID


def test_graph_null_pointers_and_workspace_are_rejected():
    assert _lib.load().mde_knn_graph_long_ws_bytes(10, 100, None) == _lib.MDE_E_INVALID
    assert _count(10, 100, idx=None) == _lib.MDE_E_INVALID
    assert _count(10, 100, ws=None) == _lib.MDE_E_INVALID
    assert _count(10, 100, out=False) == _lib.MDE_E_INVALID
    assert _emit(10, 100, ws=None) == _lib.MDE_E_INVALID
    assert _emit(10, 100, edges=None) == _lib.MDE_E_INVALID
    assert _emit(10, 100, weights=None) == _lib.MDE_E_INVALID
    need = _graph_ws(1000, 200)
    for call in (_count, _emit):
        assert call(1000, 200, ws_bytes=need - 1) == _lib.MDE_E_INVALID
        assert call(1000, 200, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _count(1000, 256, ws_bytes=need) == _lib.MDE_E_INVALID


def test_graph_too_many_entries_are_unsupported():
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_graph_long_ws_bytes(1 << 23, 256, C.byref(need)) == _lib.MDE_E_UNSUPPORTED
    assert _count(1 << 23, 256) == _lib.MDE_E_UNSUPPORTED
    assert _emit(1 << 23, 256) == _lib.MDE_E_UNSUPPORTED
