"""CPU: the C ABI of the neighbour-graph builder (`mde_knn_graph_count` / `mde_knn_graph_emit`, include/mde_b200.h) is
exported, additive (the ABI version is still 1), and rejects bad arguments before it touches a device."""
import ctypes as C
import os

import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
NAMES = ("mde_knn_graph_max_k", "mde_knn_graph_ws_bytes", "mde_knn_graph_count", "mde_knn_graph_emit")


def _count(n, k, idx=FAKE, ws=FAKE, ws_bytes=1 << 40, out=True):
    lib = _lib.load()
    p = C.c_int64(-7)
    code = lib.mde_knn_graph_count(idx, n, k, ws, ws_bytes, C.byref(p) if out else None, None)
    assert p.value == -7  # nothing written on a refusal
    return code


def _emit(n, k, ws=FAKE, ws_bytes=1 << 40, edges=FAKE, weights=FAKE):
    return _lib.load().mde_knn_graph_emit(n, k, ws, ws_bytes, edges, weights, None)


def _ws(n, k):
    need = C.c_size_t(0)
    assert _lib.load().mde_knn_graph_ws_bytes(n, k, C.byref(need)) == 0
    return need.value


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header


def test_workspace_grows_with_n_and_k():
    assert _lib.load().mde_knn_graph_max_k() == 64
    base = _ws(10000, 15)
    assert base % 1024 == 0
    assert _ws(20000, 15) > base and _ws(10000, 16) > base and _ws(10000, 64) > _ws(10000, 24) > base
    assert _ws(1, 1) > 0
    # about 25 bytes per entry at large n k
    big, bigger = _ws(10 ** 6, 15), _ws(2 * 10 ** 6, 15)
    assert 20 * 15 * 10 ** 6 < bigger - big < 30 * 15 * 10 ** 6


@pytest.mark.parametrize("n,k", [(10, 0), (10, -1), (10, 65), (0, 5), (-3, 5)])
def test_bad_shapes_are_rejected(n, k):
    lib = _lib.load()
    need = C.c_size_t(0)
    assert lib.mde_knn_graph_ws_bytes(n, k, C.byref(need)) == _lib.MDE_E_INVALID
    assert _count(n, k) == _lib.MDE_E_INVALID
    assert _emit(n, k) == _lib.MDE_E_INVALID
    with pytest.raises(_lib.MdeError):
        _lib.check(_count(n, k))


def test_null_pointers_are_rejected():
    lib = _lib.load()
    assert lib.mde_knn_graph_ws_bytes(10, 3, None) == _lib.MDE_E_INVALID
    assert _count(10, 3, idx=None) == _lib.MDE_E_INVALID
    assert _count(10, 3, ws=None) == _lib.MDE_E_INVALID
    assert _count(10, 3, out=False) == _lib.MDE_E_INVALID
    assert _emit(10, 3, ws=None) == _lib.MDE_E_INVALID
    assert _emit(10, 3, edges=None) == _lib.MDE_E_INVALID
    assert _emit(10, 3, weights=None) == _lib.MDE_E_INVALID


def test_workspace_too_small_or_misaligned_is_rejected():
    need = _ws(1000, 15)
    for call in (_count, _emit):
        assert call(1000, 15, ws_bytes=need - 1) == _lib.MDE_E_INVALID
        assert call(1000, 15, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
        assert call(1000, 15, ws=FAKE + 8, ws_bytes=need) == _lib.MDE_E_INVALID
    # the workspace of a smaller problem is too small for a larger one
    assert _count(1100, 15, ws_bytes=need) == _lib.MDE_E_INVALID
    assert _count(1000, 20, ws_bytes=need) == _lib.MDE_E_INVALID


def test_too_many_entries_are_unsupported():
    lib = _lib.load()
    need = C.c_size_t(0)
    assert lib.mde_knn_graph_ws_bytes(1 << 26, 32, C.byref(need)) == _lib.MDE_E_UNSUPPORTED
    assert _count(1 << 26, 32) == _lib.MDE_E_UNSUPPORTED
    assert _emit(1 << 26, 32) == _lib.MDE_E_UNSUPPORTED
