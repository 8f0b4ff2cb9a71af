"""CPU: the C ABI of the approximate k-nearest-neighbour search (`mde_knn_approx`, include/mde_b200.h) is exported,
additive (the ABI version is still 1), and rejects bad arguments before it touches a device."""
import ctypes as C
import os

import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call


def _call(n, d, k, ws=FAKE, ws_bytes=1 << 40):
    lib = _lib.load()
    return lib.mde_knn_approx(FAKE, n, d, k, C.c_uint64(1), FAKE, FAKE, ws, ws_bytes, None)


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in ("mde_knn_approx_max_k", "mde_knn_approx_ws_bytes", "mde_knn_approx", "mde_knn_approx_ex"):
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header


def test_workspace_size_and_limits():
    lib = _lib.load()
    assert lib.mde_knn_approx_max_k() == 64
    narrow, wide, large = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    assert lib.mde_knn_approx_ws_bytes(10000, 50, 15, C.byref(narrow)) == 0
    assert lib.mde_knn_approx_ws_bytes(10000, 50, 50, C.byref(wide)) == 0
    assert lib.mde_knn_approx_ws_bytes(20000, 50, 15, C.byref(large)) == 0
    assert 0 < narrow.value < wide.value and narrow.value < large.value
    assert narrow.value % 1024 == 0 and wide.value % 1024 == 0
    small = C.c_size_t(0)
    for n, d, k in ((1, 4, 1), (10, 0, 1), (10, 4, 0), (100, 4, 65), (10, 4, 10)):
        assert lib.mde_knn_approx_ws_bytes(n, d, k, C.byref(small)) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("n,d,k", [(10, 4, 0), (100, 4, 65), (30, 4, 30), (10, 4, 10), (1, 4, 1), (10, 0, 3)])
def test_bad_shapes_raise(n, d, k):
    assert _call(n, d, k) == _lib.MDE_E_INVALID
    with pytest.raises(_lib.MdeError):
        _lib.check(_call(n, d, k))


def test_workspace_too_small_or_misaligned_raises():
    lib = _lib.load()
    need = C.c_size_t(0)
    assert lib.mde_knn_approx_ws_bytes(1000, 8, 15, C.byref(need)) == 0
    assert _call(1000, 8, 15, ws_bytes=need.value - 1) == _lib.MDE_E_INVALID
    assert _call(1000, 8, 15, ws=FAKE + 512, ws_bytes=need.value) == _lib.MDE_E_INVALID
    with pytest.raises(_lib.MdeError):
        _lib.check(_call(1000, 8, 15, ws=FAKE + 8, ws_bytes=need.value))


def test_null_pointers_and_too_many_rows():
    lib = _lib.load()
    assert lib.mde_knn_approx(None, 10, 4, 3, C.c_uint64(1), FAKE, FAKE, FAKE, 1 << 40, None) == _lib.MDE_E_INVALID
    assert lib.mde_knn_approx(FAKE, 10, 4, 3, C.c_uint64(1), FAKE, FAKE, None, 1 << 40, None) == _lib.MDE_E_INVALID
    assert _call(1 << 31, 4, 15) == _lib.MDE_E_UNSUPPORTED
