"""CPU: the C ABI of the approximate k-nearest-neighbour search of CSR matrices (`mde_knn_approx_csr`,
include/mde_b200.h) is exported, additive (the ABI version is still 1), and rejects bad arguments before it touches a
device."""
import ctypes as C
import os

import pytest

from pymde_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
NAMES = ("mde_knn_approx_csr_ws_bytes", "mde_knn_approx_csr", "mde_knn_approx_csr_ex")


def _call(n, d, k, nnz=100, ws=FAKE, ws_bytes=1 << 40, indptr=FAKE, indices=FAKE, values=FAKE):
    lib = _lib.load()
    return lib.mde_knn_approx_csr(indptr, indices, values, n, d, nnz, k, C.c_uint64(1), FAKE, FAKE, ws, ws_bytes,
                                  None)


def _ws(n, d, nnz, k):
    b = C.c_size_t(0)
    assert _lib.load().mde_knn_approx_csr_ws_bytes(n, d, nnz, k, C.byref(b)) == 0
    return b.value


def test_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in NAMES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
        assert "int %s(" % name in header


def test_workspace_size_grows_with_rows_nonzeros_and_list_length():
    base = _ws(10000, 5000, 200000, 15)
    assert base % 1024 == 0
    assert _ws(20000, 5000, 200000, 15) > base  # n
    assert _ws(10000, 5000, 400000, 15) > base  # nnz
    assert _ws(10000, 5000, 200000, 50) > base  # K_b = 96 instead of 32
    assert _ws(10000, 5000, 200000, 24) == base  # the same K_b
    for args in ((20000, 5000, 200000, 15), (10000, 5000, 400000, 15), (10000, 5000, 200000, 50), (2, 1, 0, 1)):
        assert _ws(*args) % 1024 == 0


@pytest.mark.parametrize("n,d,nnz,k", [(1, 4, 0, 1), (10, 0, 5, 1), (10, 4, -1, 1), (10, 4, 5, 0), (100, 4, 5, 65),
                                       (10, 4, 5, 10)])
def test_workspace_query_rejects_bad_shapes(n, d, nnz, k):
    b = C.c_size_t(0)
    assert _lib.load().mde_knn_approx_csr_ws_bytes(n, d, nnz, k, C.byref(b)) == _lib.MDE_E_INVALID
    assert _lib.load().mde_knn_approx_csr_ws_bytes(10, 4, 5, 3, None) == _lib.MDE_E_INVALID


@pytest.mark.parametrize("n,d,k", [(10, 4, 0), (100, 4, 65), (30, 4, 30), (10, 4, 10), (1, 4, 1), (10, 0, 3)])
def test_bad_shapes_raise(n, d, k):
    assert _call(n, d, k) == _lib.MDE_E_INVALID
    with pytest.raises(_lib.MdeError):
        _lib.check(_call(n, d, k))


def test_negative_nnz_is_invalid():
    assert _call(10, 4, 3, nnz=-1) == _lib.MDE_E_INVALID


def test_workspace_too_small_or_misaligned_raises():
    need = _ws(1000, 300, 5000, 15)
    assert _call(1000, 300, 15, nnz=5000, ws_bytes=need - 1) == _lib.MDE_E_INVALID
    assert _call(1000, 300, 15, nnz=5000, ws=FAKE + 512, ws_bytes=need) == _lib.MDE_E_INVALID
    with pytest.raises(_lib.MdeError):
        _lib.check(_call(1000, 300, 15, nnz=5000, ws=FAKE + 8, ws_bytes=need))


def test_null_pointers_and_too_many_rows():
    lib = _lib.load()
    assert _call(10, 4, 3, indptr=None) == _lib.MDE_E_INVALID
    assert _call(10, 4, 3, indices=None) == _lib.MDE_E_INVALID
    assert _call(10, 4, 3, values=None) == _lib.MDE_E_INVALID
    assert _call(10, 4, 3, ws=None) == _lib.MDE_E_INVALID
    assert lib.mde_knn_approx_csr(FAKE, FAKE, FAKE, 10, 4, 100, 3, C.c_uint64(1), None, FAKE, FAKE, 1 << 40,
                                  None) == _lib.MDE_E_INVALID
    assert lib.mde_knn_approx_csr(FAKE, FAKE, FAKE, 10, 4, 100, 3, C.c_uint64(1), FAKE, None, FAKE, 1 << 40,
                                  None) == _lib.MDE_E_INVALID
    assert _call(1 << 31, 4, 15) == _lib.MDE_E_UNSUPPORTED
    it = C.c_int(-7)
    assert lib.mde_knn_approx_csr_ex(FAKE, FAKE, FAKE, 10, 4, 100, 65, C.c_uint64(1), FAKE, FAKE, FAKE, 1 << 40, None,
                                     C.byref(it)) == _lib.MDE_E_INVALID
    assert it.value == -7  # nothing written on a rejected call
