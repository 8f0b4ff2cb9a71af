"""CPU: the C ABI for callable distortion functions on the device solver (include/mde_b200.h, mde_external_t) is
exported and bound, it is additive (the ABI version is still 1), and PYMDE_B200_EXTERNAL is validated."""
import ctypes as C
import os

import pytest

from pymde_b200 import _lib, external

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_symbols_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    for name in ("mde_solver_create_external", "mde_solver_set_external"):
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for decl in ("typedef struct mde_external", "int mde_solver_create_external(", "int mde_solver_set_external("):
        assert decl in header


def test_descriptor_layout_matches_the_header():
    """Six pointer-sized fields in header order: d, fpp, loss, graph, fn, user."""
    names = [f[0] for f in _lib.mde_external_t._fields_]
    assert names == ["d", "fpp", "loss", "graph", "fn", "user"]
    assert C.sizeof(_lib.mde_external_t) == 6 * C.sizeof(C.c_void_p)


def test_null_arguments_are_rejected_without_a_device():
    lib = _lib.load()
    x = _lib.mde_external_t()
    handle = C.c_void_p()
    opts = _lib.mde_solver_opts_t()
    opts.world_size = 2  # callables run on one GPU only
    assert lib.mde_solver_create_external(C.byref(handle), None, 10, 2, C.byref(opts), C.byref(x), None) == \
        _lib.MDE_E_INVALID
    assert lib.mde_solver_set_external(None, C.byref(x), None) == _lib.MDE_E_INVALID


def test_forced_mode_is_validated(monkeypatch):
    monkeypatch.delenv("PYMDE_B200_EXTERNAL", raising=False)
    assert external.forced_mode() is None
    for mode in ("graph", "hook", "generic"):
        monkeypatch.setenv("PYMDE_B200_EXTERNAL", mode)
        assert external.forced_mode() == mode
    monkeypatch.setenv("PYMDE_B200_EXTERNAL", "fast")
    with pytest.raises(ValueError):
        external.forced_mode()
