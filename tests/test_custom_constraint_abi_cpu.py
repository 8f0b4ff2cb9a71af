"""CPU: the C ABI for user-defined constraints on the device solver (include/mde_b200.h, mde_constraint_part_t) is
exported and bound, it is additive (the ABI version is still 1, the built-in entry refuses the new constraint id),
its arguments are checked before any device work, and PYMDE_B200_CONSTRAINT is validated."""
import ctypes as C
import os

import pytest

from pymde_b200 import _lib, external

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        return fh.read()


def test_new_symbols_are_exported_and_declared():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    for name in ("mde_solver_create_custom", "mde_solver_set_constraint_part"):
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
    header = _header()
    for decl in ("MDE_CONSTRAINT_CUSTOM = 3", "typedef int (*mde_constraint_fn)(void* user, int which",
                 "typedef struct mde_constraint_part", "int mde_solver_create_custom(",
                 "int mde_solver_set_constraint_part("):
        assert decl in header, decl
    assert _lib.CONSTRAINT_CUSTOM == 3


def test_descriptor_layout_matches_the_header():
    """Seven pointer-sized fields in header order: u, xt, gt, retract_graph, tangent_graph, fn, user."""
    names = [f[0] for f in _lib.mde_constraint_part_t._fields_]
    assert names == ["u", "xt", "gt", "retract_graph", "tangent_graph", "fn", "user"]
    assert C.sizeof(_lib.mde_constraint_part_t) == 7 * C.sizeof(C.c_void_p)
    header = _header()
    body = header[header.index("typedef struct mde_constraint_part {"):header.index("} mde_constraint_part_t;")]
    order = [body.index(" %s;" % name) for name in names]
    assert order == sorted(order)
    # the callable-function descriptor is unchanged
    assert [f[0] for f in _lib.mde_external_t._fields_] == ["d", "fpp", "loss", "graph", "fn", "user"]


def _hook_part():
    """A hook-mode descriptor with aligned (never dereferenced) buffer addresses."""
    c = _lib.mde_constraint_part_t()
    c.u, c.xt, c.gt = 0x10000, 0x20000, 0x30000
    cb = _lib.CONSTRAINT_FN(lambda user, which, stream: 0)
    c.fn = cb
    return c, cb


def test_invalid_arguments_are_rejected_without_a_device():
    lib = _lib.load()
    handle = C.c_void_p()
    fake_edges = C.c_void_p(0x40000)  # never read: every case below fails before the edges are touched
    opts = _lib.mde_solver_opts_t()
    opts.constraint, opts.memory_size, opts.max_iter, opts.mode, opts.world_size = 3, 10, 4, 2, 1
    c, _cb = _hook_part()
    create = lambda e, o, part: lib.mde_solver_create_custom(C.byref(handle), e, 10, 2, o, None, part, None)
    assert create(None, C.byref(opts), C.byref(c)) == _lib.MDE_E_INVALID      # no edges
    assert create(fake_edges, None, C.byref(c)) == _lib.MDE_E_INVALID         # no options
    assert create(fake_edges, C.byref(opts), None) == _lib.MDE_E_INVALID      # no constraint part
    opts.world_size = 2                                                        # one GPU only
    assert create(fake_edges, C.byref(opts), C.byref(c)) == _lib.MDE_E_INVALID
    opts.world_size = 1
    opts.constraint = 0                                                        # the id must be MDE_CONSTRAINT_CUSTOM
    assert create(fake_edges, C.byref(opts), C.byref(c)) == _lib.MDE_E_INVALID
    opts.constraint = 3
    bad = _lib.mde_constraint_part_t()
    bad.u, bad.xt, bad.gt, bad.fn = 0x10000, 0x20000, 0x30004, c.fn            # gt not 16-byte aligned
    assert create(fake_edges, C.byref(opts), C.byref(bad)) == _lib.MDE_E_INVALID
    bad.gt, bad.fn = 0x30000, _lib.CONSTRAINT_FN()                              # neither graphs nor a hook
    assert create(fake_edges, C.byref(opts), C.byref(bad)) == _lib.MDE_E_INVALID
    bad.fn, bad.retract_graph = c.fn, 0x50000                                   # one graph only
    assert create(fake_edges, C.byref(opts), C.byref(bad)) == _lib.MDE_E_INVALID
    assert not handle
    assert lib.mde_solver_set_constraint_part(None, C.byref(c), None) == _lib.MDE_E_INVALID


def test_builtin_entry_refuses_the_custom_id():
    lib = _lib.load()
    handle = C.c_void_p()
    opts = _lib.mde_solver_opts_t()
    opts.constraint, opts.memory_size, opts.max_iter, opts.mode, opts.world_size = 3, 10, 4, 2, 1
    assert lib.mde_solver_create(C.byref(handle), C.c_void_p(0x40000), 10, 2, C.byref(opts), None) == \
        _lib.MDE_E_INVALID
    assert not handle


def test_constraint_mode_is_validated(monkeypatch):
    monkeypatch.delenv("PYMDE_B200_CONSTRAINT", raising=False)
    assert external.constraint_mode() is None
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "generic")
    assert external.constraint_mode() is None
    for mode in ("device", "graph", "hook"):
        monkeypatch.setenv("PYMDE_B200_CONSTRAINT", mode)
        assert external.constraint_mode() == mode
    monkeypatch.setenv("PYMDE_B200_CONSTRAINT", "fast")
    with pytest.raises(ValueError):
        external.constraint_mode()
