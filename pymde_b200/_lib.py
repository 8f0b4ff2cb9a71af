"""ctypes binding of libmde_b200.so (the C ABI declared in include/mde_b200.h).

This is the stub a maintainer of the reference would add to reach the CUDA path (see
INTEGRATION.md).  There is NO fallback: if the shared library is missing or a call fails,
an exception is raised -- the product never routes around the CUDA extension.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmde_b200.so")

# error codes (include/mde_b200.h)
MDE_E_INVALID, MDE_E_UNSUPPORTED, MDE_E_NAN, MDE_E_ALLOC, MDE_E_COMM = -1, -2, -3, -4, -5
IPC_HANDLE_BYTES = 64
CONSTRAINT_CENTERED, CONSTRAINT_STANDARDIZED, CONSTRAINT_ANCHORED, CONSTRAINT_CUSTOM = 0, 1, 2, 3
DTYPE_FP16, DTYPE_BF16 = 1, 2  # MDE_DTYPE_* element codes of the mde_knn16* searches
DTYPE_U8, DTYPE_S8 = 3, 4  # and of the mde_knn8* searches


class MdeError(RuntimeError):
    def __init__(self, code, msg):
        super(MdeError, self).__init__("libmde_b200: %s (code %d)" % (msg, code))
        self.code = code


class mde_fn_t(C.Structure):
    _fields_ = [("fn_att", C.c_int32), ("fn_rep", C.c_int32), ("att", C.c_float * 3),
                ("rep", C.c_float * 3), ("push_pull", C.c_int32)]


class mde_solver_opts_t(C.Structure):
    _fields_ = [("constraint", C.c_int32), ("memory_size", C.c_int32), ("max_iter", C.c_int32),
                ("mode", C.c_int32), ("n_anchors", C.c_int64), ("anchors", C.c_void_p),
                ("anchor_values", C.c_void_p), ("world_size", C.c_int32), ("reserved", C.c_int32)]


class mde_ell_host_t(C.Structure):
    """Host copy of the ELL pull records (include/mde_b200.h; CPU tests decode it)."""
    _fields_ = [("rec", C.POINTER(C.c_ubyte)), ("rec_off", C.POINTER(C.c_uint32)),
                ("bkt_tile", C.POINTER(C.c_int32)), ("bkt_wt0", C.POINTER(C.c_int32)),
                ("cta_wt0", C.POINTER(C.c_int32)), ("cta_bkt0", C.POINTER(C.c_int32)),
                ("rec_bytes", C.c_int64), ("nrec", C.c_int64), ("nslots", C.c_int64), ("nentries", C.c_int64),
                ("npadded", C.c_int64), ("nbkt", C.c_int32), ("ncta", C.c_int32), ("tile_rows_log2", C.c_int32),
                ("reserved", C.c_int32)]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p)
# (user, d, fpp, loss, stream) -> int: the caller's part of an evaluation of a callable distortion function
EXTERNAL_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)


class mde_external_t(C.Structure):
    _fields_ = [("d", C.c_void_p), ("fpp", C.c_void_p), ("loss", C.c_void_p), ("graph", C.c_void_p),
                ("fn", EXTERNAL_FN), ("user", C.c_void_p)]


# (user, which: 0 retract / 1 tangent, stream) -> int: the caller's part of a user-defined constraint
CONSTRAINT_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_void_p)


class mde_constraint_part_t(C.Structure):
    _fields_ = [("u", C.c_void_p), ("xt", C.c_void_p), ("gt", C.c_void_p), ("retract_graph", C.c_void_p),
                ("tangent_graph", C.c_void_p), ("fn", CONSTRAINT_FN), ("user", C.c_void_p)]

# name -> (restype, argtypes); every symbol include/mde_b200.h declares
SIGNATURES = {
    "mde_abi_version": (C.c_int, []),
    "mde_error_string": (C.c_char_p, [C.c_int]),
    "mde_launch_count": (C.c_uint64, []),
    "mde_edges_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                   C.c_void_p, C.POINTER(mde_fn_t), C.c_int64, C.c_void_p]),
    "mde_edges_create_ex": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.POINTER(mde_fn_t), C.c_int64, C.c_int, C.c_void_p]),
    "mde_edges_destroy": (C.c_int, [C.c_void_p]),
    "mde_edges_count": (C.c_int64, [C.c_void_p]),
    "mde_edges_nbytes": (C.c_int64, [C.c_void_p]),
    "mde_edges_kind": (C.c_int, [C.c_void_p]),
    "mde_edges_deterministic": (C.c_int, [C.c_void_p]),
    "mde_ell_host_layout": (C.c_int, [C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_int, C.c_int, C.POINTER(mde_ell_host_t)]),
    "mde_ell_device_layout": (C.c_int, [C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_int, C.c_int, C.POINTER(mde_ell_host_t), C.c_void_p]),
    "mde_ell_host_free": (None, [C.POINTER(mde_ell_host_t)]),
    "mde_distortion": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mde_edge_outputs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mde_function_eval": (C.c_int, [C.POINTER(mde_fn_t), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_void_p, C.c_void_p]),
    "mde_scatter_external": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mde_project_ws_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "mde_project_centered": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "mde_project_standardized": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "mde_project_status": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_void_p]),
    "mde_tangent_standardized": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "mde_solver_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int,
                                    C.POINTER(mde_solver_opts_t), C.c_void_p]),
    "mde_solver_destroy": (C.c_int, [C.c_void_p]),
    "mde_solver_begin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]),
    "mde_solver_begin_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p]),
    "mde_solver_run": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]),
    "mde_solver_debug_times": (C.c_int, [C.c_void_p, C.POINTER(C.c_ulonglong), C.c_void_p]),
    "mde_solver_debug_run_steps": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "mde_solver_debug_lbfgs": (C.c_int, [C.c_void_p] + [C.c_void_p] * 5 + [C.POINTER(C.c_int), C.POINTER(C.c_double),
                                                                          C.POINTER(C.c_int), C.c_void_p]),
    "mde_solver_x": (C.c_void_p, [C.c_void_p]),
    "mde_solver_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_int64), C.c_void_p]),
    "mde_solver_set_allreduce": (C.c_int, [C.c_void_p, ALLREDUCE_FN, C.c_void_p]),
    "mde_solver_create_external": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int,
                                             C.POINTER(mde_solver_opts_t), C.POINTER(mde_external_t), C.c_void_p]),
    "mde_solver_set_external": (C.c_int, [C.c_void_p, C.POINTER(mde_external_t), C.c_void_p]),
    "mde_solver_create_custom": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int,
                                           C.POINTER(mde_solver_opts_t), C.POINTER(mde_external_t),
                                           C.POINTER(mde_constraint_part_t), C.c_void_p]),
    "mde_solver_set_constraint_part": (C.c_int, [C.c_void_p, C.POINTER(mde_constraint_part_t), C.c_void_p]),
    "mde_knn_max_k": (C.c_int, []),
    "mde_knn_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                          C.c_void_p]),
    "mde_knn_ex": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_csr_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.POINTER(C.c_size_t)]),
    "mde_knn_csr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_void_p,
                              C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn_csr_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_wide_max_k": (C.c_int, []),
    "mde_knn_wide_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_wide": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_size_t, C.c_void_p]),
    "mde_knn_wide_ex": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_csr_wide_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.POINTER(C.c_size_t)]),
    "mde_knn_csr_wide": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn_csr_wide_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_long_max_k": (C.c_int, []),
    "mde_knn_long_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_long": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_size_t, C.c_void_p]),
    "mde_knn_long_ex": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_csr_long_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.POINTER(C.c_size_t)]),
    "mde_knn_csr_long": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn_csr_long_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_approx_max_k": (C.c_int, []),
    "mde_knn_approx_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_approx": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn_approx_ex": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn16_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn16": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                            C.c_size_t, C.c_void_p]),
    "mde_knn16_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn16_wide_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn16_wide": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn16_wide_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn16_long_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn16_long": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn16_long_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_long_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_long_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_dbg_knn_long_slices": (C.c_int, [C.c_int64, C.c_int64, C.c_int]),  # host-only (CPU tests)
    "mde_knn16_long_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn16_long_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn8_long_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn8_long_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn16_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn16_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_csr_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int,
                                            C.POINTER(C.c_size_t)]),
    "mde_knn_csr_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64,
                                   C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn_csr_rows_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64,
                                      C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.POINTER(C.c_int)]),
    "mde_knn16_approx_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn16_approx": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn16_approx_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn8_max_d": (C.c_int, [C.c_int]),
    "mde_knn8_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn8": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                           C.c_size_t, C.c_void_p]),
    "mde_knn8_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn8_wide_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn8_wide": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn8_wide_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn8_long_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn8_long": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn8_long_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn8_approx_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn8_approx": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn8_approx_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn8_rows_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn8_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]),
    "mde_knn_approx_csr_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_approx_csr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                     C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mde_knn_approx_csr_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                        C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                        C.POINTER(C.c_int)]),
    "mde_pair_dist_csr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_void_p]),
    "mde_knn_graph_max_k": (C.c_int, []),
    "mde_knn_graph_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_graph_count": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64),
                                      C.c_void_p]),
    "mde_knn_graph_emit": (C.c_int, [C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "mde_knn_graph_long_max_k": (C.c_int, []),
    "mde_knn_graph_long_ws_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "mde_knn_graph_long_count": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_size_t,
                                           C.POINTER(C.c_int64), C.c_void_p]),
    "mde_knn_graph_long_emit": (C.c_int, [C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                          C.c_void_p]),
    "mde_graph_hops_ws_bytes":(C.c_int64, [C.c_int64]),
    "mde_graph_hops": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_double,
                                 C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                 C.c_int64, C.c_void_p]),
    "mde_graph_sssp_ws_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "mde_graph_sssp": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_double,
                                 C.c_double, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                 C.c_void_p, C.c_int64, C.c_void_p]),
    "mde_graph_knn_max_k": (C.c_int, []),
    "mde_graph_knn_ws_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "mde_graph_knn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_double, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "mde_graph_knn_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int,
                                     C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "mde_graph_knn_long_max_k": (C.c_int, []),
    "mde_graph_knn_long": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_double, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "mde_graph_knn_long_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                          C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_void_p]),
    "mde_solver_comm_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
    "mde_solver_comm_connect": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
}

# host-only debug entry points (scalar solver logic; used by CPU tests)
DEBUG_SIGNATURES = {
    "mde_dbg_ls_new": (C.c_void_p, [C.c_double, C.c_double, C.c_float, C.c_float]),
    "mde_dbg_ls_free": (None, [C.c_void_p]),
    "mde_dbg_feed_policy": (C.c_int, [C.c_int64, C.c_int64]),
    "mde_dbg_ls_t": (C.c_double, [C.c_void_p]),
    "mde_dbg_ls_step": (C.c_int, [C.c_void_p, C.c_double, C.c_float, C.c_int]),
    "mde_dbg_ls_result": (None, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                 C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mde_dbg_lbfgs_new": (C.c_void_p, [C.c_int]),
    "mde_dbg_lbfgs_free": (None, [C.c_void_p]),
    "mde_dbg_lbfgs_step": (None, [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double] +
                           [C.POINTER(C.c_double)] * 5 +
                           [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double),
                            C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "mde_dbg_lbfgs_reset": (None, [C.c_void_p]),
    "mde_dbg_lbfgs_cand": (C.c_int, [C.c_void_p]),
    "mde_dbg_knn_slices": (C.c_int, [C.c_int64, C.c_int64, C.c_int]),
    "mde_dbg_knn_csr_slices": (C.c_int, [C.c_int64, C.c_int64, C.c_int]),
    "mde_dbg_knn8_gamma": (C.c_double, [C.c_int]),
}

_lib = None


def load():
    """Load libmde_b200.so; raises (never falls back) if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MdeError(MDE_E_INVALID, "shared library not built: %s (run `python -c 'import __graft_entry__ as g; "
                       "g.build()'` or pymde_b200/csrc/build.sh)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for table in (SIGNATURES, DEBUG_SIGNATURES):
        for name, (res, args) in table.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
    _lib = lib
    return lib


def check(code):
    if code != 0:
        lib = load()
        raise MdeError(code, lib.mde_error_string(code).decode())
    return code
