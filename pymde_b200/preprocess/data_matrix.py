"""Problem construction from a data matrix (interface of pymde/preprocess/data_matrix.py).

k-nearest neighbours are computed EXACTLY on the GPU by the library's own kernels (`mde_knn`: wgmma tensor-core
cross terms with a running top-32 per row and an exact fp32 re-rank, csrc/mde_knn.cu) for k <= 24, by their wide
variants (`mde_knn_wide`: a running top-96 per row in shared memory) for 24 < k <= 64; larger k uses row chunks of a
library GEMM + top-k, which measured faster than the long variant (`mde_knn_long`: a running top-288 per row, for
k <= 256) on 70 000 x 784 at every k from 65 to 256 (DESIGN section 11.6).  The reference uses scikit-learn brute force below 10 000 rows and the approximate pynndescent
above (data_matrix.py:125-143).  `PYMDE_B200_KNN=approx` opts in to an approximate search of dense input for k <= 64
(`mde_knn_approx`: NN-descent, csrc/mde_knn_approx.cu), whose cost grows about linearly in n; it returns k rows
found by the search, not necessarily the k nearest.  It pays off for large n at large d: at 10^6 rows and d = 50 the
exact search is faster (DESIGN section 11.3).  `PYMDE_B200_KNN=approx` leaves sparse input on the exact searches; for
64 < k <= 256 it takes the exact `mde_knn_long`.  A scipy.sparse matrix is searched without densifying it for k <= 256
(`mde_knn_csr`, `mde_knn_csr_wide`, `mde_knn_csr_long`, csrc/mde_knn_sparse.cu), and its pair distances come from
sorted merges of CSR rows (`mde_pair_dist_csr`).  `PYMDE_B200_KNN_SPARSE=approx` opts in to NN-descent over the CSR
rows for k <= 64 (`mde_knn_approx_csr`, csrc/mde_knn_approx.cu), with the distances of the exact sparse search
(DESIGN section 11.4); a k above 64 takes the exact long search.

A float16 / bfloat16 matrix (a torch tensor on any device, or an np.float16 array) is searched in its own precision,
without an fp32 copy: the `mde_knn16*` entries use it as the tensor-core operand and convert each element to fp32 as
the re-rank and NN-descent read it, so neighbours and distances are those of the fp32 search on the upcast matrix
(DESIGN section 11.7).  A uint8 / int8 matrix (raw pixels, genotypes, quantised embeddings) is searched the same way
by the `mde_knn8*` entries, whose tiles multiply the 8-bit values exactly on the integer tensor cores (DESIGN section
11.9), up to `mde_knn8_max_d` columns (16 512 for uint8, 43 919 for int8); a wider one is upcast.  The routing by k
and PYMDE_B200_KNN is unchanged; the GEMM path, and every other dtype, still work on an fp32 copy.

The dense exact searches are exact on data far from the origin and on far-apart clusters: the kernels centre the
columns when that bounds the score error more tightly (a 16-bit matrix near the origin stays its own exact operand)
and certify every row, searching the rows that fail directly (DESIGN section 11), and the GEMM path scores
candidates with fp64 matmuls of the centred matrix, independent of torch's TF32 setting, then re-ranks them by fp32
distance and index.

`knn_rows_device` searches only a range of rows against all rows (`mde_knn_rows`, `mde_knn16_rows`,
`mde_knn8_rows`, and `mde_knn_csr_rows` for a scipy.sparse matrix), exactly, at a cost that scales with the rows searched:
`pymde_b200.embed_new_points` searches the new rows of a stacked matrix with it (DESIGN section 11.8).  Its dense
route for k > 64 is the row range of the GEMM path; `knn_rows_device_long` instead takes a dense matrix up to k = 256
to the long row search (`mde_knn_long_rows`, `mde_knn16_long_rows`, `mde_knn8_long_rows`), which reads a 16-bit or
8-bit matrix in place and gives the rows of the full long search, certified, bit for bit."""
import ctypes as C
import os

import numpy as np
import scipy.sparse as sp
import torch

from .. import util
from .graph import EdgeListGraph, Graph
from .preprocess import sample_edges  # noqa: F401  (the reference exposes it here as well)


# element types the dense search kernels read in place -> (prefix of their C entries, MDE_DTYPE_* code or None for
# the fp32 entries, which take none; include/mde_b200.h)
_SEARCH_DTYPES = {torch.float32: ("knn", None), torch.float16: ("knn16", 1), torch.bfloat16: ("knn16", 2),
                  torch.uint8: ("knn8", 3), torch.int8: ("knn8", 4)}


def _kernel_dtype(X):
    """Whether the dense search entries read X (a tensor) in its own dtype: fp32, 16-bit, or 8-bit with at most
    `mde_knn8_max_d` columns (beyond that the integer tile sums could leave int32)."""
    fam = _SEARCH_DTYPES.get(X.dtype)
    if fam is None or fam[0] != "knn8":
        return fam is not None
    from .. import _lib
    return X.shape[-1] <= _lib.load().mde_knn8_max_d(fam[1])


def _to_device_matrix(data, device, keep_dtype=False):
    """The dense matrix on `device`, in fp32; with `keep_dtype`, a dense matrix whose dtype the search kernels read
    in place (`_kernel_dtype`: float16 / bfloat16, uint8 / int8) keeps it (uploaded at 2 or 1 bytes per value)."""
    sparse = sp.issparse(data)
    if sparse:
        data = data.toarray()
    if isinstance(data, np.ndarray):
        data = torch.from_numpy(np.ascontiguousarray(data))
    if keep_dtype and not sparse and _kernel_dtype(data):
        return data.to(device=device)
    return data.to(device=device, dtype=torch.float32)


def _entries(lib, X, suffix=""):
    """(workspace-size function, search function, leading arguments) of the dense search entry `suffix` ("", "_wide",
    "_long", "_rows", "_approx") of X's dtype: (X,) for the fp32 entries, (X, dtype code) for the others."""
    prefix, code = _SEARCH_DTYPES[X.dtype]
    name = "mde_%s%s" % (prefix, suffix)
    args = (X.data_ptr(),) if code is None else (X.data_ptr(), code)
    return getattr(lib, name + "_ws_bytes"), getattr(lib, name), args


def _to_device_csr(data, device):
    """Canonical CSR of a scipy.sparse matrix on `device`: (indptr int64 [n+1], indices int32 [nnz], values fp32
    [nnz], (n, d)), with duplicates summed and the indices of every row sorted, uploaded once."""
    A = sp.csr_matrix(data, copy=True)
    A.sum_duplicates()  # also sorts the indices of every row
    indptr = torch.from_numpy(A.indptr.astype(np.int64))
    indices = torch.from_numpy(A.indices.astype(np.int32))
    values = torch.from_numpy(A.data.astype(np.float32))
    return (indptr.to(device), indices.to(device), values.to(device)), A.shape


def knn_sparse_device(csr, shape, k):
    """(indices [n, k] int32, squared distances [n, k] fp32) of the k nearest rows of every row of a device CSR
    matrix from `_to_device_csr`, ascending by (distance, index); the kernel behind `mde_knn_csr` for k <= 24,
    `mde_knn_csr_wide` for 24 < k <= 64 and `mde_knn_csr_long` for 64 < k <= 256 (include/mde_b200.h)."""
    from .. import _lib
    lib = _lib.load()
    if k > lib.mde_knn_wide_max_k():
        ws_bytes, search = lib.mde_knn_csr_long_ws_bytes, lib.mde_knn_csr_long
    elif k > lib.mde_knn_max_k():
        ws_bytes, search = lib.mde_knn_csr_wide_ws_bytes, lib.mde_knn_csr_wide
    else:
        ws_bytes, search = lib.mde_knn_csr_ws_bytes, lib.mde_knn_csr
    indptr, indices, values = csr
    n, d = shape
    nnz = int(indices.shape[0])
    dev = indptr.device
    need = C.c_size_t(0)
    _lib.check(ws_bytes(int(n), int(d), nnz, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    d2 = torch.empty((n, k), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(search(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), int(n), int(d), nnz, int(k),
                          idx.data_ptr(), d2.data_ptr(), ws.data_ptr() + off, need.value, stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def knn_sparse_rows_device(csr, shape, k, row_begin, row_end):
    """(indices [r, k] int32, squared distances [r, k] fp32), r = row_end - row_begin: row r of the result is row
    row_begin + r of `knn_sparse_device` on the same device CSR matrix and k, bit for bit, ties included
    (`mde_knn_csr_rows`, include/mde_b200.h; 1 <= k <= 256).  The tiles sweep only the query rows, so the cost of the
    search proper scales with r n rather than n^2; the preparation still covers the whole matrix."""
    from .. import _lib
    lib = _lib.load()
    indptr, indices, values = csr
    n, d = int(shape[0]), int(shape[1])
    row_begin, row_end, k = int(row_begin), int(row_end), int(k)
    nnz = int(indices.shape[0])
    dev = indptr.device
    r = row_end - row_begin
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_csr_rows_ws_bytes(n, d, nnz, r, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((r, k), dtype=torch.int32, device=dev)
    d2 = torch.empty((r, k), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.mde_knn_csr_rows(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), n, d, nnz,
                                        row_begin, row_end, k, idx.data_ptr(), d2.data_ptr(), ws.data_ptr() + off,
                                        need.value, stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def knn_approx_sparse_device(csr, shape, k, seed=None):
    """(indices [n, k] int32, squared distances [n, k] fp32) of k rows found for every row of a device CSR matrix from
    `_to_device_csr` by NN-descent, ascending by (distance, index), with the distances of `knn_sparse_device`
    (`mde_knn_approx_csr`, include/mde_b200.h).  `seed` defaults to a draw from the module RNG, so
    `pymde_b200.seed(s)` reproduces the result."""
    from .. import _lib
    lib = _lib.load()
    if seed is None:
        seed = int(util.np_rng().integers(0, 2 ** 62))
    indptr, indices, values = csr
    n, d = shape
    nnz = int(indices.shape[0])
    dev = indptr.device
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_approx_csr_ws_bytes(int(n), int(d), nnz, int(k), C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    d2 = torch.empty((n, k), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.mde_knn_approx_csr(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), int(n), int(d),
                                          nnz, int(k), C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(),
                                          ws.data_ptr() + off, need.value, stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def _pair_dist_csr(csr, shape, pairs):
    """||x_a - x_b|| (fp32, fp64 sums) of the device int64 row pairs [p, 2] of a device CSR matrix."""
    from .. import _lib
    lib = _lib.load()
    indptr, indices, values = csr
    pairs = pairs.to(dtype=torch.int64).contiguous()
    out = torch.empty(pairs.shape[0], dtype=torch.float32, device=pairs.device)
    with torch.cuda.device(pairs.device):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.mde_pair_dist_csr(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), int(shape[0]),
                                         int(shape[1]), pairs.data_ptr(), int(pairs.shape[0]), out.data_ptr(),
                                         stream))
    return out


def _knn_graph(idx, d2, n, max_distance, dev):
    keep = torch.ones_like(d2, dtype=torch.bool) if max_distance is None else d2.sqrt() <= max_distance
    i = torch.arange(n, device=dev)[:, None].expand_as(idx)
    e = torch.stack([i[keep], idx[keep].long()], 1).cpu()
    return Graph.from_edges(e, None, n_items=n)


def knn_device(X, k):
    """(indices [n, k] int32, squared distances [n, k] fp32) of the k nearest rows of every row of the CUDA fp32
    matrix X, ascending; the wgmma kernel behind `mde_knn` for k <= 24, `mde_knn_wide` for 24 < k <= 64 and
    `mde_knn_long` for 64 < k <= 256 (include/mde_b200.h).  A float16 / bfloat16 X is read in place by the
    `mde_knn16*` entries and a uint8 / int8 X by the `mde_knn8*` entries (upcast above `mde_knn8_max_d` columns),
    with the result of X.float()."""
    from .. import _lib
    lib = _lib.load()
    X = (X if _kernel_dtype(X) else X.float()).contiguous()
    suffix = "_long" if k > lib.mde_knn_wide_max_k() else "_wide" if k > lib.mde_knn_max_k() else ""
    ws_bytes, search, args = _entries(lib, X, suffix)
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check(ws_bytes(int(n), int(d), C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=X.device)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device=X.device)
    d2 = torch.empty((n, k), dtype=torch.float32, device=X.device)
    with torch.cuda.device(X.device):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(search(*args, int(n), int(d), int(k), idx.data_ptr(), d2.data_ptr(), ws.data_ptr() + off,
                          need.value, stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def knn_rows_device(X, k, row_begin, row_end):
    """(indices [r, k], squared distances [r, k] fp32), r = row_end - row_begin: row r of the result is row
    row_begin + r of the exact search of X (its k nearest rows among all n rows of X, itself excluded, ascending by
    (distance, index)).  Always exact: PYMDE_B200_KNN does not apply.  Routes:
      * a CUDA fp32 / float16 / bfloat16 / uint8 / int8 matrix with k <= 64: `mde_knn_rows` / `mde_knn16_rows` /
        `mde_knn8_rows` (int32 indices), bit for bit the rows of `knn_device`, at a cost of about r n d rather than
        n^2 d (other dtypes, and 8-bit matrices wider than `mde_knn8_max_d`, are searched in fp32);
      * a dense matrix with k > 64: the row range of `_gemm_search` (int64 indices), the rows it gives on all of X;
      * a scipy.sparse matrix with k <= 256: `knn_sparse_rows_device` (`mde_knn_csr_rows`, int32 indices), bit for
        bit the rows of `knn_sparse_device`, at a cost of about r n rather than n^2 in the tiles, without densifying;
      * a scipy.sparse matrix with k > 256: the row range of `_gemm_search` on the dense matrix."""
    from .. import _lib
    lib = _lib.load()
    n = int(X.shape[0])
    row_begin, row_end, k = int(row_begin), int(row_end), int(k)
    if not 0 <= row_begin < row_end <= n:
        raise ValueError("need 0 <= row_begin < row_end <= n; got [%d, %d) with n = %d" % (row_begin, row_end, n))
    if not 1 <= k <= n - 1:
        raise ValueError("need 1 <= k <= n - 1; got k = %d with n = %d" % (k, n))
    if sp.issparse(X):
        dev = util.cuda_device()
        if k > lib.mde_knn_long_max_k():
            return _gemm_search(_to_device_matrix(X, dev), k, row_begin=row_begin, row_end=row_end)
        return knn_sparse_rows_device(*_to_device_csr(X, dev), k, row_begin, row_end)
    X = (X if _kernel_dtype(X) else X.float()).contiguous()
    if k > lib.mde_knn_wide_max_k():
        return _gemm_search(X.float(), k, row_begin=row_begin, row_end=row_end)
    return _dense_rows(lib, X, k, row_begin, row_end, "_rows")


def knn_rows_device_long(X, k, row_begin, row_end):
    """(indices [r, k] int32, squared distances [r, k] fp32), r = row_end - row_begin, for 1 <= k <= 256: row r of
    the result is row row_begin + r of the full long search of X (`knn_device` at k > 64), bit for bit, ties included;
    always exact (PYMDE_B200_KNN does not apply).  Routes:
      * a CUDA fp32 / float16 / bfloat16 / uint8 / int8 matrix: `mde_knn_long_rows` / `mde_knn16_long_rows` /
        `mde_knn8_long_rows`, read in place, at a cost of about r n d (the candidate sweep is split across the SMs
        when the query rows are few, DESIGN section 11.8); other dtypes, and 8-bit matrices wider than
        `mde_knn8_max_d`, are searched in fp32;
      * a scipy.sparse matrix: `knn_sparse_rows_device` (`mde_knn_csr_rows`), without densifying it.
    ValueError for a bad range or a k outside [1, min(256, n - 1)]."""
    from .. import _lib
    lib = _lib.load()
    n = int(X.shape[0])
    row_begin, row_end, k = int(row_begin), int(row_end), int(k)
    max_k = int(lib.mde_knn_long_max_k())
    if not 1 <= k <= max_k:
        raise ValueError("need 1 <= k <= %d; got k = %d" % (max_k, k))
    if not 0 <= row_begin < row_end <= n:
        raise ValueError("need 0 <= row_begin < row_end <= n; got [%d, %d) with n = %d" % (row_begin, row_end, n))
    if k > n - 1:
        raise ValueError("need 1 <= k <= n - 1; got k = %d with n = %d" % (k, n))
    if sp.issparse(X):
        return knn_sparse_rows_device(*_to_device_csr(X, util.cuda_device()), k, row_begin, row_end)
    if not (isinstance(X, torch.Tensor) and X.is_cuda):  # a host matrix is uploaded in its own dtype
        X = _to_device_matrix(X, util.cuda_device(), keep_dtype=True)
    X = (X if _kernel_dtype(X) else X.float()).contiguous()
    return _dense_rows(lib, X, k, row_begin, row_end, "_long_rows")


def _dense_rows(lib, X, k, row_begin, row_end, suffix):
    """The row-range entry `suffix` ("_rows" or "_long_rows") of X's dtype on rows [row_begin, row_end) of the CUDA
    matrix X: (indices [r, k] int32, squared distances [r, k] fp32)."""
    from .. import _lib
    ws_bytes, search, args = _entries(lib, X, suffix)
    n, d, r = int(X.shape[0]), int(X.shape[1]), row_end - row_begin
    need = C.c_size_t(0)
    _lib.check(ws_bytes(n, d, r, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=X.device)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((r, k), dtype=torch.int32, device=X.device)
    d2 = torch.empty((r, k), dtype=torch.float32, device=X.device)
    with torch.cuda.device(X.device):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(search(*args, n, d, row_begin, row_end, k, idx.data_ptr(), d2.data_ptr(), ws.data_ptr() + off,
                          need.value, stream, None))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def knn_approx_device(X, k, seed=None):
    """(indices [n, k] int32, squared distances [n, k] fp32) of k rows found for every row of the CUDA fp32 matrix X
    by NN-descent, ascending by (distance, index), with the exact fp32 distances of `knn_device`
    (`mde_knn_approx`, include/mde_b200.h).  `seed` defaults to a draw from the module RNG, so `pymde_b200.seed(s)`
    reproduces the result.  A float16 / bfloat16 X is read in place (`mde_knn16_approx`), and so is a uint8 / int8 X
    (`mde_knn8_approx`), with the result of X.float()."""
    from .. import _lib
    lib = _lib.load()
    if seed is None:
        seed = int(util.np_rng().integers(0, 2 ** 62))
    X = (X if _kernel_dtype(X) else X.float()).contiguous()
    n, d = X.shape
    ws_bytes, search, args = _entries(lib, X, "_approx")
    need = C.c_size_t(0)
    _lib.check(ws_bytes(int(n), int(d), int(k), C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=X.device)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device=X.device)
    d2 = torch.empty((n, k), dtype=torch.float32, device=X.device)
    with torch.cuda.device(X.device):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(search(*args, int(n), int(d), int(k), C.c_uint64(seed), idx.data_ptr(), d2.data_ptr(),
                          ws.data_ptr() + off, need.value, stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def _search(data, k, dev, chunk_rows=None):
    """The neighbour search of `k_nearest_neighbors`: (idx [n, k'], squared distances [n, k'] fp32, n) of the
    k' = min(k, n - 1) nearest rows of every row, from the search kernels (int32 indices), or from row chunks of a
    library GEMM + top-k (int64 indices) for k' > 256, dense input with 64 < k' <= 256 (unless PYMDE_B200_KNN=approx),
    `chunk_rows` or PYMDE_B200_KNN=gemm.  A dense float16 / bfloat16 / uint8 / int8 matrix stays in its dtype on the
    search kernels (`_kernel_dtype`) and is upcast for the GEMM path."""
    from .. import _lib
    lib = _lib.load()
    mode = os.environ.get("PYMDE_B200_KNN", "kernel")
    use_kernel = chunk_rows is None and mode != "gemm"
    if sp.issparse(data):
        n = data.shape[0]
        k = int(min(k, n - 1))
        if use_kernel and 1 <= k <= lib.mde_knn_long_max_k():
            csr, shape = _to_device_csr(data, dev)
            # PYMDE_B200_KNN=approx does not reach here: sparse input has its own opt-in
            # NN-descent covers k <= 64; above that PYMDE_B200_KNN_SPARSE=approx takes the exact long search
            if os.environ.get("PYMDE_B200_KNN_SPARSE") == "approx" and k <= lib.mde_knn_approx_max_k():
                idx, d2 = knn_approx_sparse_device(csr, shape, k)
            else:
                idx, d2 = knn_sparse_device(csr, shape, k)
            return idx, d2, n
    X = _to_device_matrix(data, dev, keep_dtype=True)
    n = X.shape[0]
    k = int(min(k, n - 1))
    if use_kernel and 1 <= k <= lib.mde_knn_wide_max_k():
        # "approx" applies to dense input only: scipy.sparse input keeps the exact sparse searches above
        idx, d2 = knn_approx_device(X, k) if mode == "approx" else knn_device(X, k)
        return idx, d2, n
    if use_kernel and mode == "approx" and k <= lib.mde_knn_long_max_k():
        # above NN-descent's k the opt-in takes the exact long search (mde_knn_long); by default 64 < k <= 256 stays
        # on the GEMM path below, which measured faster on 70 000 x 784 at k = 65 .. 256 (DESIGN section 11.6)
        idx, d2 = knn_device(X, k)
        return idx, d2, n
    idx, d2 = _gemm_search(X.float(), k, chunk_rows)
    return idx, d2, n


def _gemm_search(X, k, chunk_rows=None, row_begin=0, row_end=None):
    """(idx [n, k] int64, squared distances [n, k] fp32) of the k nearest rows of every row of the device fp32 matrix
    X, by row chunks of a library GEMM: candidate scores ||x||^2 - 2 q.x of the fp64 column-centred matrix (fp64
    matmuls, whatever torch.backends.cuda.matmul.allow_tf32 says; centring keeps the cancellation of data far from the
    origin out of the scores), the k + 8 best kept, then re-ranked by their fp32 squared distances (sum of squared fp32
    differences) and index, ascending.  With a row range, only the chunks of the full search that hold rows
    [row_begin, row_end) are searched (against all n rows), with the same arithmetic, and those rows returned: the
    rows the full search gives, bit for bit."""
    n, d = X.shape
    row_end = n if row_end is None else row_end
    dev = X.device
    Xd = X.double()
    Xd -= Xd.mean(0)
    sq = (Xd * Xd).sum(1)
    kc = min(k + 8, n - 1)
    rows = chunk_rows or max(256, min(n, int(2 ** 26 // max(n, 1))))
    sub = max(1, int(2 ** 26 // max(kc * d, 1)))  # rows per fp32 re-rank batch (256 MB of differences)
    idxs, vals = [], []
    first = row_begin // rows * rows
    for s0 in range(first, row_end, rows):
        Q = Xd[s0:s0 + rows]
        score = sq[None, :] - 2.0 * (Q @ Xd.T)  # ||q||^2 is constant along a row
        score[torch.arange(Q.shape[0], device=dev), torch.arange(s0, s0 + Q.shape[0], device=dev)] = float("inf")
        cand = torch.topk(score, kc, dim=1, largest=False)[1]
        del score
        cand = torch.sort(cand, 1)[0]  # index order, so that the stable sort below breaks ties by index
        for r0 in range(0, cand.shape[0], sub):
            c = cand[r0:r0 + sub]
            d2 = ((X[s0 + r0:s0 + r0 + c.shape[0], None, :] - X[c]) ** 2).sum(-1)
            d2, pos = torch.sort(d2, dim=1, stable=True)
            idxs.append(torch.gather(c, 1, pos[:, :k])); vals.append(d2[:, :k])
    lo, hi = row_begin - first, row_end - first
    return torch.cat(idxs)[lo:hi], torch.cat(vals)[lo:hi]


def k_nearest_neighbors(data, k, max_distance=None, verbose=False, device=None, chunk_rows=None):
    """Graph whose edges join each row to its k nearest rows (Euclidean); reciprocal pairs get weight 2."""
    dev = util.cuda_device(device)
    idx, d2, n = _search(data, k, dev, chunk_rows)
    return _knn_graph(idx, d2, n, max_distance, dev)


def _device_knn_graph(data, k, max_distance, device, max_k):
    """`k_nearest_neighbors`' graph assembled on the device; ValueError when min(k, n - 1) > max_k."""
    from .graph import knn_edge_list
    n = data.shape[0]
    if min(k, n - 1) > max_k:
        raise ValueError("min(k, n - 1) must be at most %d (use k_nearest_neighbors, which builds the host Graph)"
                         % max_k)
    dev = util.cuda_device(device)
    idx, d2, n = _search(data, k, dev)
    if max_distance is not None:
        idx = torch.where(d2.sqrt() <= max_distance, idx, -1)  # (a NaN distance is dropped, as in _knn_graph)
    return knn_edge_list(idx, n)


def k_nearest_neighbors_device(data, k, max_distance=None, device=None):
    """The graph of `k_nearest_neighbors` -- same search, same edges and weights -- assembled on the device from the
    neighbour lists (`graph.knn_edge_list`) and returned as an `EdgeListGraph` there.  The lists of the search
    kernels and of PYMDE_B200_KNN=gemm qualify when min(k, n - 1) <= 64; larger k raises ValueError (use
    `k_nearest_neighbors_device_long` up to 256, or `k_nearest_neighbors`, which builds the host Graph)."""
    from .. import _lib
    return _device_knn_graph(data, k, max_distance, device, int(_lib.load().mde_knn_graph_max_k()))


def k_nearest_neighbors_device_long(data, k, max_distance=None, device=None):
    """`k_nearest_neighbors_device` for min(k, n - 1) <= 256 (`mde_knn_graph_long_max_k()`); larger k raises
    ValueError."""
    from .. import _lib
    return _device_knn_graph(data, k, max_distance, device, int(_lib.load().mde_knn_graph_long_max_k()))


def _pair_distances(data, retain_fraction, dev):
    """(pairs [p, 2] int64 with i < j, Euclidean distances [p] fp32, n) of `distances`, on the device: all pairs in
    row-major order, or `sample_edges`' sample in its draw order.  A dense float16 / bfloat16 / uint8 / int8 matrix
    stays in its dtype; each chunk of pairs is upcast, which gives the distances of the fp32 matrix."""
    if sp.issparse(data):
        csr, shape = _to_device_csr(data, dev)
        n = shape[0]
    else:
        X = _to_device_matrix(data, dev, keep_dtype=True)
        n = X.shape[0]
    n_all = n * (n - 1) // 2
    if retain_fraction >= 1.0:
        edges = torch.triu_indices(n, n, 1, device=dev).T
    else:
        edges = sample_edges(n, int(retain_fraction * n_all), device=dev)
    if sp.issparse(data):
        return edges, _pair_dist_csr(csr, shape, edges), n
    out = torch.empty(edges.shape[0], dtype=torch.float32, device=dev)
    step = 1 << 22
    for s0 in range(0, edges.shape[0], step):
        e = edges[s0:s0 + step]
        out[s0:s0 + step] = (X[e[:, 0]].float() - X[e[:, 1]].float()).norm(dim=1)
    return edges, out, n


def distances(data, retain_fraction=1.0, verbose=False, device=None):
    """Graph of pairwise Euclidean distances: all (n choose 2) pairs, or a uniform sample of them."""
    dev = util.cuda_device(device)
    edges, out, n = _pair_distances(data, retain_fraction, dev)
    return Graph.from_edges(edges.cpu(), out.cpu(), n_items=n)


def distances_device(data, retain_fraction=1.0, device=None):
    """The graph of `distances` -- same pairs, same draws, same distance bits -- as an `EdgeListGraph` on the
    device: the pairs sorted by (i, j), without the zero and +inf distances that `Graph` drops (NaN is kept)."""
    dev = util.cuda_device(device)
    edges, out, n = _pair_distances(data, retain_fraction, dev)
    order = torch.argsort(edges[:, 0] * n + edges[:, 1])  # (the pairs are distinct: no ties)
    edges, out = edges[order], out[order]
    keep = (out != 0) & (out != float("inf"))
    return EdgeListGraph(edges[keep], out[keep], n)
