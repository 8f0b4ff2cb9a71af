"""Problem construction from a data matrix (interface of pymde/preprocess/data_matrix.py).

k-nearest neighbours are computed EXACTLY on the GPU by the library's own kernel (`mde_knn`: wgmma tensor-core
cross terms with a running top-32 per row and an exact fp32 re-rank, csrc/mde_knn.cu) for k <= 24; larger k uses row
chunks of a library GEMM + top-k.  The reference uses scikit-learn brute force below 10 000 rows and the approximate
pynndescent above (data_matrix.py:125-143)."""
import ctypes as C
import os

import numpy as np
import scipy.sparse as sp
import torch

from .. import util
from .graph import Graph
from .preprocess import sample_edges  # noqa: F401  (the reference exposes it here as well)


def _to_device_matrix(data, device):
    if sp.issparse(data):
        data = data.toarray()
    if isinstance(data, np.ndarray):
        data = torch.from_numpy(np.ascontiguousarray(data))
    return data.to(device=device, dtype=torch.float32)


def knn_device(X, k):
    """(indices [n, k] int32, squared distances [n, k] fp32) of the k nearest rows of every row of the CUDA fp32
    matrix X, ascending; the wgmma kernel behind `mde_knn` (include/mde_b200.h)."""
    from .. import _lib
    lib = _lib.load()
    X = X.contiguous()
    n, d = X.shape
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_ws_bytes(int(n), int(d), C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=X.device)
    off = (-ws.data_ptr()) % 1024
    idx = torch.empty((n, k), dtype=torch.int32, device=X.device)
    d2 = torch.empty((n, k), dtype=torch.float32, device=X.device)
    with torch.cuda.device(X.device):
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.mde_knn(X.data_ptr(), int(n), int(d), int(k), idx.data_ptr(), d2.data_ptr(),
                               ws.data_ptr() + off, need.value, stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return idx, d2


def k_nearest_neighbors(data, k, max_distance=None, verbose=False, device=None, chunk_rows=None):
    """Graph whose edges join each row to its k nearest rows (Euclidean); reciprocal pairs get weight 2."""
    dev = util.cuda_device(device)
    X = _to_device_matrix(data, dev)
    n = X.shape[0]
    k = int(min(k, n - 1))
    from .. import _lib
    if (chunk_rows is None and 1 <= k <= _lib.load().mde_knn_max_k()
            and os.environ.get("PYMDE_B200_KNN", "kernel") != "gemm"):
        idx, d2 = knn_device(X, k)
        keep = torch.ones_like(d2, dtype=torch.bool) if max_distance is None else d2.sqrt() <= max_distance
        i = torch.arange(n, device=dev)[:, None].expand_as(idx)
        e = torch.stack([i[keep], idx[keep].long()], 1).cpu()
        return Graph.from_edges(e, None, n_items=n)
    sq = (X * X).sum(1)
    rows = chunk_rows or max(256, min(n, int(2 ** 27 // max(n, 1))))
    src, dst = [], []
    for s0 in range(0, n, rows):
        Q = X[s0:s0 + rows]
        d2 = (sq[s0:s0 + rows, None] + sq[None, :] - 2.0 * (Q @ X.T)).clamp_(min=0)
        d2[torch.arange(Q.shape[0], device=dev), torch.arange(s0, s0 + Q.shape[0], device=dev)] = float("inf")
        val, idx = torch.topk(d2, k, dim=1, largest=False)
        keep = torch.ones_like(val, dtype=torch.bool) if max_distance is None else val.sqrt() <= max_distance
        i = torch.arange(s0, s0 + Q.shape[0], device=dev)[:, None].expand_as(idx)
        src.append(i[keep]); dst.append(idx[keep])
    e = torch.stack([torch.cat(src), torch.cat(dst)], 1).cpu()
    return Graph.from_edges(e, None, n_items=n)


def distances(data, retain_fraction=1.0, verbose=False, device=None):
    """Graph of pairwise Euclidean distances: all (n choose 2) pairs, or a uniform sample of them."""
    dev = util.cuda_device(device)
    X = _to_device_matrix(data, dev)
    n = X.shape[0]
    n_all = n * (n - 1) // 2
    if retain_fraction >= 1.0:
        edges = torch.triu_indices(n, n, 1, device=dev).T
    else:
        edges = sample_edges(n, int(retain_fraction * n_all), device=dev)
    out = torch.empty(edges.shape[0], dtype=torch.float32, device=dev)
    step = 1 << 22
    for s0 in range(0, edges.shape[0], step):
        e = edges[s0:s0 + step]
        out[s0:s0 + step] = (X[e[:, 0]] - X[e[:, 1]]).norm(dim=1)
    g = Graph.from_edges(edges.cpu(), out.cpu(), n_items=n)
    return g
