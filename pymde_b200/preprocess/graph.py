"""Weighted graphs for MDE problem construction (interface of pymde/preprocess/graph.py:75-256).

A `Graph` wraps a symmetric scipy CSR adjacency matrix.  `edges` lists each undirected edge once,
(i, j) with i < j, sorted by (i, j); `distances` / `weights` are the matching values.  Problem
construction is one-shot host work (SURVEY section 2 rows 12-15: outside the hot path); the resulting
edge tensors are what the CUDA path consumes."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch


def _as_numpy(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


class Graph(object):
    def __init__(self, adjacency_matrix):
        A = adjacency_matrix
        if isinstance(A, torch.Tensor):
            A = A.detach().cpu().numpy()
        if isinstance(A, np.ndarray):
            A = sp.csr_matrix(A)
        elif sp.issparse(A) and not isinstance(A, sp.csr_matrix):
            A = A.tocsr()
        elif not sp.issparse(A):
            raise ValueError("adjacency_matrix must be a dense array, tensor or scipy sparse matrix")
        A = A.copy()
        A.data[A.data == np.inf] = 0  # unreachable pairs carry no edge
        A.eliminate_zeros()
        diag = A.diagonal() > 0
        if diag.any():
            raise ValueError("Adjacency matrices must not contain self edges; the following nodes were "
                             "found to have self edges: ", np.argwhere(diag).flatten())
        self._A = A
        self._edges = None
        self._values = None

    @staticmethod
    def from_edges(edges, weights=None, n_items=None):
        """Graph from an edge list; repeated (or reciprocal) edges have their weights summed."""
        e = _as_numpy(edges).astype(np.int64).copy()
        w = np.ones(e.shape[0], dtype=np.float32) if weights is None else _as_numpy(weights).astype(np.float32)
        lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
        n = int(hi.max()) + 1 if n_items is None else int(n_items)
        upper = sp.coo_matrix((w, (lo, hi)), shape=(n, n)).tocsr()  # duplicates are summed here
        return Graph((upper + upper.T).tocsr())

    # --- adjacency -----------------------------------------------------------------------
    @property
    def adjacency_matrix(self):
        return self._A

    A = adjacency_matrix

    @property
    def n_items(self):
        return self._A.shape[0]

    @property
    def n_all_edges(self):
        return self.n_items * (self.n_items - 1) // 2

    def _materialise(self):
        if self._edges is None:
            U = sp.triu(self._A, k=1, format="csr").tocoo()  # row-major => sorted by (i, j)
            order = np.lexsort((U.col, U.row))
            self._edges = torch.tensor(np.stack([U.row[order], U.col[order]], 1).astype(np.int64))
            self._values = torch.tensor(U.data[order].astype(np.float32))

    @property
    def edges(self):
        self._materialise()
        return self._edges

    @property
    def distances(self):
        self._materialise()
        return self._values

    weights = distances

    @property
    def n_edges(self):
        return int(self.edges.shape[0])

    def neighbors(self, node):
        return self._A.indices[self._A.indptr[node]:self._A.indptr[node + 1]]

    def neighbor_distances(self, node):
        return self._A.data[self._A.indptr[node]:self._A.indptr[node + 1]]

    def draw(self, embedding_dim=2, standardized=False, device=None, verbose=False):
        """Embed the graph for drawing (pymde/preprocess/graph.py:200-256): shortest-path distances (at most 1e7
        of them), WeightedQuadratic loss + Centered, or Cubic penalty + Standardized.  Returns the embedding;
        plotting is out of scope here."""
        from .. import constraints, problem
        from ..functions import losses, penalties
        if bool((self.distances < 0).any()):
            raise ValueError("Graphs with negative edge weights cannot be drawn.")
        if self.n_edges < self.n_all_edges:
            dg = shortest_paths(self, retain_fraction=min(1.0, 1e7 / self.n_all_edges), verbose=verbose)
        else:
            dg = self
        if not standardized:
            constraint, f = constraints.Centered(), losses.WeightedQuadratic(dg.distances)
        else:
            constraint, f = constraints.Standardized(), penalties.Cubic(1 / dg.distances)
        mde = problem.MDE(n_items=self.n_items, embedding_dim=embedding_dim, edges=dg.edges, distortion_function=f,
                          constraint=constraint, device=device)
        return mde.embed(verbose=verbose)

    def __getitem__(self, key):
        return self._A[key]

    def __setitem__(self, key, value):
        raise AttributeError("Graph objects are immutable.")


class EdgeListGraph(object):
    """Result of the device shortest-path search: an edge list that never left the GPU.  Quacks like the part of
    `Graph` the recipes use (`edges` sorted by (i, j), `distances`, `n_items`); `to_graph()` builds the scipy-backed
    object when somebody needs the adjacency matrix."""

    def __init__(self, edges, distances, n_items):
        self.edges, self.distances, self._n = edges, distances, int(n_items)
        self.weights = distances

    @property
    def n_items(self):
        return self._n

    @property
    def n_edges(self):
        return int(self.edges.shape[0])

    @property
    def n_all_edges(self):
        return self._n * (self._n - 1) // 2

    def to_graph(self):
        return Graph.from_edges(self.edges.cpu().numpy(), self.distances.cpu().numpy(), n_items=self._n)


_PATH_WS_BUDGET = 8 << 30  # device scratch of the weighted engine: caps its batch of sources


def _is_unweighted(A):
    return bool((A.data == 1.0).all())


def _device_csr(A, dev):
    """Undirected device CSR of `A` for the weighted engine: the entries of A and of A^T (the semantics of scipy's
    `dijkstra(directed=False)`, also for an asymmetric A), with parallel entries reduced to the shortest one --
    the same shortest paths as keeping them all, at half the relaxations for a symmetric A.  (scipy's Dijkstra
    treats parallel entries the same way for float64 data, but sums them when it converts another dtype.)  int32
    indptr and indices, fp32 weights.  Negative weights raise ValueError (scipy's Dijkstra rejects them too)."""
    if A.nnz and float(A.data.min()) < 0:
        raise ValueError("shortest paths need non-negative edge weights")
    n = A.shape[0]
    coo = A.tocoo()
    r = torch.tensor(coo.row.astype(np.int64), device=dev)
    c = torch.tensor(coo.col.astype(np.int64), device=dev)
    w = torch.tensor(coo.data.astype(np.float32), device=dev)
    r, c, w = torch.cat([r, c]), torch.cat([c, r]), torch.cat([w, w])
    order = torch.argsort(w, stable=True)          # within one (row, col) key the shortest entry comes first
    key = (r * n + c)[order]
    order = order[torch.argsort(key, stable=True)]
    key, w = (r * n + c)[order], w[order]
    first = torch.ones_like(key, dtype=torch.bool)
    first[1:] = key[1:] != key[:-1]
    key, w = key[first], w[first]
    rows = key // n
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n), 0)
    return indptr.int(), (key % n).int(), w.contiguous()


def _path_ws(ws_bytes_fn, n, nsrc, dev):
    """Scratch for the weighted engine: the batch of sources grows with the memory it is given (fewer batches,
    fewer synchronising rounds), up to a quarter of the free device memory or _PATH_WS_BUDGET."""
    per32 = int(ws_bytes_fn(n, 64)) - int(ws_bytes_fn(n, 32))
    free = torch.cuda.mem_get_info(dev)[0]
    budget = min(_PATH_WS_BUDGET, free // 4)
    batch = max(32, min((nsrc + 31) // 32 * 32, int(budget // max(per32, 1)) * 32))
    return torch.empty(int(ws_bytes_fn(n, batch)), dtype=torch.uint8, device=dev)


def _collect_pairs(run, n, retain_fraction, dev):
    """Shared tail of the shortest-path engines: `run(src, dst, len, cap, count)` appends (s, v, length) triples;
    the buffers are sized from the expected sample, the call is repeated with larger ones when they overflowed (the
    same seed draws the same sample), and the result is sorted by (s, v) into an `EdgeListGraph`."""
    expected = min(1.0, float(retain_fraction)) * n * (n - 1) / 2
    cap = int(expected * 1.02 + 4 * (expected ** 0.5) + 1024)
    while True:
        src = torch.empty(cap, dtype=torch.int32, device=dev)
        dst = torch.empty(cap, dtype=torch.int32, device=dev)
        ln = torch.empty(cap, dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            run(src, dst, ln, cap, count)
        got = int(count.item())
        if got <= cap:
            break
        cap = int(got * 1.01) + 1024  # (only when the estimate was exceeded: same seed => same sample)
    src, dst, ln = src[:got].long(), dst[:got].long(), ln[:got]
    order = torch.argsort(src * n + dst)
    return EdgeListGraph(torch.stack([src[order], dst[order]], 1), ln[order], n)


def shortest_paths_device(graph, max_length=None, retain_fraction=1.0, device=None, seed=None):
    """Shortest paths on the GPU.  Same contract as `shortest_paths` -- pairs (i < j) within `max_length`, each kept
    with probability `retain_fraction` -- but the sample is drawn by a counter-based hash seeded from the module RNG,
    and the result stays on the device as an `EdgeListGraph`.  Unweighted graphs use hop counts (`mde_graph_hops`:
    bit-parallel multi-source BFS, 256 sources per pass over the adjacency); weighted ones `mde_graph_sssp`
    (batched frontier Bellman-Ford with fp64 lengths, equal to scipy's Dijkstra after the cast to fp32).  The same
    seed selects the same pairs in both engines."""
    import ctypes as C
    from .. import _lib, util
    A = graph.adjacency_matrix if isinstance(graph, Graph) else Graph(graph).adjacency_matrix
    n = A.shape[0]
    dev = util.cuda_device(device)
    lib = _lib.load()
    if seed is None:
        seed = int(util.np_rng().integers(0, 2 ** 62))
    unlimited = max_length is None or not np.isfinite(max_length)
    if _is_unweighted(A):
        indptr = torch.tensor(A.indptr.astype(np.int32), device=dev)
        indices = torch.tensor(A.indices.astype(np.int32), device=dev)
        ws = torch.empty(int(lib.mde_graph_hops_ws_bytes(n)), dtype=torch.uint8, device=dev)
        limit = 0 if unlimited else int(max_length)

        def run(src, dst, ln, cap, count):
            _lib.check(lib.mde_graph_hops(indptr.data_ptr(), indices.data_ptr(), n, 0, n, limit, float(retain_fraction),
                                          C.c_uint64(seed), src.data_ptr(), dst.data_ptr(), ln.data_ptr(), cap,
                                          count.data_ptr(), ws.data_ptr(), ws.numel(), util.stream_ptr(dev)))
    else:
        indptr, indices, weights = _device_csr(A, dev)
        ws = _path_ws(lib.mde_graph_sssp_ws_bytes, n, n, dev)
        limit = 0.0 if unlimited else float(max_length)

        def run(src, dst, ln, cap, count):
            _lib.check(lib.mde_graph_sssp(indptr.data_ptr(), indices.data_ptr(), weights.data_ptr(), n, 0, n, limit,
                                          float(retain_fraction), C.c_uint64(seed), src.data_ptr(), dst.data_ptr(),
                                          ln.data_ptr(), cap, count.data_ptr(), ws.data_ptr(), ws.numel(),
                                          util.stream_ptr(dev)))
    return _collect_pairs(run, n, retain_fraction, dev)


def k_nearest_neighbors_device(graph, k, max_distance=None, device=None):
    """k-nearest-neighbour graph under the shortest-path metric, on the GPU (`mde_graph_knn`).  Every node's k
    nearest nodes within `max_distance` (ties broken by node index), as undirected pairs (i < j) sorted by (i, j);
    a pair that is a neighbour in both directions gets weight 2, otherwise 1 -- the edges and weights that
    `k_nearest_neighbors` gives when no lengths tie.  Returns an `EdgeListGraph` on the device."""
    return _knn_device(graph, k, max_distance, device, long=False)


def k_nearest_neighbors_device_long(graph, k, max_distance=None, device=None):
    """`k_nearest_neighbors_device` for 1 <= k <= 256 (`mde_graph_knn_long`, the same lists as `mde_graph_knn` for
    k <= 64).  Where lengths tie at the k-th place the lowest node indices are kept, where the host
    `k_nearest_neighbors` keeps an arbitrary subset of the tied nodes."""
    return _knn_device(graph, k, max_distance, device, long=True)


def _knn_device(graph, k, max_distance, device, long):
    from .. import _lib, util
    A = graph.adjacency_matrix if isinstance(graph, Graph) else Graph(graph).adjacency_matrix
    n = A.shape[0]
    k = int(k)
    lib = _lib.load()
    max_k = int(lib.mde_graph_knn_long_max_k() if long else lib.mde_graph_knn_max_k())
    if not 1 <= k <= max_k:
        raise ValueError("k must be between 1 and %d" % max_k)
    dev = util.cuda_device(device)
    indptr, indices, weights = _device_csr(A, dev)
    wptr = None if _is_unweighted(A) else weights.data_ptr()
    ws = _path_ws(lib.mde_graph_knn_ws_bytes, n, n, dev)
    idx = torch.empty(n * k, dtype=torch.int32, device=dev)
    ln = torch.empty(n * k, dtype=torch.float32, device=dev)
    limit = 0.0 if (max_distance is None or not np.isfinite(max_distance)) else float(max_distance)
    search = lib.mde_graph_knn_long if long else lib.mde_graph_knn
    with torch.cuda.device(dev):
        _lib.check(search(indptr.data_ptr(), indices.data_ptr(), wptr, n, k, limit, idx.data_ptr(), ln.data_ptr(),
                          ws.data_ptr(), ws.numel(), util.stream_ptr(dev)))
    del ws, ln
    return knn_edge_list(idx.view(n, k), n)


def _knn_limit(max_distance):
    """The search radius of `mde_graph_knn`: None, inf or a value <= 0 mean unlimited."""
    if max_distance is None or not np.isfinite(max_distance) or float(max_distance) <= 0:
        return np.inf
    return float(max_distance)


def knn_rows_device(graph, k, s_begin, s_end, max_distance=None, device=None):
    """Shortest-path k-nearest neighbours of the nodes s_begin .. s_end - 1 only, on the GPU (`mde_graph_knn_rows`):
    (idx [rows, k] int32, len [rows, k] fp32) on the device, row r being row s_begin + r of `mde_graph_knn` bit for
    bit -- the k smallest (length, node index) pairs within `max_distance`, the node itself excluded, padded with
    -1 / inf.  The workspace still holds an n x B distance tile (B >= 32), so the memory is that of the full search
    on the same graph; the time is that of the searched rows."""
    return _knn_rows_device(graph, k, s_begin, s_end, max_distance, device, long=False)


def knn_rows_device_long(graph, k, s_begin, s_end, max_distance=None, device=None):
    """`knn_rows_device` for 1 <= k <= 256 (`mde_graph_knn_long_rows`): row r is row s_begin + r of
    `mde_graph_knn_long` bit for bit, and equals `knn_rows_host`."""
    return _knn_rows_device(graph, k, s_begin, s_end, max_distance, device, long=True)


def _knn_rows_device(graph, k, s_begin, s_end, max_distance, device, long):
    from .. import _lib, util
    A = graph.adjacency_matrix if isinstance(graph, Graph) else Graph(graph).adjacency_matrix
    n = A.shape[0]
    k, s_begin, s_end = int(k), int(s_begin), int(s_end)
    lib = _lib.load()
    max_k = int(lib.mde_graph_knn_long_max_k() if long else lib.mde_graph_knn_max_k())
    if not 1 <= k <= max_k:
        raise ValueError("k must be between 1 and %d" % max_k)
    if not 0 <= s_begin <= s_end <= n:
        raise ValueError("the rows [%d, %d) are not a range of the %d nodes" % (s_begin, s_end, n))
    dev = util.cuda_device(device)
    rows = s_end - s_begin
    idx = torch.empty((rows, k), dtype=torch.int32, device=dev)
    ln = torch.empty((rows, k), dtype=torch.float32, device=dev)
    if rows == 0:
        return idx, ln
    indptr, indices, weights = _device_csr(A, dev)
    wptr = None if _is_unweighted(A) else weights.data_ptr()
    ws = _path_ws(lib.mde_graph_knn_ws_bytes, n, rows, dev)
    limit = _knn_limit(max_distance)
    search = lib.mde_graph_knn_long_rows if long else lib.mde_graph_knn_rows
    with torch.cuda.device(dev):
        _lib.check(search(indptr.data_ptr(), indices.data_ptr(), wptr, n, s_begin, s_end, k,
                          0.0 if np.isinf(limit) else limit, idx.data_ptr(), ln.data_ptr(), ws.data_ptr(), ws.numel(),
                          util.stream_ptr(dev)))
    return idx, ln


def _smallest_pairs(D, rows, k):
    """Per row of D [c, n] (fp64, inf = unreached), the k smallest finite (D, column) pairs in lexicographic order,
    the column rows[i] of row i excluded: (idx [c, k] int32, len [c, k] fp64), padded with -1 / inf."""
    c, n = D.shape
    D = D.copy()
    D[np.arange(c), rows] = np.inf
    idx = np.full((c, k), -1, dtype=np.int32)
    ln = np.full((c, k), np.inf)
    kth = np.partition(D, k - 1, axis=1)[:, k - 1] if k < n else np.full(c, np.inf)
    r, j = np.nonzero((D <= kth[:, None]) & np.isfinite(D))  # every pair at most the k-th length, ties included
    d = D[r, j]
    order = np.lexsort((j, d, r))
    r, j, d = r[order], j[order], d[order]
    start = np.searchsorted(r, np.arange(c))
    slot = np.arange(r.size) - start[r]
    keep = slot < k
    idx[r[keep], slot[keep]] = j[keep]
    ln[r[keep], slot[keep]] = d[keep]
    return idx, ln


def knn_rows_host(graph, k, s_begin, s_end, max_distance=None):
    """The host restatement of `knn_rows_device` for any k >= 1: scipy's Dijkstra (undirected, `limit` =
    max_distance) from the nodes s_begin .. s_end - 1 in row chunks, then per row the k smallest (fp64 length, node
    index) pairs, the node itself excluded.  Returns numpy (idx [rows, k] int32, len [rows, k] fp32), padded with
    -1 / inf: the device search's lists exactly, since its lengths are scipy's."""
    A = graph.adjacency_matrix if isinstance(graph, Graph) else Graph(graph).adjacency_matrix
    n = A.shape[0]
    k, s_begin, s_end = int(k), int(s_begin), int(s_end)
    if k < 1:
        raise ValueError("k must be at least 1")
    if not 0 <= s_begin <= s_end <= n:
        raise ValueError("the rows [%d, %d) are not a range of the %d nodes" % (s_begin, s_end, n))
    A = A.astype(np.float64)  # (float64: parallel entries count as the shortest one, as on the device)
    limit = _knn_limit(max_distance)
    idx = np.full((s_end - s_begin, k), -1, dtype=np.int32)
    ln = np.full((s_end - s_begin, k), np.inf, dtype=np.float32)
    chunk = max(1, min(n, int(2e7 // max(n, 1))))
    for r0 in range(s_begin, s_end, chunk):
        rows = np.arange(r0, min(s_end, r0 + chunk))
        D = csgraph.dijkstra(A, directed=False, indices=rows, limit=limit)
        i, d = _smallest_pairs(D, rows, k)
        idx[r0 - s_begin:r0 - s_begin + rows.size] = i
        ln[r0 - s_begin:r0 - s_begin + rows.size] = d.astype(np.float32)
    return idx, ln


def knn_edge_list(idx, n):
    """`EdgeListGraph` of the neighbour lists idx [n, k] (device int32, -1 = no entry, 1 <= k <= 256) on their
    device: the edges and weights `Graph.from_edges` gives for the directed pairs (i, idx[i, s]) -- every unordered
    pair once as (i, j), i < j, sorted by (i, j), weighted by the number of entries i -> j and j -> i
    (`mde_knn_graph_long_count` / `mde_knn_graph_long_emit`, include/mde_b200.h).  An entry equal to its own row or outside
    [-1, n) raises ValueError, as `Graph` does for a self edge."""
    import ctypes as C
    from .. import _lib
    lib = _lib.load()
    n = int(n)
    idx = idx.to(dtype=torch.int32).contiguous()
    if idx.dim() != 2 or idx.shape[0] != n:
        raise ValueError("neighbour lists must have shape (n, k)")
    k = int(idx.shape[1])
    if not 1 <= k <= int(lib.mde_knn_graph_long_max_k()):
        raise ValueError("k must be between 1 and %d" % int(lib.mde_knn_graph_long_max_k()))
    dev = idx.device
    need = C.c_size_t(0)
    _lib.check(lib.mde_knn_graph_long_ws_bytes(n, k, C.byref(need)))
    ws = torch.empty(need.value + 1024, dtype=torch.uint8, device=dev)
    off = (-ws.data_ptr()) % 1024
    count = C.c_int64(0)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        code = lib.mde_knn_graph_long_count(idx.data_ptr(), n, k, ws.data_ptr() + off, need.value, C.byref(count), stream)
        if code == _lib.MDE_E_INVALID:
            raise ValueError("neighbour lists must hold row indices in [0, n) other than the row itself, or -1")
        _lib.check(code)
        p = int(count.value)
        edges = torch.empty((p, 2), dtype=torch.int64, device=dev)
        weights = torch.empty(p, dtype=torch.float32, device=dev)
        if p:
            _lib.check(lib.mde_knn_graph_long_emit(n, k, ws.data_ptr() + off, need.value, edges.data_ptr(),
                                              weights.data_ptr(), stream))
        torch.cuda.current_stream().synchronize()  # (the scratch buffer is released on return)
    return EdgeListGraph(edges, weights, n)


def shortest_paths(graph, max_length=None, retain_fraction=1.0, n_workers=None, verbose=False):
    """Shortest-path distances as a Graph (interface of pymde/preprocess/graph.py:345-474): unreachable pairs and
    pairs beyond `max_length` are dropped; with `retain_fraction` < 1 every remaining pair is kept with that
    probability (Bernoulli draws from the module RNG seeded by `pymde_b200.seed`, like the reference's per-row
    sampling), which bounds memory on large graphs.  Unweighted graphs use BFS hop counts, weighted ones Dijkstra
    (scipy.sparse.csgraph), in row chunks."""
    from .. import util
    del n_workers
    if sp.issparse(graph):
        graph = Graph(graph)
    elif not isinstance(graph, Graph):
        raise ValueError("`graph` must be a pymde.Graph instance or scipy.sparse adjacency matrix.")
    A = graph.adjacency_matrix
    unweighted = bool((A.data == 1.0).all())
    limit = np.inf if max_length is None else float(max_length)
    n = graph.n_items
    rows, cols, vals = [], [], []
    chunk = max(1, min(n, int(2e7 // max(n, 1))))
    for s0 in range(0, n, chunk):
        idx = np.arange(s0, min(n, s0 + chunk))
        D = csgraph.dijkstra(A, directed=False, indices=idx, unweighted=unweighted, limit=limit)
        r, c = np.nonzero(np.isfinite(D) & (D > 0))
        keep = c > idx[r]
        if retain_fraction < 1.0:
            keep &= util.np_rng().uniform(size=keep.size) <= retain_fraction
        rows.append(idx[r][keep]); cols.append(c[keep]); vals.append(D[r, c][keep])
    rows, cols, vals = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    return Graph.from_edges(np.stack([rows, cols], 1), vals.astype(np.float32), n_items=n)


def scale(graph, natural_length):
    """New graph whose distances have RMS `natural_length` (pymde/preprocess/graph.py:259-279)."""
    d = graph.distances
    alpha = float(natural_length) / float(d.pow(2).mean().sqrt())
    return Graph.from_edges(graph.edges, alpha * d, n_items=graph.n_items)


def breadth_first_order(csgraph_matrix, i_start, directed=True, return_predecessors=True):
    """Hop counts from `i_start` (inf where unreachable) and BFS predecessors (-9999 where none), the pair the
    reference's Cython helper returns (pymde/preprocess/graph.py:286-308)."""
    del return_predecessors
    order, pred = csgraph.breadth_first_order(csgraph_matrix, i_start, directed=directed, return_predecessors=True)
    n = csgraph_matrix.shape[0]
    lengths = np.full(n, np.inf, dtype=np.float32)
    lengths[i_start] = 0.0
    for v in order[1:]:  # BFS order: a node's predecessor is always settled before the node
        lengths[v] = lengths[pred[v]] + 1.0
    pred = pred.astype(np.int32)
    pred[pred < 0] = -9999
    return lengths, pred


def k_nearest_neighbors(graph, k, graph_distances=False, max_distance=None, verbose=False):
    """k nearest neighbours of every node under the shortest-path metric."""
    A = graph.adjacency_matrix
    n = graph.n_items
    unweighted = bool((A.data == 1.0).all())
    limit = np.inf if max_distance is None else float(max_distance)
    src, dst, val = [], [], []
    chunk = max(1, min(n, int(2e7 // max(n, 1))))
    for s0 in range(0, n, chunk):
        idx = np.arange(s0, min(n, s0 + chunk))
        D = csgraph.dijkstra(A, directed=False, indices=idx, unweighted=unweighted, limit=limit)
        D[np.arange(len(idx)), idx] = np.inf
        kk = min(k, n - 1)
        nb = np.argpartition(D, kk - 1, axis=1)[:, :kk]
        dd = np.take_along_axis(D, nb, 1)
        ok = np.isfinite(dd)
        src.append(np.repeat(idx, kk)[ok.ravel()]); dst.append(nb.ravel()[ok.ravel()]); val.append(dd.ravel()[ok.ravel()])
    e = np.stack([np.concatenate(src), np.concatenate(dst)], 1)
    if graph_distances:
        lo, hi = np.minimum(e[:, 0], e[:, 1]), np.maximum(e[:, 0], e[:, 1])
        key, first = np.unique(lo * n + hi, return_index=True)
        return Graph.from_edges(np.stack([key // n, key % n], 1), np.concatenate(val)[first].astype(np.float32), n)
    return Graph.from_edges(e, None, n_items=n)
