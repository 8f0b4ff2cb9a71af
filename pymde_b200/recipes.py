"""Recipes for constructing MDE problems (signatures of pymde/recipes.py:103-503).

The recipes build edges / weights / deviations, pick the constraint and the initial iterate, and return a
`pymde_b200.MDE` whose `embed()` runs on the CUDA path.  `device` defaults to the current CUDA device."""
import numpy as np
import scipy.sparse
import torch

from . import constraints, preprocess, problem, quadratic, util
from .functions import losses, penalties
from .preprocess import Graph


def _remove_anchor_anchor_edges(edges, data, anchors):
    """Edges whose both ends are anchored carry no information (pymde/recipes.py:15-100)."""
    if anchors.shape[0] == 0:
        return edges, data
    a = anchors.to(edges.device)
    both = torch.isin(edges[:, 0], a) & torch.isin(edges[:, 1], a)
    return edges[~both], data[~both]


def _knn_graph_max_k(long=False):
    """mde_knn_graph_max_k(), or mde_knn_graph_long_max_k(): longer neighbour lists are assembled into a host Graph."""
    from . import _lib
    lib = _lib.load()
    return int(lib.mde_knn_graph_long_max_k() if long else lib.mde_knn_graph_max_k())


def _graph_knn_long(A, k):
    """A graph's k-NN search above mde_graph_knn_max_k() takes the long device search (`mde_graph_knn_long*`) when
    the graph searches run on the device and k <= mde_graph_knn_long_max_k()."""
    from . import _lib
    from .preprocess import generic
    lib = _lib.load()
    return (generic._graph_on_device(A)
            and int(lib.mde_graph_knn_max_k()) < k <= int(lib.mde_graph_knn_long_max_k()))


def preserve_distances(data, embedding_dim=2, loss=losses.Absolute, constraint=None, max_distances=5e7,
                       device=None, verbose=False):
    """MDE problem preserving original distances (pymde/recipes.py:103-218).  For a data matrix the pair distances
    are computed and assembled into the edge list on the device (`data_matrix.distances_device`)."""
    if not isinstance(data, (np.ndarray, torch.Tensor, Graph)) and not scipy.sparse.issparse(data):
        raise ValueError("`data` must be a np.ndarray/torch.Tensor/scipy.sparse matrix, or a pymde.Graph.")
    dev = util.cuda_device(device)
    n_items = data.n_items if isinstance(data, Graph) else data.shape[0]
    retain_fraction = max_distances / (n_items * (n_items - 1) / 2)
    if isinstance(data, Graph):
        graph = preprocess.distances(data, retain_fraction=retain_fraction, verbose=verbose, device=dev)
    else:
        graph = preprocess.data_matrix.distances_device(data, retain_fraction=retain_fraction, device=dev)
    edges = graph.edges.to(dev)
    deviations = graph.distances.to(dev)
    if constraint is None:
        constraint = constraints.Centered()
    elif isinstance(constraint, constraints._Standardized):
        deviations = preprocess.scale(deviations, constraint.natural_length(n_items, embedding_dim))
    elif isinstance(constraint, constraints.Anchored):
        edges, deviations = _remove_anchor_anchor_edges(edges, deviations, constraint.anchors)
    return problem.MDE(n_items=n_items, embedding_dim=embedding_dim, edges=edges,
                       distortion_function=loss(deviations), constraint=constraint, device=dev)


def preserve_neighbors(data, embedding_dim=2, attractive_penalty=penalties.Log1p, repulsive_penalty=penalties.Log,
                       constraint=None, n_neighbors=None, repulsive_fraction=None, max_distance=None,
                       init="quadratic", device=None, verbose=False):
    """MDE problem preserving local structure (pymde/recipes.py:221-448).  For a data matrix the neighbour graph is
    assembled on the device from the search's lists (`data_matrix.k_nearest_neighbors_device`, or
    `k_nearest_neighbors_device_long` above 64) when min(n_neighbors, n - 1) <= 256; larger n_neighbors keep the
    chunked GEMM search and the host `Graph`.  For a `Graph` whose searches run on the device, k <= 64 takes
    `graph.k_nearest_neighbors_device` and 64 < k <= 256 `graph.k_nearest_neighbors_device_long`; both keep the
    lowest node indices where shortest-path lengths tie at the k-th place (scipy's route, for larger k, tiny graphs
    or PYMDE_B200_SHORTEST_PATHS=host, keeps an arbitrary subset of the tied nodes)."""
    dev = util.cuda_device(device)
    if isinstance(data, Graph):
        n = data.n_items
    elif data.shape[0] <= 1:
        raise ValueError("The data matrix must have at least two rows.")
    else:
        n = data.shape[0]
    if n_neighbors is None:
        n_neighbors = int(max(min(15, (n * (n - 1) / 2) * 0.01 / n), 5))
    if n_neighbors > n:
        problem.LOGGER.warning("Requested n_neighbors %d > number of items %d. Setting n_neighbors to %d"
                               % (n_neighbors, n, n - 1))
        n_neighbors = n - 1
    if constraint is None:
        constraint = constraints.Centered() if repulsive_penalty is not None else constraints.Standardized()
    if isinstance(data, Graph) and max_distance is None:
        max_distance = (3 * torch.quantile(data.distances, 0.75)).item()
    if verbose:
        problem.LOGGER.info("Computing %d-nearest neighbors, with max_distance=%s" % (n_neighbors, max_distance))

    k = min(n_neighbors, n - 1)
    if isinstance(data, Graph) and _graph_knn_long(data.adjacency_matrix, k):
        knn = preprocess.graph.k_nearest_neighbors_device_long(data, k, max_distance=max_distance, device=dev)
    elif isinstance(data, Graph) or k > _knn_graph_max_k(long=True):
        knn = preprocess.k_nearest_neighbors(data, k=n_neighbors, max_distance=max_distance, verbose=verbose,
                                             device=dev)
    else:
        dm = preprocess.data_matrix
        build = dm.k_nearest_neighbors_device if k <= _knn_graph_max_k() else dm.k_nearest_neighbors_device_long
        knn = build(data, n_neighbors, max_distance=max_distance, device=dev)
    edges = knn.edges.to(dev)
    weights = knn.weights.to(dev)
    if isinstance(constraint, constraints.Anchored):
        edges, weights = _remove_anchor_anchor_edges(edges, weights, constraint.anchors)

    if init == "quadratic":
        if verbose:
            problem.LOGGER.info("Computing quadratic initialization.")
        X_init = quadratic.spectral(n, embedding_dim, edges, weights, max_iter=1000, device=dev)
        if not isinstance(constraint, (constraints._Centered, constraints._Standardized)):
            constraint.project_onto_constraint(X_init, inplace=True)
    elif init == "random":
        X_init = constraint.initialization(n, embedding_dim, dev)
    else:
        raise ValueError("Unsupported value '%s' for keyword argument `init`; the supported values are "
                         "'quadratic' and 'random'." % init)

    if repulsive_penalty is not None:
        if repulsive_fraction is None:
            repulsive_fraction = 0.5 if isinstance(constraint, constraints._Standardized) else 1
        n_choose_2 = int(n * (n - 1) / 2)
        n_repulsive = min(int(repulsive_fraction * edges.shape[0]), n_choose_2 - edges.shape[0])
        negative_edges = preprocess.sample_edges(n, n_repulsive, exclude=edges, device=dev).to(dev)
        negative_weights = -torch.ones(negative_edges.shape[0], dtype=X_init.dtype, device=dev)
        if isinstance(constraint, constraints.Anchored):
            negative_edges, negative_weights = _remove_anchor_anchor_edges(negative_edges, negative_weights,
                                                                           constraint.anchors)
        edges = torch.cat([edges, negative_edges])
        weights = torch.cat([weights, negative_weights])
        f = penalties.PushAndPull(weights, attractive_penalty=attractive_penalty,
                                  repulsive_penalty=repulsive_penalty)
    else:
        f = attractive_penalty(weights)

    mde = problem.MDE(n_items=n, embedding_dim=embedding_dim, edges=edges, distortion_function=f,
                      constraint=constraint, device=dev)
    mde._X_init = X_init.to(dev).float().contiguous()
    d = mde.distances(mde._X_init)
    if bool((d == 0).any()):  # overlapping points make E non-differentiable: perturb (recipes.py:438-447)
        mde._X_init = mde._X_init + 1e-4 * torch.randn_like(mde._X_init)
    return mde


def laplacian_embedding(data, embedding_dim=2, n_neighbors=None, max_distance=None, init="quadratic",
                        device=None, verbose=False):
    """Quadratic penalties + standardization on the k-NN graph (pymde/recipes.py:451-503)."""
    return preserve_neighbors(data, embedding_dim=embedding_dim, attractive_penalty=penalties.Quadratic,
                              repulsive_penalty=None, n_neighbors=n_neighbors, max_distance=max_distance,
                              init=init, device=device, verbose=verbose)


# ---- embedding new points next to a fitted embedding ------------------------------------------------------------------

def _lists_graph(lists, n):
    """(edges [p, 2] int64, weights [p] fp32) of `Graph.from_edges` on the directed pairs (i, lists[i, s]) (-1 = no
    entry): on the device by `graph.knn_edge_list` for CUDA lists of up to 256 columns, else the host `Graph`."""
    from .preprocess.graph import knn_edge_list
    if lists.is_cuda and lists.shape[1] <= _knn_graph_max_k(long=True):
        g = knn_edge_list(lists, n)
        return g.edges, g.weights
    keep = lists >= 0
    rows = torch.arange(n, device=lists.device)[:, None].expand_as(lists)
    e = torch.stack([rows[keep], lists[keep].long()], 1).cpu()
    g = Graph.from_edges(e, None, n_items=n)
    return g.edges.to(lists.device).long(), g.weights.to(lists.device).float()


def _new_points_graph(idx, n_old, repulsive_fraction):
    """Steps 2-4 of `embed_new_points` on the neighbour lists idx [n_new, k] of the new points (global ids: old points
    0 .. n_old - 1, new points n_old .. n - 1; -1 = no entry), on idx's device.  `repulsive_fraction` None: no
    repulsive edges.  Returns (items, lists, edges, weights):
      items    [n_local] global id of every local item: the new points (local 0 .. n_new - 1), then the old points
               the lists or the repulsive edges reference, ascending;
      lists    [n_local, k] int32 local lists (old rows -1);
      edges    [p, 2] local pairs i < j: the attractive edges of `Graph.from_edges` on the lists (a mutual new-new
               pair weighs 2, a new-old pair 1), then the repulsive pairs (weight -1);
      weights  [p] fp32."""
    n_new, k = int(idx.shape[0]), int(idx.shape[1])
    n = n_old + n_new
    dev = idx.device
    idx = idx.long()
    valid = idx >= 0
    new = torch.arange(n_old, n, device=dev)
    att = torch.stack([new[:, None].expand_as(idx)[valid], idx[valid]], 1)
    att_keys = torch.unique(preprocess.preprocess._keys(att, n))
    rep = torch.empty((0, 2), dtype=torch.int64, device=dev)
    if repulsive_fraction is not None:
        p_att = int(att_keys.numel())
        available = n_new * (n - 1) - n_new * (n_new - 1) // 2 - p_att
        n_rep = min(int(repulsive_fraction * p_att), available)
        exclude = torch.stack([att_keys // n, att_keys % n], 1)
        rep = preprocess.preprocess.sample_edges_touching(n, n_old, n_rep, exclude=exclude, device=dev)
    ends = torch.cat([idx[valid], rep.reshape(-1)])
    items = torch.cat([new, torch.unique(ends[ends < n_old])])
    local = torch.full((n,), -1, dtype=torch.int64, device=dev)
    local[items] = torch.arange(items.numel(), device=dev)
    lists = torch.full((items.numel(), k), -1, dtype=torch.int32, device=dev)
    lists[:n_new] = torch.where(valid, local[idx.clamp(min=0)], -1).to(torch.int32)
    edges, weights = _lists_graph(lists, items.numel())
    rep = torch.sort(local[rep], dim=1).values
    edges = torch.cat([edges.long(), rep])
    weights = torch.cat([weights.float(), -torch.ones(rep.shape[0], dtype=torch.float32, device=dev)])
    return items, lists, edges, weights


def _new_points_init(items, lists, n_new, embedding, att_edges):
    """Step 5 of `embed_new_points`: the initial iterate [n_local, m] fp32.  Old rows are exactly their `embedding`
    rows; a new point starts at the mean of the embedding rows of its old neighbours, or at the column mean of
    `embedding` when it has none; when an attractive edge (local pairs `att_edges`) then has length 0, 1e-4 randn is
    added to the new rows only (pymde/recipes.py:438-447 perturbs every row)."""
    emb = embedding.float()
    X = torch.empty((int(items.numel()), emb.shape[1]), dtype=torch.float32, device=emb.device)
    X[n_new:] = emb[items[n_new:]]
    nb = lists[:n_new].long()
    old = nb >= n_new
    cnt = old.sum(1, keepdim=True)
    sums = torch.where(old[..., None], X[nb.clamp(min=0)], 0.0).sum(1)
    X[:n_new] = torch.where(cnt > 0, sums / cnt.clamp(min=1), emb.mean(0))
    if att_edges.shape[0] and bool(((X[att_edges[:, 0]] - X[att_edges[:, 1]]).norm(dim=1) == 0).any()):
        X[:n_new] += 1e-4 * torch.randn_like(X[:n_new])
    return X


def _stacked_matrix(data, new_data, dev):
    """[data; new_data] for the search: a scipy.sparse CSR matrix when either is sparse, else a device tensor (fp32
    when the two dtypes differ; a float16 / bfloat16 pair stays 16-bit and a uint8 / int8 pair 8-bit)."""
    if scipy.sparse.issparse(data) or scipy.sparse.issparse(new_data):
        return scipy.sparse.vstack([scipy.sparse.csr_matrix(data), scipy.sparse.csr_matrix(new_data)]).tocsr()
    a, b = (torch.as_tensor(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x for x in (data, new_data))
    if a.dtype != b.dtype:
        a, b = a.float(), b.float()
    return torch.cat([a.to(dev), b.to(dev)])


def _check_new_graph(data, new_data):
    """`new_data` must span the n_old nodes of `data` and the new ones after them, and hold only edges that touch a
    new node (ValueError otherwise)."""
    n_old, n = data.n_items, new_data.n_items
    if n < n_old:
        raise ValueError("`new_data` has %d nodes; it must hold the %d nodes of `data` and the new ones after them"
                         % (n, n_old))
    B = new_data.adjacency_matrix.tocoo()
    if bool(((B.row < n_old) & (B.col < n_old)).any()):
        raise ValueError("`new_data` holds an edge between two fitted nodes (both < %d); pass only the edges that "
                         "touch a new node" % n_old)


def _union_graph(data, new_data):
    """Adjacency matrix [n, n] of the graph the new nodes are searched in: `data`'s matrix (n_old nodes) padded to
    n = new_data.n_items, plus `new_data`'s.  After `_check_new_graph` the two share no entry, so the sum is their
    union."""
    n_old, n = data.n_items, new_data.n_items
    A = data.adjacency_matrix
    indptr = np.concatenate([A.indptr, np.full(n - n_old, A.indptr[-1], dtype=A.indptr.dtype)])
    padded = scipy.sparse.csr_matrix((A.data, A.indices, indptr), shape=(n, n))
    return (padded + new_data.adjacency_matrix.tocsr()).tocsr()


def _graph_new_lists(data, new_data, k, max_distance, dev):
    """Neighbour lists [n_new, k] (global ids, -1 = none, on `dev`) of the new nodes n_old .. n - 1 in the union of
    the two graphs: when the graph searches run on the device, `graph.knn_rows_device` for k <= 64 and
    `graph.knn_rows_device_long` for k <= 256, else the host row search (`graph.knn_rows_host`), which gives the
    same lists.  `max_distance` None: preserve_neighbors' rule, 3 times the 75th percentile of the union's edge
    lengths."""
    from .preprocess import generic
    from .preprocess import graph as G
    n_old, n = data.n_items, new_data.n_items
    union = _union_graph(data, new_data)
    if max_distance is None:
        # the union's edges are those of `data` and of `new_data`, disjoint: the same lengths as Graph(union).distances
        lengths = torch.cat([data.distances, new_data.distances])
        max_distance = (3 * torch.quantile(lengths, 0.75)).item() if lengths.numel() else np.inf
    if generic._graph_on_device(union) and k <= generic._graph_knn_max_k():
        idx, _ = G.knn_rows_device(union, k, n_old, n, max_distance=max_distance, device=dev)
        return idx
    if _graph_knn_long(union, k):
        idx, _ = G.knn_rows_device_long(union, k, n_old, n, max_distance=max_distance, device=dev)
        return idx
    idx, _ = G.knn_rows_host(union, k, n_old, n, max_distance=max_distance)
    return torch.from_numpy(idx).to(dev)


def _dense_new_lists(X, k, n_old, n):
    """(indices, squared distances) of the new rows n_old .. n - 1 of the stacked matrix X: a float16 / bfloat16 /
    uint8 / int8 matrix with 64 < k <= 256 takes the long row search (`data_matrix.knn_rows_device_long`, read in
    place), every other case `data_matrix.knn_rows_device` (k <= 64, sparse input, and the GEMM rows for fp32 at
    k > 64 and for k > 256).  fp32 stays on the GEMM rows because they measured faster on it (DESIGN section 11.8);
    for a 16-bit or 8-bit matrix they would make an fp32 and an fp64 copy of the whole stack."""
    dm = preprocess.data_matrix
    from . import _lib
    lib = _lib.load()
    narrow = isinstance(X, torch.Tensor) and X.dtype in (torch.float16, torch.bfloat16, torch.uint8, torch.int8)
    if narrow and lib.mde_knn_wide_max_k() < k <= lib.mde_knn_long_max_k():
        return dm.knn_rows_device_long(X, k, n_old, n)
    return dm.knn_rows_device(X, k, n_old, n)


def _new_points_mde(data, embedding, new_data, n_neighbors=None, attractive_penalty=penalties.Log1p,
                    repulsive_penalty=penalties.Log, repulsive_fraction=None, max_distance=None, device=None):
    """Steps 1-5 of `embed_new_points`: (the anchored `MDE` over the new points and the old points they reference,
    with its initial iterate in `_X_init`; items, the global id of each of its items: new points n_old .. n - 1
    first), or (None, None) when there are no new rows.  `data` and `new_data` are two data matrices, or two Graphs
    (`new_data` over the n_old fitted and the new nodes, holding only edges that touch a new node); every check
    runs before the device is touched."""
    graph = isinstance(data, Graph)
    if graph != isinstance(new_data, Graph):
        raise ValueError("`data` and `new_data` must both be data matrices or both be Graphs")
    if not isinstance(embedding, (np.ndarray, torch.Tensor)) or embedding.ndim != 2:
        raise ValueError("`embedding` must be a 2-D array (n_old x embedding_dim)")
    if graph:
        n_old, n_new = data.n_items, new_data.n_items - data.n_items
        _check_new_graph(data, new_data)
        if int(embedding.shape[0]) != n_old:
            raise ValueError("`embedding` has %d rows; `data` has %d nodes" % (int(embedding.shape[0]), n_old))
    else:
        if len(data.shape) != 2 or len(new_data.shape) != 2:
            raise ValueError("`data` and `new_data` must be 2-D matrices")
        n_old, n_new = int(data.shape[0]), int(new_data.shape[0])
        if int(embedding.shape[0]) != n_old:
            raise ValueError("`embedding` has %d rows; `data` has %d" % (int(embedding.shape[0]), n_old))
        if int(new_data.shape[1]) != int(data.shape[1]):
            raise ValueError("`new_data` has %d columns; `data` has %d" % (int(new_data.shape[1]),
                                                                          int(data.shape[1])))
    if n_new == 0:
        return None, None
    if n_old < 1:
        raise ValueError("`data` must hold at least one fitted row")
    dev = util.cuda_device(device)
    n = n_old + n_new
    if n_neighbors is None:
        n_neighbors = int(max(min(15, (n * (n - 1) / 2) * 0.01 / n), 5))
    k = int(min(n_neighbors, n - 1))
    if graph:
        idx = _graph_new_lists(data, new_data, k, max_distance, dev)
    else:
        idx, d2 = _dense_new_lists(_stacked_matrix(data, new_data, dev), k, n_old, n)
        idx = idx.to(dev)
        if max_distance is not None:
            idx = torch.where(d2.to(dev).sqrt() <= max_distance, idx, -1)  # (a NaN distance is dropped)
    if repulsive_penalty is not None and repulsive_fraction is None:
        repulsive_fraction = 1
    items, lists, edges, weights = _new_points_graph(
        idx, n_old, repulsive_fraction if repulsive_penalty is not None else None)
    emb = torch.as_tensor(embedding).to(device=dev, dtype=torch.float32)
    n_att = int((weights > 0).sum())
    X_init = _new_points_init(items, lists, n_new, emb, edges[:n_att])
    if repulsive_penalty is not None:
        f = penalties.PushAndPull(weights, attractive_penalty=attractive_penalty, repulsive_penalty=repulsive_penalty)
    else:
        f = attractive_penalty(weights)
    anchors = torch.arange(n_new, int(items.numel()), device=dev)
    constraint = constraints.Anchored(anchors, X_init[n_new:].clone())
    mde = problem.MDE(n_items=int(items.numel()), embedding_dim=int(emb.shape[1]), edges=edges,
                      distortion_function=f, constraint=constraint, device=dev)
    mde._X_init = X_init.contiguous()
    return mde, items


def embed_new_points(data, embedding, new_data, n_neighbors=None, attractive_penalty=penalties.Log1p,
                     repulsive_penalty=penalties.Log, repulsive_fraction=None, max_distance=None, eps=1e-5,
                     max_iter=300, device=None, verbose=False):
    """Embed the rows of `new_data` next to `embedding`, the fitted embedding of the rows of `data`, leaving
    `embedding` untouched: the "transform" step of an embedding.  Returns the new rows' embedding, an
    (n_new x embedding_dim) fp32 tensor on the device.

    The workflow the reference documents (docs "Embedding new points") runs `preserve_neighbors` on the stacked data
    with every fitted row anchored, and so pays for a search, a spectral initialisation and a solve over all rows.
    Here only the new rows are searched, against all rows (`data_matrix.knn_rows_device`: exact, with a cost of about
    n_new n d), and only the new points and the fitted points they touch enter the solve:
      * attractive edges: `Graph.from_edges` on the new points' lists of their min(n_neighbors, n - 1) nearest rows
        (`n_neighbors` defaults to `preserve_neighbors`' rule at n = n_old + n_new; entries beyond `max_distance`
        dropped): a mutual new-new pair weighs 2, a new-old pair 1.  Unlike the reference workflow, the fitted points'
        own neighbour lists add no edges (that would need their n^2 search);
      * repulsive edges (none when `repulsive_penalty` is None): repulsive_fraction (default 1) times as many pairs
        as attractive ones, each with a uniform new point at one end and a uniform row at the other, distinct and not
        attractive, drawn from the module RNG (`pymde_b200.seed(s)` reproduces them);
      * the fitted points are anchored at their `embedding` rows; a new point starts at the mean of its fitted
        neighbours' rows (the column mean of `embedding` when it has none);
      * the anchored problem is solved on the device (`MDE.embed(eps, max_iter)`).
    `data` and `new_data` are dense (numpy, torch; fp32, or float16 / bfloat16 / uint8 / int8 searched in place) or
    scipy.sparse matrices with the same columns.  Dense input is searched by the row-range tensor-core search
    `mde_knn_rows` up to k = 64, which gives the rows of the full exact search bit for bit.  Above that a 16-bit or
    8-bit matrix takes the long row search up to k = 256 (`data_matrix.knn_rows_device_long`: the rows of the full
    long search bit for bit, read in place, without an fp32 copy), and an fp32 matrix, or any k > 256, the row range
    of the GEMM path.  Sparse input is stacked on the host and searched without densifying it
    (`mde_knn_csr_rows`, k <= 256): the tiles sweep only the new rows, and the result is that of the full sparse
    search.

    Graphs: `data` is the `Graph` of the n_old fitted nodes, and `new_data` a `Graph` over n_old + n_new nodes that
    holds the edges of the new nodes n_old .. n - 1 -- every edge has at least one end >= n_old, and a new node
    without edges is allowed -- e.g. `Graph.from_edges(new_edges, weights, n_items=n_old + n_new)`.  The new nodes'
    lists are their nearest nodes under the shortest-path metric of the union of the two graphs, within
    `max_distance` (default: 3 times the 75th percentile of the union's edge lengths, `preserve_neighbors`' rule;
    inf: unlimited), ties broken by node index.  Only the new nodes are searched: on graphs the device searches take,
    `graph.knn_rows_device` (`mde_graph_knn_rows`, the rows of the full device search bit for bit) for k <= 64 and
    `graph.knn_rows_device_long` (`mde_graph_knn_long_rows`) for 64 < k <= 256; otherwise the host row search
    `graph.knn_rows_host` (scipy's Dijkstra), which gives the same lists."""
    mde, _ = _new_points_mde(data, embedding, new_data, n_neighbors=n_neighbors,
                             attractive_penalty=attractive_penalty, repulsive_penalty=repulsive_penalty,
                             repulsive_fraction=repulsive_fraction, max_distance=max_distance, device=device)
    if mde is None:
        return torch.empty((0, int(embedding.shape[1])), dtype=torch.float32, device=util.cuda_device(device))
    X = mde.embed(eps=eps, max_iter=max_iter, verbose=verbose)
    n_new = new_data.n_items - data.n_items if isinstance(new_data, Graph) else int(new_data.shape[0])
    return X[:n_new].contiguous()
