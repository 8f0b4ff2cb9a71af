"""Edge sampling and scaling utilities (interface of pymde/preprocess/preprocess.py)."""
import numpy as np
import torch

from .. import util


def _keys(e, n):
    lo = torch.minimum(e[:, 0], e[:, 1])
    hi = torch.maximum(e[:, 0], e[:, 1])
    return lo * n + hi


def _generator(seed, dev):
    gen = torch.Generator(device=dev)
    gen.manual_seed(int(seed) if seed is not None else int(util.np_rng().integers(0, 2 ** 62)))
    return gen


def _sample_keys(draw, n, num_edges, exclude, dev):
    """Keys lo * n + hi of at most `num_edges` distinct pairs from rounds of draw(m) -> [m, 2] pairs: self pairs
    dropped, pairs canonicalised, those in `exclude` (pairs [p, 2], any order) filtered out with a sorted search on
    64-bit keys, duplicates removed keeping draw order; at most 64 rounds."""
    excl = None
    if exclude is not None and int(exclude.shape[0]):
        ex = exclude if isinstance(exclude, torch.Tensor) else torch.as_tensor(np.asarray(exclude))
        excl = torch.sort(_keys(ex.to(dev).long(), n)).values
    got = torch.empty(0, dtype=torch.int64, device=dev)
    draws = 0
    while got.numel() < num_edges and draws < 64:
        want = num_edges - got.numel()
        e = draw(int(want * 1.15) + 1024)
        e = e[e[:, 0] != e[:, 1]]
        key = _keys(e, n)
        if excl is not None:
            pos = torch.searchsorted(excl, key).clamp_(max=excl.numel() - 1)
            key = key[excl[pos] != key]
        key = torch.cat([got, key])
        # de-duplicate keeping first occurrences (stable draw order)
        srt, order = torch.sort(key, stable=True)
        first = torch.ones_like(srt, dtype=torch.bool)
        first[1:] = srt[1:] != srt[:-1]
        keep = torch.sort(order[first]).values
        got = key[keep][:num_edges]
        draws += 1
    return got


def sample_edges(n, num_edges, exclude=None, seed=None, device=None):
    """Uniformly sample (at most) `num_edges` distinct pairs i < j, none of them in `exclude`.

    Pairs are drawn on the device, canonicalised, de-duplicated in draw order and filtered against the
    excluded set with a sorted search on 64-bit keys (the reference does the same with a
    triangular-number bijection + np.unique on the host, preprocess.py:11-80).  Like the reference the
    result may hold fewer than `num_edges` rows."""
    n = int(n)
    num_edges = int(num_edges)
    n_all = n * (n - 1) // 2
    n_excl = 0 if exclude is None else int(exclude.shape[0])
    if num_edges > n_all - n_excl:
        raise ValueError("Cannot sample more than (%d choose 2) - %d = %d edges. (requested: %d edges)"
                         % (n, n_excl, n_all - n_excl, num_edges))
    dev = torch.device("cpu") if device is None and not torch.cuda.is_available() else util.cuda_device(device)
    gen = _generator(seed, dev)
    got = _sample_keys(lambda m: torch.randint(0, n, (m, 2), generator=gen, device=dev), n, num_edges, exclude, dev)
    return torch.stack([got // n, got % n], 1)


def sample_edges_touching(n, first, num_edges, exclude=None, seed=None, device=None):
    """At most `num_edges` distinct pairs i < j with at least one end in [first, n), none of them in `exclude`: u
    uniform over [first, n), v uniform over [0, n), v != u, then `sample_edges`' canonicalisation, draw-order
    de-duplication and exclusion.  `seed` defaults to a draw from the module RNG, so `pymde_b200.seed(s)` reproduces
    the pairs.  On `device` (a CPU device is allowed: the draws are the generator's on that device)."""
    n, first, num_edges = int(n), int(first), int(num_edges)
    dev = torch.device(device) if device is not None else util.cuda_device()
    gen = _generator(seed, dev)

    def draw(m):
        u = torch.randint(first, n, (m,), generator=gen, device=dev)
        v = torch.randint(0, n, (m,), generator=gen, device=dev)
        return torch.stack([u, v], 1)
    got = _sample_keys(draw, n, num_edges, exclude, dev)
    return torch.stack([got // n, got % n], 1)


def dissimilar_edges(n_items, similar_edges, num_edges=None, seed=None):
    """Edges NOT in `similar_edges`, approximately as many as there are similar ones."""
    if num_edges is None:
        num_edges = similar_edges.shape[0]
    return sample_edges(n_items, num_edges, exclude=similar_edges, seed=seed)


def deduplicate_edges(edges):
    e = edges if isinstance(edges, torch.Tensor) else torch.as_tensor(np.asarray(edges))
    lo, hi = torch.minimum(e[:, 0], e[:, 1]), torch.maximum(e[:, 0], e[:, 1])
    return torch.unique(torch.stack([lo, hi], 1), dim=0)


def scale(distances, natural_length):
    """Rescale so that RMS(distances) == natural_length (preprocess.py:132-138)."""
    rms = distances.float().pow(2).mean().sqrt()
    return (float(natural_length) / rms) * distances
