"""`pymde_b200.embed_new_points` on ten Gaussian blobs in R^32: 20 000 fitted rows, 2 000 new rows from the same blobs.

The fitted rows stay where they were (the anchors of the solved problem are the embedding's rows, bit for bit), the
result is reproducible under MDE_B200_DETERMINISTIC=1, and its quality -- the share of new points whose nearest fitted
point in the embedding carries their blob label -- is compared with the reference workflow, `preserve_neighbors` on
the stacked data with every fitted row anchored (reference docs, "Embedding new points").

Measured on an H100 80GB HBM3 (700 W power limit): accuracy 1.000 for `embed_new_points` and 0.998 for the
reference workflow on this data (fp16, scipy.sparse and no-repulsion inputs: 1.000 each).  The floor (0.97) and the margin (0.02 below the reference workflow) leave room for
noise."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

N_OLD, N_NEW, D = 20000, 2000, 32
FLOOR, MARGIN = 0.97, 0.02


def _blobs(n, seed):
    centres = np.random.default_rng(123).standard_normal((10, D)) * 2.0
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, 10, n)
    return (centres[lab] + rng.standard_normal((n, D))).astype(np.float32), lab


@pytest.fixture(scope="module")
def fitted():
    import pymde_b200 as pm
    data, lab = _blobs(N_OLD, 1)
    new, new_lab = _blobs(N_NEW, 2)
    pm.seed(0)
    emb = pm.preserve_neighbors(data).embed()
    return data, lab, new, new_lab, emb


def _accuracy(emb_old, lab_old, emb_new, lab_new):
    E = emb_old.double()
    Y = emb_new.double()
    d = torch.cdist(Y, E)
    nearest = d.argmin(1).cpu().numpy()
    return float((lab_old[nearest] == lab_new).mean())


def test_anchors_stay_and_the_output_is_finite(fitted):
    from pymde_b200 import recipes
    data, _, new, _, emb = fitted
    mde, items = recipes._new_points_mde(data, emb, new)
    assert torch.equal(items[:N_NEW].cpu(), torch.arange(N_OLD, N_OLD + N_NEW))
    assert bool((items[N_NEW:] < N_OLD).all()) and bool((items[N_NEW + 1:] > items[N_NEW:-1]).all())
    X = mde.embed()
    assert torch.equal(X[N_NEW:], emb[items[N_NEW:]])
    out = X[:N_NEW]
    assert out.shape == (N_NEW, 2) and bool(torch.isfinite(out).all())
    # the problem holds only the new points and the fitted points they touch
    assert mde.n_items < N_OLD + N_NEW


def test_deterministic_mode_repeats_bit_for_bit(fitted, monkeypatch):
    import pymde_b200 as pm
    data, _, new, _, emb = fitted
    monkeypatch.setenv("MDE_B200_DETERMINISTIC", "1")
    pm.seed(0)
    a = pm.embed_new_points(data, emb, new)
    pm.seed(0)
    b = pm.embed_new_points(data, emb, new)
    assert a.dtype == torch.float32 and a.is_cuda and a.shape == (N_NEW, 2)
    assert torch.equal(a, b)


def test_quality_against_the_reference_workflow(fitted):
    import pymde_b200 as pm
    data, lab, new, new_lab, emb = fitted
    pm.seed(0)
    ours = pm.embed_new_points(data, emb, new)
    acc = _accuracy(emb, lab, ours, new_lab)
    pm.seed(0)
    stacked = np.vstack([data, new])
    ref = pm.preserve_neighbors(stacked, constraint=pm.Anchored(torch.arange(N_OLD, device="cuda"), emb)).embed()
    acc_ref = _accuracy(emb, lab, ref[N_OLD:], new_lab)
    print("accuracy: embed_new_points %.4f, reference workflow %.4f" % (acc, acc_ref))
    assert acc >= FLOOR, (acc, acc_ref)
    assert acc >= acc_ref - MARGIN, (acc, acc_ref)


def test_one_new_point(fitted):
    import pymde_b200 as pm
    data, lab, new, new_lab, emb = fitted
    out = pm.embed_new_points(data, emb, new[:1])
    assert out.shape == (1, 2) and bool(torch.isfinite(out).all())


def test_no_new_points(fitted):
    import pymde_b200 as pm
    data, _, new, _, emb = fitted
    out = pm.embed_new_points(data, emb, new[:0])
    assert out.shape == (0, 2) and out.dtype == torch.float32


def test_max_distance_leaves_points_without_attractive_edges(fitted):
    import pymde_b200 as pm
    from pymde_b200 import recipes
    data, _, new, _, emb = fitted
    far = np.concatenate([new[:50], new[:5] + 100.0])  # five new points far from everything
    mde, items = recipes._new_points_mde(data, emb, far, max_distance=8.0)
    w = mde.distortion_function.weights
    touched = torch.unique(mde.edges[w > 0].reshape(-1))
    assert int((touched < 55).sum()) < 55  # some new point has no attractive edge
    out = pm.embed_new_points(data, emb, far, max_distance=8.0)
    assert out.shape == (55, 2) and bool(torch.isfinite(out).all())


@pytest.mark.parametrize("kind", ["fp16", "sparse", "no_repulsion"])
def test_input_kinds(fitted, kind):
    import pymde_b200 as pm
    data, lab, new, new_lab, emb = fitted
    kw = {}
    if kind == "fp16":
        d, x = torch.from_numpy(data).half().cuda(), torch.from_numpy(new).half().cuda()
    elif kind == "sparse":
        d, x = sp.csr_matrix(data), sp.csr_matrix(new)
    else:
        d, x = data, new
        kw = dict(repulsive_penalty=None)
    pm.seed(0)
    out = pm.embed_new_points(d, emb, x, **kw)
    assert out.shape == (N_NEW, 2) and bool(torch.isfinite(out).all())
    acc = _accuracy(emb, lab, out, new_lab)
    print(kind, "accuracy %.4f" % acc)
    assert acc >= FLOOR - 0.05


def test_bad_input_is_rejected(fitted):
    import pymde_b200 as pm
    data, _, new, _, emb = fitted
    with pytest.raises(ValueError):
        pm.embed_new_points(data, emb[:-1], new)
    with pytest.raises(ValueError):
        pm.embed_new_points(data, emb, new[:, :-1])
    with pytest.raises(ValueError):
        pm.embed_new_points(data, emb[:, 0], new)
    with pytest.raises(ValueError):
        pm.embed_new_points(pm.Graph.from_edges(np.array([[0, 1]])), emb[:2], new)
