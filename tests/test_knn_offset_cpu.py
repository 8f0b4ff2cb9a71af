"""Why the dense exact k-nearest-neighbour searches centre their operand and certify every row, on the CPU.

The tensor-core searches (csrc/mde_knn.cu) rank candidates by s(y) = ||y^||^2 - 2 <q^, y^>~, where y^ = fl(y - mu)
are the centred fp32 values, ||y^||^2 their fp32 norm and <., .>~ the cross term of the bf16 hi / lo split
(y^ = h + l + r, |r| <= 2^-16 |y^|; products h h + h l + l h, exact in fp32, accumulated in fp32).  They keep the KK
best scores per row and re-rank those exactly.  The simulation below keeps 32 and shows the table of the families:
without centring a global offset makes the kept list rounding noise; centring repairs that, but not far-apart
clusters, whose rows must be searched directly.

The certificate needs a bound E(q) >= |s(y) - S(y)| for every y, S(y) = ||q - y||^2 - ||q - mu||^2 the exact score.
With q* = q - mu and y* = y - mu exact, u = 2^-24, K the padded width (d rounded up to 64) and M^2 >= max_y ||y^||^2:

  cross term   <q^,y^>~ - <q*,y*> = (<q^,y^>~ - <q^,y^>) + (<q^,y^> - <q*,y*>).
               The split drops l_q l_y and the residuals: per element at most (2^-16 (1 + 2^-8)^2 + 2 2^-16 (1 + 2^-8))
               |q^_j||y^_j| < 3.1 2^-16 |q^_j||y^_j|, and by Cauchy-Schwarz the sum is at most 3.1 2^-16 |q^||y^|.
               The fp32 accumulation of m = 3 K exact products adds at most 2 u per addition (2 u allows for tensor
               cores that truncate rather than round): 2 u m sum |products| <= 2 u m (1 + 2^-7) |q^||y^|.
               Centring rounds each element by at most u: |<q^,y^> - <q*,y*>| <= (2 u + u^2) |q*||y*|.
  norm         the fp32 sum of K squares, ceil(K / 32) sequential fmas per lane and a 5-level butterfly, plus the
               rounding of y^: |fl||y^||^2 - ||y*||^2| <= (ceil(K / 32) + 8) u ||y*||^2.
  score        the tile forms fl(norm - 2 cross) in one fma: at most u (M^2 + 2 |q^| M).
  underflow    at most 2^-126 per product and per square: (2 m + K) 2^-126.

So E(q) = sigma (2 a_cross |q^| M + a_norm M^2 + a_abs) with a_cross = 3.1 2^-16 + 2.01 u + 2 u m + u and
a_norm = (ceil(K / 32) + 9) u; sigma = 2 covers the second-order factors (1 + 2^-7, |y^| against |y*|).  A centred
16-bit operand replaces the split term by 2 eps + eps^2 (eps = 2^-11 fp16, 2^-8 bf16) with m = K, and fp16 adds 2^-25
per element for its subnormals.  The searches centre only when that gives the smaller bound: uncentred (mu = 0), a
16-bit element is its own exact operand and a_cross = 2 u m + u, which is what keeps 16-bit data near the origin on
the tensor cores.  The check below measures the score error of the simulated split on every row and
candidate of the families against E(q) / sigma: the bound holds without the safety factor.

A row is certified when d2_k (1 + delta) / (1 - delta) - ||q^||^2 + E(q) < t - E(q), where t is the worst kept score
and d2_k the k-th re-ranked fp32 distance (delta = (ceil(d / 32) + 8) u bounds the re-rank's relative rounding): every
row not kept scored at least t, so its exact distance D is at least t - E + ||q*||^2 > d2_k (1 + delta) / (1 - delta),
and its fp32 distance, at least D (1 - delta), exceeds d2_k."""
import math

import numpy as np
import pytest
import torch

from tests.test_gpu_knn_offset import FAR, OFFSET, family

U = 2.0 ** -24


def split(X):
    h = X.to(torch.bfloat16).float()
    l = (X - h).to(torch.bfloat16).float()
    return h, l


def scores(X, centre):
    """The simulated tile scores [n, n] (fp32) and the fp32 centred matrix and norms."""
    Xc = X - X.double().mean(0).float() if centre else X
    h, l = split(Xc)
    norms = (Xc * Xc).sum(1)
    cross = h @ h.T + h @ l.T + l @ h.T
    s = torch.addcmul(norms[None, :], cross, torch.tensor(-2.0))  # one rounding, as the tile's fma
    s.fill_diagonal_(float("inf"))
    return s, Xc, norms


def wrong_fraction(X, k, centre, kk=32):
    """Fraction of rows whose k-th returned neighbour (top kk by score, re-ranked exactly) is farther than the true."""
    s, _, _ = scores(X, centre)
    cand = torch.topk(s, kk, dim=1, largest=False)[1]
    Xd = X.double()
    exact = ((Xd[:, None, :] - Xd[cand]) ** 2).sum(-1)
    got = torch.sort(exact, 1)[0][:, k - 1]
    Xc = Xd - Xd.mean(0)
    full = ((Xc * Xc).sum(1)[:, None] + (Xc * Xc).sum(1)[None, :] - 2.0 * Xc @ Xc.T)
    full.fill_diagonal_(float("inf"))
    want = torch.topk(full, k, dim=1, largest=False)[0][:, k - 1]
    return float((got > want * (1 + 1e-6) + 1e-12).double().mean())


@pytest.mark.parametrize("name", ["iso16"] + OFFSET + ["far_r1000_d16", "far_r30_d8"])
def test_families_separate_a_centred_search_from_an_uncentred_one(name):
    X = torch.from_numpy(family(name))
    raw, cen = wrong_fraction(X, 15, False), wrong_fraction(X, 15, True)
    if name == "iso16":
        assert raw == 0 and cen == 0
    elif name in OFFSET:
        assert cen == 0
        if name != "off100_d8":  # (0.7 % of its rows in the table)
            assert raw > 0.9, raw
        else:
            assert raw > 0
    else:
        assert raw > 0.3 and cen > 0.3, (raw, cen)


def error_bound(d, qn, M2):
    K = (d + 63) // 64 * 64
    m = 3 * K
    a_cross = 3.1 * 2.0 ** -16 + 2.01 * U + 2 * U * m + U
    a_norm = ((K + 31) // 32 + 9) * U
    a_abs = (2 * m + K) * 2.0 ** -126
    return 2 * a_cross * qn.sqrt() * math.sqrt(M2) + a_norm * M2 + a_abs


@pytest.mark.parametrize("name", ["iso16"] + OFFSET + FAR + ["relu_shift", "pixels", "dup_off500"])
def test_score_error_is_within_the_certificate_bound(name):
    X = torch.from_numpy(family(name, n=2000))
    s, Xc, norms = scores(X, True)
    Xd = X.double()
    mu = Xd.mean(0).float().double()  # the fp32 mean the search subtracts
    Xs = Xd - mu
    exact = (Xs * Xs).sum(1)[None, :] - 2.0 * Xs @ Xs.T  # S(y), in fp64
    exact.fill_diagonal_(float("inf"))
    E = error_bound(X.shape[1], norms.double(), float(norms.max()))
    err = (s.double() - exact).nan_to_num(0.0, posinf=0.0).abs()
    worst = float((err / E[:, None]).max())
    assert worst <= 1.0, worst
    # the fp32 norms of the queries too (the certificate's right-hand E)
    assert bool(((norms.double() - (Xs * Xs).sum(1)).abs() <= E).all())
