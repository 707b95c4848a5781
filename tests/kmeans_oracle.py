"""CPU definition of KMeans.transform, KMeans.score and the k-means++ seeding (csrc/kmeans_dist.cuh, scorers.cu,
kmeanspp.cu).

* ``sqdist`` is scikit-learn's _euclidean_dense_dense (sk:cluster/_k_means_common.pyx:16-43) vectorised: features in
  groups of four, ((d0 d0 + d1 d1) + d2 d2) + d3 d3 added to the running result, then the rest one at a time, in fp64
  numpy operations (each rounded once, no FMA).
* ``kmeans_plusplus`` is sklearn.cluster._kmeans._kmeans_plusplus with unit weights on the rows as given, with
  scikit-learn's draws and EXACT sums (integers in units of the smallest binary exponent).  For every decision it reports
  the margin, relative to the potential: the draw to the two prefix sums around it, and the best candidate's potential
  to the next different one.
"""
from bisect import bisect_left
from fractions import Fraction
import math

import numpy as np

U = 2.0 ** -53


def sqdist(X, C):
    """[n, k] squared distances of the rows X [n, d] to the centres C [k, d] (both widened to float64)."""
    X = np.asarray(X, np.float64)
    C = np.asarray(C, np.float64)
    if len(X) > 4096:
        return np.concatenate([sqdist(X[i:i + 4096], C) for i in range(0, len(X), 4096)])
    D = X[:, None, :] - C[None, :, :]
    sq = D * D
    d = X.shape[1]
    s = np.zeros((X.shape[0], C.shape[0]))
    for g in range(d // 4):
        j = 4 * g
        s = s + (((sq[..., j] + sq[..., j + 1]) + sq[..., j + 2]) + sq[..., j + 3])
    for j in range(d - d % 4, d):
        s = s + sq[..., j]
    return s


def transform(X, C):
    return np.sqrt(sqdist(X, C))


def inertia_terms(X, C, labels):
    """per-row squared distance to the row's own centre"""
    X = np.asarray(X, np.float64)
    out = np.empty(len(X))
    for c in np.unique(labels):
        sel = labels == c
        out[sel] = sqdist(X[sel], C[c:c + 1])[:, 0]
    return out


def gamma(n):
    return n * U / (1 - n * U)


def _units(v):
    """exact integers m_i and a common exponent e with v_i = m_i * 2**e (v >= 0, finite)"""
    mant, ex = np.frexp(v)
    m = (mant * 2.0 ** 53).astype(np.int64)
    nz = v > 0
    e = int(ex[nz].min()) - 53 if nz.any() else 0
    shift = np.where(nz, ex - 53 - e, 0)
    return [int(a) << int(b) for a, b in zip(m.tolist(), shift.tolist())], e


def _exact(v):
    ints, e = _units(v)
    return sum(ints), e


def kmeans_plusplus(X, k, random_state=None, n_local_trials=None):
    """-> (indices, draw margins, choice margins).  Margins are relative to the potential of their round."""
    from sklearn.utils import check_random_state
    X = np.asarray(X, np.float64)
    n = len(X)
    L = 2 + int(np.log(k)) if n_local_trials is None else int(n_local_trials)
    rs = check_random_state(random_state)
    w = np.ones(n)
    first = int(rs.choice(n, p=w / w.sum()))
    idx = [first]
    closest = sqdist(X, X[first:first + 1])[:, 0]
    draw_margins, choice_margins = [], []
    for _ in range(1, k):
        u = rs.uniform(size=L)
        ints, e = _units(closest)
        cum = list(_accumulate(ints))
        pot = cum[-1]
        cands = []
        for ul in u:
            r = Fraction(float(ul)) * pot
            i = min(bisect_left(cum, r), n - 1)
            cands.append(i)
            if pot > 0:
                hi = cum[i] - r
                lo = r - (cum[i - 1] if i > 0 else 0)
                draw_margins.append(float(min(hi, lo) / pot) if i > 0 else float(hi / pot))
        news = [np.minimum(closest, sqdist(X, X[c:c + 1])[:, 0]) for c in cands]
        pots = [Fraction(*_exact_ratio(v)) for v in news]
        best = min(range(L), key=lambda l: (pots[l], l))
        others = [p for p in pots if p != pots[best]]
        if others and pots[best] > 0:
            choice_margins.append(float((min(others) - pots[best]) / pots[best]))
        idx.append(cands[best])
        closest = news[best]
    return np.array(idx, np.int64), np.array(draw_margins), np.array(choice_margins)


def _exact_ratio(v):
    s, e = _exact(v)
    return (s * 2 ** e, 1) if e >= 0 else (s, 2 ** -e)


def _accumulate(ints):
    t = 0
    for a in ints:
        t += a
        yield t


def seeding_bound(n):
    """relative error of the GPU's prefix sums and potentials (kmeanspp.cu: 31 roundings per level of its 32-ary tree,
    the nesting adds, the product u * pot), with a factor 4 to spare"""
    levels = 2 + max(1, math.ceil(math.log(max(n, 2), 32)))
    return 4 * (31 * levels + levels + 2) * U
