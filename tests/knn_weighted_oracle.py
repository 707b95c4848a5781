"""Test infrastructure: the CPU definition of ``KNeighborsClassifier(weights='distance')`` (never imported by the product
package).

The neighbours are ``kneighbors_oracle.kneighbors``: the set sklearn's index-order heap keeps (the one the uniform vote uses),
in canonical ascending (distance, training index) order, with exact fp64 distances.  On top of them, plain numpy:

1. weights (sk:neighbors/_base.py:74-114): ``1 / d`` (a correctly rounded division); in a row with a distance of exactly 0,
   1 where ``d == 0`` and 0 elsewhere;
2. label (sk:neighbors/_classification.py:281-307, sk:utils/extmath.py:791-862 ``weighted_mode``): per class c the row sum of
   ``template_c`` (the weight where the neighbour's class is c, 0.0 elsewhere) under numpy's association (``row_sum``), the
   lowest class with the largest sum;
3. proba (_classification.py:398-410): per class the weights added one column at a time from 0.0, divided by the row sum
   (``row_sum`` again, over the classes).

``row_sum`` restates numpy's float64 ``np.sum(a, axis=1)`` (pairwise_sum, numpy/_core/src/umath/loops_utils.h.src) with every
addition written out, so that the kernels have an explicit association to follow.
"""
import numpy as np

import kneighbors_oracle as kno


def row_sum(a):
    """np.sum(a, axis=1) for a float64 [n, m] array, association spelled out: below 8 columns, sequential from 0.0; up to
    128, eight accumulators seeded with columns 0-7, the following whole groups of 8 added column-wise, combined as
    ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), the remaining columns added sequentially; above 128, split at
    n2 = m/2 - (m/2) % 8 and the two halves' sums added."""
    a = np.asarray(a, dtype=np.float64)
    m = a.shape[1]
    if m < 8:
        res = np.zeros(a.shape[0])
        for i in range(m):
            res = res + a[:, i]
        return res
    if m <= 128:
        r = [a[:, j].copy() for j in range(8)]
        i = 8
        while i < m - m % 8:
            for j in range(8):
                r[j] = r[j] + a[:, i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(i, m):
            res = res + a[:, i]
        return res
    n2 = m // 2
    n2 -= n2 % 8
    return row_sum(a[:, :n2]) + row_sum(a[:, n2:])


def weights(dist):
    """rule 1: 1 / d, or the zero-distance indicator in rows that have a zero distance"""
    with np.errstate(divide="ignore"):
        w = 1.0 / dist
    zero = (dist == 0.0).any(axis=1)
    w[zero] = (dist[zero] == 0.0).astype(np.float64)
    return w


def vote(w, cls, n_classes):
    """rules 2 and 3 on the neighbours' weights and classes [n, k] (canonical order) -> (label int32 [n], proba [n, C])"""
    n, k = cls.shape
    best = np.zeros(n)
    label = np.zeros(n, np.int32)
    for c in range(n_classes):
        W = row_sum(np.where(cls == c, w, 0.0))
        win = W > best
        label[win] = c
        best[win] = W[win]
    P = np.zeros((n, n_classes))
    rows = np.arange(n)
    for i in range(k):
        P[rows, cls[:, i]] += w[:, i]
    return label, P / row_sum(P)[:, None]


def predict(spec, X, k=None):
    """-> (label int32 [n], proba float64 [n, C]) of the weights='distance' model `spec` (its own k unless given)"""
    k = int(spec["k"]) if k is None else int(k)
    dist, ind = kno.kneighbors(spec, X, k)
    cls = np.asarray(spec["y"], np.int64)[ind]
    return vote(weights(dist), cls, len(spec["classes"]))


def cross_class_ties(spec, X, k=None):
    """bool [n]: rows whose neighbour set holds two equally distant rows of different classes.  There sklearn's own label can
    depend on its undefined order among equal distances (for k >= 8, where numpy's row sum is pairwise)."""
    k = int(spec["k"]) if k is None else int(k)
    dist, ind = kno.kneighbors(spec, X, k)
    cls = np.asarray(spec["y"], np.int64)[ind]
    same_d = dist[:, :, None] == dist[:, None, :]
    diff_c = cls[:, :, None] != cls[:, None, :]
    return (same_d & diff_c).any(axis=(1, 2))
