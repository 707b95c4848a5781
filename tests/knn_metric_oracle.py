"""Test infrastructure: the CPU definition of ``KNeighborsClassifier(metric='manhattan' | 'chebyshev')`` (never imported by
the product package).

1. rdist (sk:metrics/_dist_metrics.pyx.tp, ManhattanDistance / ChebyshevDistance): fp64, features in order from 0.0 --
   manhattan adds ``|x_f - t_f|`` one feature at a time (a sequential loop: numpy's ``np.abs(X - t).sum(axis=1)`` is
   pairwise from 8 terms on and is NOT this definition), chebyshev takes the running maximum (exact).  Rows are widened to
   float64 first.  The distance is rdist itself.
2. The neighbour set: scikit-learn's index-order heap (sk:utils/_heap.pyx heap_push: training rows offered in index order,
   ``val >= root`` rejected, the left child preferred on ties), restated below for all queries at once.  Among rows tied
   at the k-th rdist it does NOT keep the lowest indices: which ones it keeps depends on its history.  The kept rows are
   returned in canonical ascending (rdist, training index) order, ``np.lexsort((index, rdist))``.
3. Votes: the uniform count rule (the lowest class with the most neighbours; proba = count / k) or the distance-weighted
   vote of ``knn_weighted_oracle`` (weights 1 / distance, the zero-distance rule, numpy's associations).
"""
import numpy as np

import knn_weighted_oracle as kwo

METRICS = ("manhattan", "chebyshev")


def rdist(metric, X, F):
    """[n, m] rdist of every row of X against every row of F, rule 1"""
    X = np.asarray(X, dtype=np.float64)
    F = np.asarray(F, dtype=np.float64)
    acc = np.zeros((X.shape[0], F.shape[0]))
    for f in range(X.shape[1]):
        term = np.abs(X[:, f:f + 1] - F[None, :, f])
        acc = acc + term if metric == "manhattan" else np.maximum(acc, term)
    return acc


def heap(R, k):
    """rule 2 on the rdist matrix R [n, n_train]: every row's k-slot max-heap after the pushes of training rows 0, 1, ...
    -> (values [n, k], indices [n, k]) in heap order"""
    n, m = R.shape
    hv = np.full((n, k), np.finfo(np.float64).max)
    hi = np.zeros((n, k), np.int64)
    for j in range(m):
        sel = np.nonzero(R[:, j] < hv[:, 0])[0]
        if sel.size == 0:
            continue
        val = R[sel, j]
        cur = np.zeros(sel.size, np.int64)
        active = np.ones(sel.size, bool)
        while True:
            l, r = 2 * cur + 1, 2 * cur + 2
            vl = np.where(l < k, hv[sel, np.minimum(l, k - 1)], -np.inf)
            vr = np.where(r < k, hv[sel, np.minimum(r, k - 1)], -np.inf)
            to_l = np.where(r < k, (vl >= vr) & (val < vl), vl > val)
            to_r = (r < k) & (vl < vr) & (val < vr)
            go = active & (to_l | to_r)
            if not go.any():
                break
            nxt = np.where(to_l, l, r)
            rows, src = sel[go], nxt[go]
            hv[rows, cur[go]] = hv[rows, src]
            hi[rows, cur[go]] = hi[rows, src]
            cur[go] = src
            active = go
        hv[sel, cur] = val
        hi[sel, cur] = j
    return hv, hi


def kneighbors(spec, X, n_neighbors, metric=None):
    """-> (dist float64 [n, m], ind int64 [n, m]), rule 2, in the spec's metric unless given"""
    metric = spec["metric"] if metric is None else metric
    X = np.ascontiguousarray(X, dtype=np.float64)
    F = np.ascontiguousarray(spec["fit_X"], dtype=np.float64)
    m = int(n_neighbors)
    n = X.shape[0]
    dist, ind = np.zeros((n, m)), np.zeros((n, m), np.int64)
    step = max(1, 25_000_000 // max(1, F.shape[0]))
    for lo in range(0, n, step):
        hv, hi = heap(rdist(metric, X[lo:lo + step], F), m)
        order = np.lexsort((hi, hv), axis=1)
        ind[lo:lo + step] = np.take_along_axis(hi, order, axis=1)
        dist[lo:lo + step] = np.take_along_axis(hv, order, axis=1)
    return dist, ind


def predict(spec, X, k=None, metric=None):
    """-> (label int32 [n], proba float64 [n, C]) of the model `spec` (its own k, weights and metric unless given)"""
    k = int(spec["k"]) if k is None else int(k)
    dist, ind = kneighbors(spec, X, k, metric)
    cls = np.asarray(spec["y"], np.int64)[ind]
    C = len(spec["classes"])
    if spec.get("weights", "uniform") == "distance":
        return kwo.vote(kwo.weights(dist), cls, C)
    counts = np.stack([(cls == c).sum(axis=1) for c in range(C)], axis=1)
    return np.argmax(counts, axis=1).astype(np.int32), counts / float(k)


def cross_class_ties(spec, X, k=None, metric=None):
    """bool [n]: rows whose neighbour set holds two equally distant rows of different classes"""
    k = int(spec["k"]) if k is None else int(k)
    dist, ind = kneighbors(spec, X, k, metric)
    cls = np.asarray(spec["y"], np.int64)[ind]
    return ((dist[:, :, None] == dist[:, None, :]) & (cls[:, :, None] != cls[:, None, :])).any(axis=(1, 2))
