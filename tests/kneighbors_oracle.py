"""Test infrastructure: the CPU definition of ``KNeighborsClassifier.kneighbors`` (never imported by the product package).

The neighbour SET is the oracle's restatement of sklearn's index-order heap (``oracle.knn(..., return_neighbors=True)``,
oracle/tcsdn_oracle.c), the same set ``predict`` votes on.  Each row is then put in the canonical order -- ascending
(distance, training index) -- and the distances are ``sqrt(sum_f (x_f - t_f)^2)``: fp64, features in order, a multiply and
an add per feature (numpy does not fuse them), correctly rounded square root.
"""
import numpy as np

import oracle


def kneighbors(spec, X, n_neighbors):
    """-> (dist float64 [n, m], ind int64 [n, m]) for m = n_neighbors; X is widened to float64 first."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    F = np.ascontiguousarray(spec["fit_X"], dtype=np.float64)
    m = int(n_neighbors)
    _, _, ind = oracle.knn(dict(spec, k=m), X, want_scores=False, return_neighbors=True)
    rd = np.zeros(ind.shape)
    for f in range(X.shape[1]):
        df = X[:, f:f + 1] - F[ind, f]
        rd = rd + df * df
    order = np.lexsort((ind, rd), axis=1)
    ind = np.take_along_axis(ind, order, axis=1)
    rd = np.take_along_axis(rd, order, axis=1)
    return np.sqrt(rd), ind


def canonical(dist, ind):
    """sklearn's rows put in the canonical order: ascending (distance, index)."""
    order = np.lexsort((ind, dist), axis=1)
    return np.take_along_axis(dist, order, axis=1), np.take_along_axis(ind, order, axis=1)


def exclude_self(dist, ind):
    """sklearn's rule for ``kneighbors(X=None)`` applied to a query of fit_X with m + 1 neighbours
    (sk:neighbors/_base.py:930-956): drop the row's own index, or the first column where it was not kept."""
    n, m1 = ind.shape
    keep = ind != np.arange(n)[:, None]
    keep[np.all(keep, axis=1), 0] = False
    return dist[keep].reshape(n, m1 - 1), ind[keep].reshape(n, m1 - 1)
