"""Test infrastructure: the CPU definition of ``GaussianNB.fit`` and ``KMeans.fit`` (Lloyd from an init array, n_init=1)
as csrc/fit.cu computes them (never imported by the product package).

Rows are widened to float64 first; every sum and mean below is EXACT (Python integers over a power of two per column) and
rounded once, so the GPU tests can hold the kernels' fp64 sums to a rounding bound around the exact value.

GaussianNB (sk:naive_bayes.py:385-476 with n_past = 0): per class the count, mean and variance divided by the count,
``epsilon_ = var_smoothing * max_j Var(X_j)`` added to every variance, ``class_prior_ = count / n``.

KMeans (sk:cluster/_kmeans.py:630-758 ``_kmeans_single_lloyd``, one iteration = sk:cluster/_k_means_lloyd.pyx:23-165):
1. E-step: the first minimum of the exact squared distance to the centres;
2. M-step: exact per-cluster sums and counts of the rows;
3. empty clusters (sk:cluster/_k_means_common.pyx:167-211): unless every row lies exactly on its centre, each empty
   cluster in index order takes the next row in decreasing exact distance to its centre (equal distances: lower row
   first); the row leaves its cluster's sum and count and is the empty cluster's sum, count 1.  sklearn orders the rows
   by ``np.argpartition``, which agrees for one or two empty clusters and is undefined from three on;
4. averaging (sk:cluster/_k_means_common.pyx:274-295): count > 0: exact mean; count 0 (nothing relocated, or a donor
   that gave its only row): the entry of the largest cluster (first maximum) as sklearn's loop has left it -- its mean
   when that cluster comes earlier, else its sum in sklearn's mean-centred rows, ``sum(x) - (count - 1) * mean(X)``;
5. stop when the labels did not change, or when ``sum((new - old)^2) <= mean_j(Var(X_j)) * tol``; after a stop that was
   not "labels unchanged" one more E-step; inertia last.

Made for a few tens of thousands of rows.
"""
import math
from fractions import Fraction

import numpy as np

U = 2.0 ** -53


def gamma(n):
    """Higham's gamma_n: the relative error bound of n rounded fp64 operations in a chain"""
    return n * U / (1.0 - n * U)


class ExactRows:
    """X [n][d] float64 as Python integers: X[i, j] == ints[j][i] / 2**shift[j] exactly."""

    def __init__(self, X):
        X = np.ascontiguousarray(X, np.float64)
        if not np.isfinite(X).all():
            raise ValueError("non-finite rows")
        self.X = X
        self.ints, self.shift = [], []
        for j in range(X.shape[1]):
            m, e = np.frexp(X[:, j])
            mi = (m * 2.0 ** 53).astype(np.int64).tolist()   # exact: X = mi * 2**(e - 53)
            e = (e.astype(np.int64) - 53).tolist()
            s = -min(e)
            self.ints.append(np.array([a << (b + s) for a, b in zip(mi, e)], dtype=object))
            self.shift.append(s)

    def group_sums(self, labels, k, square=False):
        """-> (S, cnt): S[c][j] = exact sum of X[i, j] (or X[i, j]^2) over rows labelled c, as a Fraction; cnt int [k]"""
        labels = np.asarray(labels)
        order = np.argsort(labels, kind="stable")
        cnt = np.bincount(labels, minlength=k)
        start = np.concatenate([[0], np.cumsum(cnt)])
        S = [[Fraction(0)] * len(self.ints) for _ in range(k)]
        for j, col in enumerate(self.ints):
            col = col[order]
            if square:
                col = col * col
            den = 1 << (self.shift[j] * (2 if square else 1))
            for c in range(k):
                if cnt[c]:
                    S[c][j] = Fraction(int(col[start[c]:start[c + 1]].sum()), den)
        return S, cnt


def _round(F):
    return np.array([[float(v) for v in row] for row in F], dtype=np.float64)


def _sq_dist_exact(x, c):
    return sum((Fraction(float(a)) - Fraction(float(b))) ** 2 for a, b in zip(x, c))


def gnb_fit(X, y, var_smoothing=1e-9):
    """-> dict: classes, class_count, class_prior, theta, var, epsilon (float64, each the exact value rounded once) and
    theta_exact, var_exact (without epsilon), epsilon_exact (Fractions)"""
    E = ExactRows(X)
    n, d = E.X.shape
    classes, yi = np.unique(np.asarray(y), return_inverse=True)
    C = len(classes)
    S1, cnt = E.group_sums(yi, C)
    S2, _ = E.group_sums(yi, C, square=True)
    A1, _ = E.group_sums(np.zeros(n, np.int64), 1)
    A2, _ = E.group_sums(np.zeros(n, np.int64), 1, square=True)
    theta = [[S1[c][j] / int(cnt[c]) for j in range(d)] for c in range(C)]
    var = [[S2[c][j] / int(cnt[c]) - theta[c][j] ** 2 for j in range(d)] for c in range(C)]
    eps = Fraction(var_smoothing) * max(A2[0][j] / n - (A1[0][j] / n) ** 2 for j in range(d))
    return dict(classes=classes, class_count=cnt.astype(np.float64), class_prior=np.array([int(c) / n for c in cnt]),
                theta=_round(theta), var=_round([[v + eps for v in row] for row in var]), epsilon=float(eps),
                theta_exact=theta, var_exact=var, epsilon_exact=eps)


def _sq_dist(X, C):
    """fp64 ||x - c||^2 [n][k] by differences: within gamma(d + 2) relative of the exact value"""
    out = np.empty((len(X), len(C)))
    for s in range(0, len(X), 4096):
        out[s:s + 4096] = ((X[s:s + 4096, None, :] - C[None, :, :]) ** 2).sum(axis=2)
    return out


def estep(X, centers):
    """labels int32 [n]: the first minimum of the exact ||x - c||^2.  Rows whose fp64 distances cannot settle it are
    decided with Fractions."""
    X = np.asarray(X, np.float64)
    D = _sq_dist(X, centers)
    labels = np.argmin(D, axis=1).astype(np.int32)
    best = D[np.arange(len(X)), labels]
    band = D <= (best * (1.0 + 4.0 * gamma(X.shape[1] + 3)))[:, None]
    for i in np.nonzero(band.sum(axis=1) > 1)[0]:
        cand = np.nonzero(band[i])[0]
        exact = [_sq_dist_exact(X[i], centers[c]) for c in cand]
        labels[i] = cand[int(np.argmin(exact))]        # Fractions compare exactly; argmin takes the first
    return labels


def farthest(X, centers, labels, m):
    """the m rows farthest from their own centre (exact distance, decreasing; equal distances: lower row first), and
    whether the largest distance is 0"""
    X = np.asarray(X, np.float64)
    dist = ((X - centers[labels]) ** 2).sum(axis=1)
    kth = np.sort(dist)[-m]
    cand = np.nonzero(dist >= kth * (1.0 - 4.0 * gamma(X.shape[1] + 3)))[0]
    exact = {int(i): _sq_dist_exact(X[i], centers[labels[i]]) for i in cand}
    order = sorted(exact, key=lambda i: (-exact[i], i))[:m]
    return order, exact[order[0]] == 0


def kmeans_fit(X, init, max_iter=300, tol=1e-4):
    """-> dict: labels int32 [n], centers float64 [k][d] (exact values rounded once), centers_exact (Fractions),
    counts (the last M-step's cluster counts, after relocation), n_iter, inertia (math.fsum of the fp64 terms (x - c)^2 for the final centres: within 3u of exact), n_relocated
    (rows moved into empty clusters over the run)"""
    E = ExactRows(X)
    X = E.X
    n, d = X.shape
    centers = np.array(init, dtype=np.float64)
    k = len(centers)
    mean_x = X.mean(axis=0)                       # what sklearn centres the rows on
    tol_ = float(np.mean(np.var(X, axis=0)) * tol)
    labels_old = np.full(n, -1, np.int32)
    strict, relocated = False, 0
    exact = None
    for it in range(max_iter):
        labels = estep(X, centers)
        S, cnt = E.group_sums(labels, k)
        cnt = [int(c) for c in cnt]
        empty = [c for c in range(k) if cnt[c] == 0]
        if empty:
            far, all_zero = farthest(X, centers, labels, len(empty))
            if not all_zero:
                for to, r in zip(empty, far):
                    frm = int(labels[r])
                    row = [Fraction(float(v)) for v in X[r]]
                    S[frm] = [a - b for a, b in zip(S[frm], row)]
                    S[to] = row
                    cnt[frm] -= 1
                    cnt[to] = 1
                    relocated += 1
        big = int(np.argmax(cnt))
        exact = [None] * k
        for c in range(k):
            if cnt[c]:
                exact[c] = [s / cnt[c] for s in S[c]]
            elif big < c:
                exact[c] = [Fraction(float(v)) for v in exact[big]]      # sklearn copies the rounded mean
            else:
                exact[c] = [S[big][j] - (cnt[big] - 1) * Fraction(float(mean_x[j])) for j in range(d)]
        new = _round(exact)
        shift = float(((new - centers) ** 2).sum())
        centers = new
        if np.array_equal(labels, labels_old):
            strict = True
            break
        if shift <= tol_:
            break
        labels_old = labels
    if not strict:
        labels = estep(X, centers)
    return dict(labels=labels, centers=centers, centers_exact=exact, counts=cnt, n_iter=it + 1,
                inertia=inertia(X, centers, labels), n_relocated=relocated)


def inertia(X, centers, labels):
    """math.fsum of the fp64 terms (x - c_label)^2: within 3u relative of the exact inertia"""
    X = np.asarray(X, np.float64)
    return math.fsum(((X - centers[labels]) ** 2).ravel().tolist())
