"""CPU definition of SVC.predict_proba from one-vs-one decision values (test infrastructure): libsvm's Platt sigmoid and
pairwise coupling (sk:svm/src/libsvm/svm.cpp:2035-2043, 2046-2106, 2921-2958), vectorised over rows with the same
elementwise fp64 operations in the same order.  Rows leave the coupling loop independently (a per-row active mask).  The
only operation that is not a correctly rounded IEEE operation is exp (numpy's here, glibc's in scikit-learn, CUDA's on
the GPU).

``proba(dec, A, B)`` -> (p [n, C], rounds [n], margin [n]):
    rounds  libsvm's ``iter`` when the row stopped: the update rounds it ran
    margin  the smallest |max_error - eps| / eps over every stopping test of the row: how far the row was from taking one
            round more or fewer (rows under about 1e-9 could stop differently when exp differs in its last bit)
"""
import os

import numpy as np


def platt(dec, A, B):
    """r(i, j) for every pair: min(max(sigmoid_predict(dec, A, B), 1e-7), 1 - 1e-7) with libsvm's min / max"""
    f = dec * A + B
    with np.errstate(over="ignore"):
        en = np.exp(-f)
        ep = np.exp(f)
    s = np.where(f >= 0, en / (1.0 + en), 1.0 / (1 + ep))
    lo, hi = 1e-7, 1 - 1e-7
    s = np.where(s > lo, s, lo)
    return np.where(s < hi, s, hi)


def proba(dec, A, B):
    dec = np.asarray(dec, np.float64)
    n, P = dec.shape
    C = int(round((1 + np.sqrt(1 + 8 * P)) / 2))
    assert C * (C - 1) // 2 == P
    r = platt(dec, np.asarray(A, np.float64)[None, :], np.asarray(B, np.float64)[None, :])
    R = [[None] * C for _ in range(C)]                 # R[i][j]: r_ij [n]
    p = 0
    for i in range(C):
        for j in range(i + 1, C):
            R[i][j] = r[:, p]
            R[j][i] = 1 - r[:, p]
            p += 1
    Q = [[None] * C for _ in range(C)]
    for t in range(C):
        q = np.zeros(n)
        for j in range(C):
            if j != t:
                q = q + R[j][t] * R[j][t]
        Q[t][t] = q
        for j in range(t + 1, C):
            Q[t][j] = -R[j][t] * R[t][j]
            Q[j][t] = Q[t][j]
    k = C
    pr = [np.full(n, 1.0 / k) for _ in range(C)]
    eps, max_iter = 0.005 / k, max(100, k)
    rounds = np.full(n, max_iter, np.int64)
    margin = np.full(n, np.inf)
    active = np.ones(n, bool)
    for it in range(max_iter):
        if not active.any():
            break
        a = active
        Qp = [None] * C
        pQp = np.zeros(a.sum())
        for t in range(C):
            q = np.zeros(a.sum())
            for j in range(C):
                q = q + Q[t][j][a] * pr[j][a]
            Qp[t] = q
            pQp = pQp + pr[t][a] * q
        max_error = np.zeros(a.sum())
        for t in range(C):
            e = np.abs(Qp[t] - pQp)
            max_error = np.where(e > max_error, e, max_error)
        idx = np.flatnonzero(a)
        margin[idx] = np.minimum(margin[idx], np.abs(max_error - eps) / eps)
        stop = max_error < eps
        rounds[idx[stop]] = it
        active[idx[stop]] = False
        go = ~stop
        idx = idx[go]
        if idx.size == 0:
            break
        Qp = [q[go] for q in Qp]
        pQp = pQp[go]
        pa = [x[idx] for x in pr]
        for t in range(C):
            qtt = Q[t][t][idx]
            diff = (-Qp[t] + pQp) / qtt
            pa[t] = pa[t] + diff
            pQp = (pQp + diff * (diff * qtt + 2 * Qp[t])) / (1 + diff) / (1 + diff)
            for j in range(C):
                Qp[j] = (Qp[j] + diff * Q[t][j][idx]) / (1 + diff)
                pa[j] = pa[j] / (1 + diff)
        for t in range(C):
            pr[t][idx] = pa[t]
    return np.column_stack(pr), rounds, margin


def libsvm_dec(sk_dec, n_classes):
    """scikit-learn's decision_function(decision_function_shape='ovo') -> libsvm's signed values [n, P] (two classes:
    scikit-learn negates libsvm's value)"""
    d = np.asarray(sk_dec, np.float64)
    return -d[:, None] if n_classes == 2 else d


# ---------------------------------------------------------------- fitted probability models shared by the CPU and GPU tests
def labels_for(X, n_classes, seed):
    """n_classes labels for rows X: the quantiles of a seeded random projection, so that any class count has data"""
    w = np.random.default_rng(seed).normal(size=X.shape[1])
    z = X @ w
    edges = np.quantile(z, np.linspace(0, 1, n_classes + 1)[1:-1])
    return np.searchsorted(edges, z).astype(np.int32)


KERNEL_KW = {"linear": {}, "poly": dict(degree=3, coef0=-0.5), "rbf": {}, "sigmoid": dict(coef0=-0.5)}


def fit(kernel, n_classes, d=12, n=600, seed=5):
    """a fitted sklearn SVC(probability=True, random_state=0, decision_function_shape='ovo') on standardised synthetic flows
    (tests/svc_kernel_oracle.py) labelled into n_classes classes; max_iter capped (parity needs no converged model)"""
    import warnings

    from sklearn.svm import SVC

    import svc_kernel_oracle as so
    X, _ = so.flows(n, seed, d)
    y = labels_for(X, n_classes, seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)        # scikit-learn 1.9 deprecates probability=True
        warnings.simplefilter("ignore", UserWarning)          # ConvergenceWarning of the capped fits
        return SVC(kernel=kernel, probability=True, random_state=0, decision_function_shape="ovo", max_iter=20000,
                   **KERNEL_KW[kernel]).fit(X, y)


def load_fixture():
    """tests/golden/svc_proba.npz -> (spec, scikit-learn's OvO decision values, its predict_proba, its version)"""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "svc_proba.npz"), allow_pickle=False)
    spec = {"kind": "svc"}
    for k in z.files:
        if k.startswith("spec."):
            v = z[k]
            spec[k[5:]] = v.item() if v.ndim == 0 else v
    for key in ("n_features", "n_classes", "degree"):
        spec[key] = int(spec[key])
    for key in ("gamma", "coef0"):
        spec[key] = float(spec[key])
    spec["break_ties"] = bool(spec["break_ties"])
    spec["kernel"], spec["decision_function_shape"] = str(spec["kernel"]), str(spec["decision_function_shape"])
    return spec, z["dec_ovo"], z["proba"], str(z["sklearn_version"])
