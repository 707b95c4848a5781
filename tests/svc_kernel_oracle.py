"""CPU restatement of the fp64 SVC definition for the linear, poly and sigmoid kernels (test infrastructure), and an exact
(fractions.Fraction) model of the linear collapsed path's certificate (csrc/svc.cu, header).

The definition (sk:svm/src/libsvm/svm.cpp:452-515, 2846-2904):
    K_s    linear dot(x, sv_s); poly powi(gamma * dot + coef0, degree); sigmoid tanh(gamma * dot + coef0)
    dec_p  sum_{s in class i} coef[j-1][s] K_s + sum_{s in class j} coef[i][s] K_s - rho_p,  rho = -intercept
    label  first class with the most votes, dec_p > 0 voting for i
Here dot is summed in feature order without FMA and the per-class sums run in support-vector order (libsvm's loop); the
CUDA kernel uses fma chains and CUDA's tanh, so values agree to a few ulps of the terms, not bit for bit.
"""
from fractions import Fraction

import numpy as np

KERNELS = ("linear", "poly", "sigmoid")


def powi(base, times):
    """libsvm's square-and-multiply loop, elementwise"""
    tmp, ret = np.array(base, dtype=np.float64), np.ones_like(base, dtype=np.float64)
    t = int(times)
    while t > 0:
        if t % 2 == 1:
            ret = ret * tmp
        tmp = tmp * tmp
        t //= 2
    return ret


def kernel_values(spec, X):
    """K [n, n_sv] of a linear / poly / sigmoid spec"""
    sv = np.asarray(spec["sv"], np.float64)
    dot = np.zeros((X.shape[0], sv.shape[0]))
    for j in range(X.shape[1]):
        dot = dot + X[:, j, None] * sv[None, :, j]
    k, g, c0 = spec["kernel"], float(spec["gamma"]), float(spec.get("coef0", 0.0))
    if k == "linear":
        return dot
    t = g * dot + c0
    if k == "poly":
        return powi(t, int(spec.get("degree", 3)))
    if k == "sigmoid":
        return np.tanh(t)
    raise ValueError(k)


def _pairs(spec):
    """per pair p = (i, j): (support-vector indices in the definition's order, their coefficients)"""
    nsup = np.asarray(spec["n_support"], np.int64)
    dual = np.asarray(spec["dual_coef"], np.float64)
    start = np.concatenate([[0], np.cumsum(nsup)])
    C = len(nsup)
    out = []
    for i in range(C):
        for j in range(i + 1, C):
            si, sj = np.arange(start[i], start[i + 1]), np.arange(start[j], start[j + 1])
            out.append((np.concatenate([si, sj]), np.concatenate([dual[j - 1, si], dual[i, sj]])))
    return out


def predict(spec, X, chunk=4096):
    """-> (labels int32 [n], dec [n, P] with libsvm's sign, scale [n, P] = sum_s |c_ps K_s| + |rho_p|)"""
    X = np.ascontiguousarray(X, np.float64)
    n = X.shape[0]
    nsup = np.asarray(spec["n_support"])
    C = len(nsup)
    P = C * (C - 1) // 2
    rho = -np.asarray(spec["intercept"], np.float64)
    pairs = _pairs(spec)
    labels = np.empty(n, np.int32)
    dec = np.empty((n, P))
    scale = np.empty((n, P))
    for r0 in range(0, n, chunk):
        K = kernel_values(spec, X[r0:r0 + chunk])
        m = K.shape[0]
        vote = np.zeros((m, C), np.int64)
        p = 0
        for i in range(C):
            for j in range(i + 1, C):
                idx, cf = pairs[p]
                s = np.zeros(m)
                for t in range(len(idx)):       # libsvm's sequential sum in support-vector order
                    s = s + cf[t] * K[:, idx[t]]
                dv = s - rho[p]
                dec[r0:r0 + m, p] = dv
                scale[r0:r0 + m, p] = np.abs(K[:, idx]) @ np.abs(cf) + abs(rho[p])
                vote[:, i] += dv > 0
                vote[:, j] += ~(dv > 0)
                p += 1
        labels[r0:r0 + m] = np.argmax(vote, axis=1)        # first maximum
    return labels, dec, scale


# ---------------------------------------------------------------- exact model of the collapsed path (csrc/svc.cu)
def fma(a, b, c):
    """a * b + c rounded once (float(Fraction) is correctly rounded)"""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def linear_params(spec):
    """the create-time parameters of svc_linear_create, with the same operations: per pair (W~, A^, rho, K, F)"""
    sv = np.asarray(spec["sv"], np.float64)
    d = sv.shape[1]
    u, tiny = 2.0 ** -53, 2.0 ** -1074
    rho = -np.asarray(spec["intercept"], np.float64)
    out = []
    for p, (idx, cf) in enumerate(_pairs(spec)):
        m = float(len(idx))
        csum = 0.0
        for c in cf:
            csum += abs(float(c))
        W, A = [], []
        for jj in range(d):
            w, a = 0.0, 0.0
            for s, c in zip(idx, cf):
                v = float(sv[s, jj])
                w = fma(float(c), v, w)
                a += abs(float(c)) * abs(v)
            W.append(w)
            A.append(float(np.nextafter(a * (1.0 + 4.0 * m * u) + m * tiny, np.inf)))
        g = (d + m + 2.0) * u / (1.0 - (d + m + 2.0) * u)
        K = float(np.nextafter(2.0 * g * (1.0 + 4.0 * (d + 3.0) * u), np.inf))
        F = float(np.nextafter(2.0 * ((csum * d + m + 2.0 * d + 8.0) * tiny), np.inf))
        out.append((W, A, float(rho[p]), K, F))
    return out


def linear_collapsed(params, x):
    """per pair (dec~, E) as svc_linear_kernel evaluates them"""
    res = []
    for W, A, rho, K, F in params:
        dv, s = 0.0, 0.0
        for w, a, xj in zip(W, A, x):
            dv = fma(w, float(xj), dv)
            s = fma(a, abs(float(xj)), s)
        dv = dv - rho
        res.append((dv, fma(K, s + abs(rho), F)))
    return res


def linear_definition(spec, x):
    """per pair the fp64 kernel's decision value: fma chains for dot(x, sv_s) and for each class's sum, then
    (sum_i + sum_j) - rho"""
    sv = np.asarray(spec["sv"], np.float64)
    kv = []
    for s in range(sv.shape[0]):
        k = 0.0
        for j in range(sv.shape[1]):
            k = fma(float(x[j]), float(sv[s, j]), k)
        kv.append(k)
    nsup = np.asarray(spec["n_support"], np.int64)
    start = np.concatenate([[0], np.cumsum(nsup)])
    dual = np.asarray(spec["dual_coef"], np.float64)
    rho = -np.asarray(spec["intercept"], np.float64)
    C = len(nsup)
    out, p = [], 0
    for i in range(C):
        for j in range(i + 1, C):
            acc_i, acc_j = 0.0, 0.0
            for s in range(start[i], start[i + 1]):
                acc_i = fma(float(dual[j - 1, s]), kv[s], acc_i)
            for s in range(start[j], start[j + 1]):
                acc_j = fma(float(dual[i, s]), kv[s], acc_j)
            out.append((acc_i + acc_j) - float(rho[p]))
            p += 1
    return out


# ---------------------------------------------------------------- fitted models shared by the CPU and GPU tests
# (kernel, SVC keyword arguments): poly degrees 0-4, coef0 < 0 and gamma in {'scale', 'auto', 0.0}
FITS = [
    ("linear", dict()),
    ("poly", dict(degree=0)),
    ("poly", dict(degree=1, coef0=-0.5, gamma="auto")),
    ("poly", dict(degree=2, coef0=-0.5)),
    ("poly", dict(degree=3, coef0=1.0, gamma=0.0)),
    ("poly", dict(degree=4, coef0=-0.25, gamma="auto")),
    ("sigmoid", dict(coef0=-0.5)),
]


def flows(n, seed, d=12):
    """standardised synthetic flow rows (linear and poly fits on raw rates can run for minutes); d > 12 appends the
    products of the first feature pairs, so that wider models exist too"""
    from traffic_classifier_sdn_b200 import synth
    X, y = synth.make_flows(n, seed=seed)
    X = np.log1p(np.abs(X))
    X = (X - X.mean(0)) / (X.std(0) + 1e-12)
    if d > 12:
        X = np.hstack([X, X[:, :d - 12] * X[:, 1:d - 11]])
    return np.ascontiguousarray(X), y


def fit(kernel, kw, n=600, seed=5, d=12, n_classes=6):
    """a fitted sklearn SVC (decision_function_shape='ovo', capped max_iter: parity needs no converged model)"""
    from sklearn.svm import SVC
    X, y = flows(n, seed, d)
    keep = y < n_classes
    return SVC(kernel=kernel, decision_function_shape="ovo", max_iter=20000, **kw).fit(X[keep], y[keep])
