"""CPU definition of SVC.fit (scikit-learn 1.9.0, probability=False, kernel 'linear' / 'poly' / 'rbf', d <= 15), so that
the GPU fit (csrc/svc_fit.cu) has something exact to be compared with on a machine without a GPU.

The host half is the package's own `svc_fit_plan` (classes, class weights, per-class C, _gamma).  The solver of one class
pair is tests/svc_fit_oracle.c, a C restatement of libsvm's Solver::Solve, compiled here on first use (into a private
temporary directory, with -ffp-contract=off, against the same libm `exp` scikit-learn's libsvm calls).  This module restates the
one-vs-one bookkeeping of svm_train around it: svm_group_classes, the sub-problems, the nonzero flags, the support-vector
order, the dual_coef layout, intercept = -rho, and scikit-learn's sign flip for two classes.
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from traffic_classifier_sdn_b200.estimators import svc_fit_plan

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "svc_fit_oracle.c")
EVENTS = ("shrink", "unshrink", "recon", "recon_by_inactive", "recon_by_free", "recon_mismatch", "fragile",
          "stopped_shrunk")
KERNELS = {"linear": 0, "poly": 1, "rbf": 2}
_LIB = None
_LOCK = threading.Lock()
_f64p = C.POINTER(C.c_double)
_i64p = C.POINTER(C.c_int64)


def lib():
    with _LOCK:
        return _load()


def _load():
    """Compile tests/svc_fit_oracle.c into a fresh directory only this process can write (tempfile.mkdtemp, mode 0700),
    once per process, and load it from there.  The directory is removed once the library is loaded."""
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="tcsdn_svc_fit_oracle_")
        try:
            so = os.path.join(tmp, "svc_fit_oracle.so")
            cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
            subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fPIC", "-std=c11", "-shared", "-o", so, _SRC, "-lm"])
            L = C.CDLL(so)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        L.svc_fit_oracle_solve.restype = C.c_int
        L.svc_fit_oracle_solve.argtypes = [_f64p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double,
                                           C.c_double, C.c_int, C.c_double, C.c_int, C.c_int64, _f64p, _f64p, _i64p,
                                           C.POINTER(C.c_int), _i64p]
        L.svc_fit_oracle_var.restype = C.c_double
        L.svc_fit_oracle_var.argtypes = [_f64p, C.c_int64]
        _LIB = L
    return _LIB


def pairwise_var(a):
    """numpy's X.var() restated (tests/svc_fit_oracle.c svc_fit_oracle_var) over the flattened values."""
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    return lib().svc_fit_oracle_var(a.ctypes.data_as(_f64p), a.size)


def fma_chain_dot(a, b):
    """The feature-order FMA chain libsvm's dot is taken to be, in exact arithmetic per step (float64 pairs)."""
    from fractions import Fraction
    s = 0.0
    for u, v in zip(a, b):
        s = float(Fraction(u) * Fraction(v) + Fraction(s))
    return s


def _solve(X, rows, n_pos, Cp, Cn, plan):
    xs = np.ascontiguousarray(X[rows])
    l = len(rows)
    alpha = np.empty(l)
    rho, it, to = C.c_double(), C.c_int64(), C.c_int()
    ev = np.zeros(8, np.int64)
    rc = lib().svc_fit_oracle_solve(xs.ctypes.data_as(_f64p), l, xs.shape[1], n_pos, Cp, Cn, KERNELS[plan["kernel"]],
                                    float(plan["_gamma"]), plan["coef0"], plan["degree"], plan["tol"],
                                    int(plan["shrinking"]), plan["max_iter"], alpha.ctypes.data_as(_f64p), C.byref(rho),
                                    C.byref(it), C.byref(to), ev.ctypes.data_as(_i64p))
    if rc != 0:
        raise MemoryError("svc_fit_oracle_solve: out of memory")
    return alpha, rho.value, it.value, to.value, ev


def fit(X, y, threads=None, **params):
    """-> dict with scikit-learn's fitted arrays (``support_``, ``support_vectors_``, ``n_support_``, ``dual_coef_``,
    ``intercept_``, ``_dual_coef_``, ``_intercept_``, ``n_iter_``, ``fit_status_``, ``class_weight_``, ``_gamma``,
    ``classes_``) and ``events``: one dict per class pair of the counts named in EVENTS."""
    plan = svc_fit_plan(params, X, y)
    plan.pop("rows")
    X = np.ascontiguousarray(np.asarray(X, dtype=np.float64))
    yi = plan["y_index"]
    Cn = len(plan["classes_"])
    # svm_group_classes: the labels 0..C-1 sorted, each class's rows in original order
    perm = np.argsort(yi, kind="stable")
    count = np.bincount(yi, minlength=Cn)
    start = np.concatenate([[0], np.cumsum(count)[:-1]])
    pairs = [(i, j) for i in range(Cn) for j in range(i + 1, Cn)]
    cw = plan["class_C"]

    def one(ij):
        i, j = ij
        rows = np.concatenate([perm[start[i]:start[i] + count[i]], perm[start[j]:start[j] + count[j]]])
        return _solve(X, rows, int(count[i]), float(cw[i]), float(cw[j]), plan)

    with ThreadPoolExecutor(max_workers=threads or min(len(pairs), os.cpu_count() or 1)) as ex:
        res = list(ex.map(one, pairs))
    nonzero = np.zeros(len(X), bool)   # grouped order
    for (i, j), (a, *_rest) in zip(pairs, res):
        nonzero[start[i]:start[i] + count[i]] |= np.abs(a[:count[i]]) > 0
        nonzero[start[j]:start[j] + count[j]] |= np.abs(a[count[i]:]) > 0
    n_support = np.array([nonzero[start[c]:start[c] + count[c]].sum() for c in range(Cn)], np.int32)
    nz_start = np.concatenate([[0], np.cumsum(n_support)[:-1]])
    total = int(n_support.sum())
    support = perm[nonzero].astype(np.int32)
    dual = np.zeros((Cn - 1, total))
    for (i, j), (a, *_rest) in zip(pairs, res):
        ai, aj = a[:count[i]], a[count[i]:]
        dual[j - 1, nz_start[i]:nz_start[i] + n_support[i]] = ai[nonzero[start[i]:start[i] + count[i]]]
        dual[i, nz_start[j]:nz_start[j] + n_support[j]] = aj[nonzero[start[j]:start[j] + count[j]]]
    rho = np.array([r[1] for r in res])
    icpt = np.where(rho != 0, -rho, 0.0)
    out = dict(support_=support, support_vectors_=X[support], n_support_=n_support, _dual_coef_=dual, _intercept_=icpt,
               dual_coef_=-dual if Cn == 2 else dual, intercept_=-icpt if Cn == 2 else icpt,
               n_iter_=np.array([r[2] for r in res], np.intc), fit_status_=int(any(r[3] for r in res)),
               class_weight_=plan["class_weight_"], _gamma=plan["_gamma"], classes_=plan["classes_"])
    out["events"] = [dict(zip(EVENTS, (int(v) for v in r[4][:len(EVENTS)]))) for r in res]
    return out


CONTRACT = ("support_", "support_vectors_", "n_support_", "dual_coef_", "intercept_", "_dual_coef_", "_intercept_",
            "n_iter_", "fit_status_", "class_weight_", "_gamma", "classes_")


def sklearn_fit(X, y, **params):
    """scikit-learn's SVC(**params).fit(X, y) as a dict of the contract's attributes."""
    import warnings
    from sklearn.svm import SVC
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sk = SVC(**params).fit(X, y)
    return {k: getattr(sk, k if k != "n_support_" else "_n_support") for k in CONTRACT}, sk


def contract_diff(a, b):
    """-> names of the contract attributes whose values differ (np.array_equal)."""
    return [k for k in CONTRACT if not np.array_equal(np.asarray(a[k]), np.asarray(b[k]))]
