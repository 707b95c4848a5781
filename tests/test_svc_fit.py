"""SVC.fit's definition (tests/svc_fit_oracle.py, tests/svc_fit_oracle.c) against scikit-learn 1.9.0: np.array_equal on
every fitted array of the GPU fit's contract, over the parameter cases the GPU tests run.  Also the premises the GPU fit
rests on (scipy's ddot is an FMA chain for d <= 15; numpy's X.var() order), the parameter refusals and the ABI argument
errors.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import _lib, synth
from traffic_classifier_sdn_b200.estimators import svc_fit_plan
from svc_fit_oracle import contract_diff, fit, fma_chain_dot, pairwise_var, sklearn_fit


def notebook_split(g):
    """The reference notebook's split of the bundled rows."""
    from sklearn.model_selection import train_test_split
    return train_test_split(g["X"], g["y"], test_size=0.5, random_state=101)


def flows(n, n_classes, seed=3):
    """Synthetic flows with `n_classes` classes (string labels), scaled to [0, 1] per feature so that every kernel
    converges in a few hundred iterations.  The unscaled cases below (integer labels) are the ones that run long enough
    to shrink."""
    X, y = synth.make_flows(n, seed=seed)
    X = (X - X.min(0)) / np.maximum(X.max(0) - X.min(0), 1e-300)
    keep = y < n_classes
    return np.ascontiguousarray(X[keep]), np.array(["ping", "dns", "voice", "game", "telnet", "quake"])[y[keep]]


def with_duplicates(n=1500, seed=4):
    X, y = flows(n, 3, seed)
    return np.vstack([X, X[:300]]), np.concatenate([y, y[:300]])


# (name, data maker, parameters); every case's iteration counts are known from this file before the GPU runs it
CASES = [
    ("rbf-6", lambda: flows(3000, 6), dict()),
    ("rbf-2", lambda: flows(3000, 2), dict()),
    ("rbf-3-C0.5", lambda: flows(3000, 3), dict(C=0.5)),
    ("rbf-C10-auto", lambda: flows(3000, 6), dict(C=10, gamma="auto")),
    ("rbf-gamma-float", lambda: flows(3000, 6), dict(gamma=2.5)),
    ("linear", lambda: flows(2000, 3), dict(kernel="linear")),
    ("poly-0", lambda: flows(2000, 3), dict(kernel="poly", degree=0)),
    ("poly-2", lambda: flows(2000, 3), dict(kernel="poly", degree=2, coef0=1.0)),
    ("poly-3", lambda: flows(2000, 3), dict(kernel="poly", degree=3, gamma="auto", coef0=0.5)),
    ("balanced", lambda: synth.make_flows(3000, seed=3), dict(class_weight="balanced")),
    ("dict-weight", lambda: flows(3000, 3), dict(class_weight={"ping": 2.0}, C=5)),
    ("no-shrinking", lambda: flows(3000, 6), dict(shrinking=False, C=10)),
    ("tol-0.1", lambda: flows(3000, 6), dict(tol=1e-1)),
    ("tol-1e-5", lambda: synth.make_flows(3000, seed=3), dict(tol=1e-5)),
    ("max-iter", lambda: flows(3000, 6), dict(max_iter=200)),
    ("max-iter-shrunk", lambda: synth.make_flows(4000, seed=5), dict(C=10, gamma="auto", max_iter=2000)),
    ("float32", lambda: tuple(a.astype(np.float32) if a.dtype == np.float64 else a for a in flows(3000, 6)), dict(C=10)),
    ("duplicates", with_duplicates, dict(C=10)),
    ("unscaled-C10", lambda: synth.make_flows(4000, seed=5), dict(C=10, gamma="auto")),
]
CASE_IDS = [c[0] for c in CASES]


def case_data(name):
    return next(c for c in CASES if c[0] == name)


@pytest.mark.parametrize("d", range(1, 16))
def test_premise_ddot_is_an_fma_chain(d):
    from scipy.linalg.blas import ddot
    rng = np.random.default_rng(d)
    for _ in range(200):
        mag = 10.0 ** rng.uniform(-3, 6, size=(2, d))
        a, b = rng.normal(size=(2, d)) * mag
        assert ddot(a, b) == fma_chain_dot(a, b), (a, b)


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 15, 16, 127, 128, 129, 130, 255, 256, 257, 1000, 1001, 4097, 12345, 65536,
                               99991, 1000003])
def test_premise_pairwise_variance_is_numpys(n):
    rng = np.random.default_rng(n)
    a = rng.normal(size=n) * 10.0 ** rng.uniform(-3, 6, size=n) + 3.0
    assert pairwise_var(a) == a.var()
    X = a[: (n // 3) * 3].reshape(-1, 3) if n >= 3 else a.reshape(-1, 1)
    assert pairwise_var(X) == X.var()


def test_definition_is_sklearn_on_the_notebook_split(golden):
    Xtr, _, ytr, _ = notebook_split(golden)
    mine = fit(Xtr, ytr)
    assert contract_diff(mine, sklearn_fit(Xtr, ytr)[0]) == []
    assert max(mine["n_iter_"]) == 591


@pytest.mark.parametrize("name", CASE_IDS)
def test_definition_is_sklearn(name):
    _, make, p = case_data(name)
    X, y = make()
    mine = fit(X, y, **p)
    assert contract_diff(mine, sklearn_fit(X, y, **p)[0]) == []
    ev = {k: sum(e[k] for e in mine["events"]) for k in mine["events"][0]}
    assert ev["recon_mismatch"] == 0            # both reconstruct_gradient branches give the same bits
    assert ev["fragile"] == 0, f"{name}: {ev['fragile']} Q entries within an ulp of a float32 rounding boundary"
    if name.startswith("max-iter"):
        assert mine["fit_status_"] == 1
    if name == "max-iter-shrunk":   # max_iter stops a pair while shrunk: rho over the active set, a permuted scatter back
        assert ev["stopped_shrunk"] > 0


def test_cases_cover_shrinking_unshrink_and_both_reconstructions():
    tot = {}
    for name in ("rbf-C10-auto", "tol-1e-5", "balanced", "unscaled-C10"):
        _, make, p = case_data(name)
        X, y = make()
        for e in fit(X, y, **p)["events"]:
            for k, v in e.items():
                tot[k] = tot.get(k, 0) + v
    assert tot["shrink"] > 0 and tot["unshrink"] > 0
    assert tot["recon_by_inactive"] > 0 and tot["recon_by_free"] > 0
    assert tot["recon_mismatch"] == 0


def test_plan_refusals_name_the_parameter():
    X, y = flows(200, 3)
    for p, word in [(dict(probability=True), "probability"), (dict(kernel="sigmoid"), "kernel"),
                    (dict(kernel="precomputed"), "kernel"), (dict(kernel=lambda a, b: a @ b.T), "kernel"),
                    (dict(C=0.0), "C"), (dict(tol=-1.0), "tol"), (dict(max_iter=-2), "max_iter"),
                    (dict(gamma=-1.0), "gamma"), (dict(degree=-1), "degree"), (dict(nu=0.5), "nu")]:
        with pytest.raises(ValueError, match=word):
            svc_fit_plan(p, X, y)
    with pytest.raises(ValueError, match="16 features"):
        svc_fit_plan({}, np.zeros((10, 16)), np.arange(10) % 2)
    Xn = X.copy()
    Xn[3, 2] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        svc_fit_plan({}, Xn, y)
    Xn[3, 2] = np.inf
    with pytest.raises(ValueError, match="infinity"):
        svc_fit_plan({}, Xn, y)
    with pytest.raises(ValueError, match="inconsistent numbers of samples"):
        svc_fit_plan({}, X, y[:-1])
    with pytest.raises(ValueError, match="The number of classes has to be greater than one; got 1 class"):
        svc_fit_plan({}, X, np.zeros(len(X)))
    # the estimator refuses the same way, before any device work
    with pytest.raises(ValueError, match="probability"):
        tc.SVC(probability=True).fit(X, y, backend="gpu")


def test_plan_gamma_and_weights_are_sklearns():
    X, y = flows(500, 3)
    for p in (dict(), dict(gamma="auto"), dict(gamma=0.7), dict(class_weight="balanced", C=3.0),
              dict(class_weight={"ping": 2.0})):
        plan = svc_fit_plan(p, X, y)
        sk = sklearn_fit(X, y, **p)[1]
        assert plan["_gamma"] == sk._gamma
        assert np.array_equal(plan["class_weight_"], sk.class_weight_)
        assert np.array_equal(plan["classes_"], sk.classes_)


def _abi_fit(x, y, n, d, ncls, cw, kernel=_lib.SVC_RBF, gamma=0.5, tol=1e-3, degree=3, max_iter=-1, loc=_lib.HOST):
    lib = _lib.load()
    h = C.c_void_p()
    rc = lib.tcsdn_svc_fit(x, y, n, d, ncls, _lib.F64, loc, kernel, gamma, 0.0, degree, cw, tol, 1, max_iter, C.byref(h),
                           None)
    return rc, h


def test_abi_argument_errors():
    X = np.ascontiguousarray(np.random.default_rng(0).normal(size=(20, 4)))
    y = np.ascontiguousarray(np.arange(20) % 2, np.int32)
    cw = np.ones(2)
    xp, yp, cp = _lib.ptr(X), _lib.ptr(y, _lib._i32p), _lib.ptr(cw, _lib._f64p)
    for args in [dict(d=16), dict(d=0), dict(n=1), dict(ncls=1), dict(kernel=_lib.SVC_SIGMOID), dict(gamma=-1.0),
                 dict(gamma=float("nan")), dict(tol=0.0), dict(degree=-1), dict(max_iter=-2), dict(loc=7)]:
        a = dict(x=xp, y=yp, n=20, d=4, ncls=2, cw=cp)
        a.update(args)
        rc, h = _abi_fit(**a)
        assert rc == _lib.EINVAL and not h.value, args
    bad = np.array([1.0, 0.0])
    assert _abi_fit(xp, yp, 20, 4, 2, _lib.ptr(bad, _lib._f64p))[0] == _lib.EINVAL
    y3 = y.copy()
    y3[0] = 5
    assert _abi_fit(xp, _lib.ptr(y3, _lib._i32p), 20, 4, 2, cp)[0] == _lib.EINVAL
    y1 = np.zeros(20, np.int32)
    assert _abi_fit(xp, _lib.ptr(y1, _lib._i32p), 20, 4, 2, cp)[0] == _lib.EINVAL   # class 1 has no rows
    assert _abi_fit(None, yp, 20, 4, 2, cp)[0] == _lib.EINVAL
    lib = _lib.load()
    assert lib.tcsdn_svc_fit_sizes(None, None, None, None, None) == _lib.EINVAL
    assert lib.tcsdn_svc_fit_read(None, None, None, None, None) == _lib.EINVAL
    lib.tcsdn_svc_fit_free(None)
    v = C.c_double()
    assert lib.tcsdn_row_var(xp, 0, 4, _lib.F64, _lib.HOST, C.byref(v), None) == _lib.EINVAL
    assert lib.tcsdn_row_var(xp, 20, 4, _lib.F64, _lib.HOST, None, None) == _lib.EINVAL
