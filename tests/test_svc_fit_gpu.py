"""SVC.fit(X, y, backend="gpu") (csrc/svc_fit.cu) against scikit-learn 1.9.0 and the CPU definition
(tests/svc_fit_oracle.py): np.array_equal on every fitted array of the contract, on the cases of tests/test_svc_fit.py
(whose iteration counts that file establishes without a GPU), plus held-out predictions, device rows, numpy's X.var() on
the device and the error paths.  The solver's hard iteration limit (max(10^7, 100 l) iterations, an error) is not
reached by any test: that takes at least ten million iterations."""
import warnings

import numpy as np
import pytest

import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import synth
from svc_fit_oracle import CONTRACT, contract_diff, fit, fma_chain_dot, sklearn_fit
from test_svc_fit import CASE_IDS, case_data, notebook_split

pytestmark = pytest.mark.gpu


def _gpu(est):
    return {k: getattr(est, k) for k in CONTRACT}


def held_out(X, n=600, seed=7):
    """Rows that were not trained on: uniform within each training column's range, in X's dtype."""
    rng = np.random.default_rng(seed)
    lo, hi = X.min(0).astype(np.float64), X.max(0).astype(np.float64)
    return np.ascontiguousarray(lo + rng.random((n, X.shape[1])) * (hi - lo), dtype=X.dtype)


def test_premise_ddot_is_an_fma_chain_here():
    """Repeated on the machine that runs the GPU fit: its OpenBLAS may pick another ddot kernel, and a failure here is a
    premise failure, not a solver bug."""
    from scipy.linalg.blas import ddot
    rng = np.random.default_rng(1)
    for d in range(1, 16):
        for _ in range(100):
            a, b = rng.normal(size=(2, d)) * 10.0 ** rng.uniform(-3, 6, size=(2, d))
            assert ddot(a, b) == fma_chain_dot(a, b), f"premise: scipy's ddot is not an FMA chain at d={d}"


@pytest.mark.parametrize("name", CASE_IDS)
def test_gpu_fit_is_sklearns_and_the_definitions(name):
    _, make, p = case_data(name)
    X, y = make()
    sk, sk_est = sklearn_fit(X, y, **p)
    mine = fit(X, y, **p)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est = tc.SVC(**p).fit(X, y, backend="gpu")
    g = _gpu(est)
    fragile = sum(e["fragile"] for e in mine["events"])
    print(f"{name}: {len(X)} rows, most iterations {max(sk['n_iter_'])}, fragile Q entries {fragile}")
    assert contract_diff(g, sk) == [], f"{name} differs from scikit-learn (fragile Q entries: {fragile})"
    assert contract_diff(g, mine) == []
    assert est.shape_fit_ == sk_est.shape_fit_ and est.n_features_in_ == sk_est.n_features_in_
    Xt = held_out(X)
    assert np.array_equal(est.predict(Xt), sk_est.predict(Xt))
    ref = tc.from_sklearn(sk_est)
    assert np.array_equal(est.decision_function(Xt), ref.decision_function(Xt))
    assert np.array_equal(est.predict(Xt), ref.predict(Xt))


def test_gpu_max_iter_warns_like_sklearn():
    _, make, p = case_data("max-iter")
    X, y = make()
    from sklearn.exceptions import ConvergenceWarning
    with pytest.warns(ConvergenceWarning, match="max_iter=200"):
        est = tc.SVC(**p).fit(X, y, backend="gpu")
    assert est.fit_status_ == 1


def test_gpu_notebook_recipe(golden):
    Xtr, Xte, ytr, yte = notebook_split(golden)
    sk, sk_est = sklearn_fit(Xtr, ytr)
    est = tc.SVC().fit(Xtr, ytr, backend="gpu")
    assert contract_diff(_gpu(est), sk) == []
    assert contract_diff(_gpu(est), fit(Xtr, ytr)) == []
    assert np.array_equal(est.predict(Xte), sk_est.predict(Xte))
    assert np.array_equal(est.predict(golden["X"]), sk_est.predict(golden["X"]))
    ref = tc.from_sklearn(sk_est)
    assert np.array_equal(est.decision_function(Xte), ref.decision_function(Xte))
    again = tc.SVC().fit(Xtr, ytr, backend="gpu")   # repeatable
    assert contract_diff(_gpu(again), _gpu(est)) == []


def test_gpu_device_rows_stay_on_the_device():
    import torch
    _, make, p = case_data("rbf-6")
    X, y = make()
    ycodes, yi = np.unique(y, return_inverse=True)

    class NoHostCopy(torch.Tensor):
        __module__ = "torch"   # a CUDA torch tensor to the estimator, whose host copies fail

        def cpu(self, *a, **k):
            raise AssertionError("device rows were copied to the host")

        def numpy(self, *a, **k):
            raise AssertionError("device rows were copied to the host")

    for dt in (np.float32, np.float64):
        Xd = np.ascontiguousarray(X.astype(dt))
        sk = sklearn_fit(Xd, yi)[0]
        t = torch.from_numpy(Xd).cuda().as_subclass(NoHostCopy)
        est = tc.SVC(gamma="scale").fit(t, torch.from_numpy(yi).cuda(), backend="gpu")
        assert contract_diff(_gpu(est), sk) == [], dt


def test_gpu_50k_rows_six_classes():
    X, y = synth.make_flows(50000, seed=3)
    sk, _ = sklearn_fit(X, y)
    est = tc.SVC().fit(X, y, backend="gpu")
    assert contract_diff(_gpu(est), sk) == []
    assert contract_diff(_gpu(est), fit(X, y)) == []
    print(f"50k: most iterations {max(sk['n_iter_'])}, {len(sk['support_'])} support vectors")


def test_gpu_errors_and_auto_route():
    import torch
    X, y = synth.make_flows(500, seed=1)
    with pytest.raises(ValueError, match="kernel"):
        tc.SVC(kernel="sigmoid").fit(X, y, backend="gpu")
    with pytest.raises(ValueError, match="16 features"):
        tc.SVC().fit(np.zeros((10, 16)), np.arange(10) % 2, backend="gpu")
    Xn = torch.from_numpy(X).cuda()
    Xn[5, 3] = float("nan")
    with pytest.raises(ValueError, match="NaN"):
        tc.SVC().fit(Xn, y, backend="gpu")
    with pytest.raises(ValueError, match="NaN"):
        tc.SVC(gamma=0.1).fit(Xn, y, backend="gpu")
    est = tc.SVC().fit(X, y)   # backend="auto" still trains with scikit-learn
    assert not hasattr(est, "support_")
    sk = sklearn_fit(X, y)[1]
    assert np.array_equal(est.predict(X), sk.predict(X))


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 15, 16, 127, 128, 129, 130, 255, 256, 257, 1000, 1001, 4097, 12345, 65536,
                               99991, 1000003])
def test_gpu_row_var_is_numpys(n):
    """tcsdn_row_var (gamma='scale' on device rows) equals np.var bit for bit, host and device rows, float32 and float64."""
    import ctypes as C
    import torch
    from traffic_classifier_sdn_b200 import _lib
    rng = np.random.default_rng(n)
    a = rng.normal(size=n) * 10.0 ** rng.uniform(-3, 6, size=n) + 3.0
    lib = _lib.load()
    for X in (a.reshape(-1, 1), a[: (n // 3) * 3].reshape(-1, 3) if n >= 3 else a.reshape(1, -1)):
        for dt, code in ((np.float64, _lib.F64), (np.float32, _lib.F32)):
            Xd = np.ascontiguousarray(X, dtype=dt)
            want = Xd.astype(np.float64).var()
            v = C.c_double()
            _lib.check(lib.tcsdn_row_var(_lib.ptr(Xd), Xd.shape[0], Xd.shape[1], code, _lib.HOST, C.byref(v), None))
            assert v.value == want, (n, dt, "host")
            t = torch.from_numpy(Xd).cuda()
            _lib.check(lib.tcsdn_row_var(C.c_void_p(t.data_ptr()), Xd.shape[0], Xd.shape[1], code, _lib.DEVICE, C.byref(v),
                                         torch.cuda.current_stream().cuda_stream))
            assert v.value == want, (n, dt, "device")
