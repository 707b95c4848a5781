"""CPU: SVC(kernel='linear' | 'poly' | 'sigmoid') import, the CPU definition against scikit-learn, and the linear collapsed
path's error bound checked exactly (fractions.Fraction) against the fp64 definition on random and decision-boundary rows."""
import io
import os
import pickle
import types

import numpy as np
import pytest

import svc_kernel_oracle as so
from traffic_classifier_sdn_b200 import modelio

# |dec - sklearn| <= DEC_REL * (sum_s |c_ps K_s| + |rho_p|): libsvm's dot is BLAS ddot (unspecified order), this definition
# sums in feature order; both are fp64, so they differ by a few ulps of the terms
DEC_REL = 1e-12


@pytest.fixture(scope="module", params=range(len(so.FITS)), ids=[f"{k}-{kw}" for k, kw in so.FITS])
def fitted(request):
    k, kw = so.FITS[request.param]
    return so.fit(k, kw)


def test_spec_roundtrip_estimator_and_pickle(fitted, tmp_path):
    spec = modelio.spec_from_estimator(fitted)
    assert spec["kernel"] == fitted.kernel and spec["degree"] == fitted.degree and spec["coef0"] == fitted.coef0
    assert spec["gamma"] == fitted._gamma
    path = os.path.join(tmp_path, "svc.pkl")
    with open(path, "wb") as fh:
        pickle.dump(fitted, fh)
    back = modelio.load_reference_pickle(path)
    assert set(back) == set(spec)
    for k, v in spec.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(back[k], v), k
        else:
            assert back[k] == v, k


def test_definition_matches_sklearn(fitted):
    spec = modelio.spec_from_estimator(fitted)
    X, _ = so.flows(3000, seed=11)
    lab, dec, scale = so.predict(spec, X)
    assert np.array_equal(fitted.classes_[lab], fitted.predict(X))
    sk = fitted.decision_function(X)
    sk = -sk[:, None] if sk.ndim == 1 else sk          # two classes: sklearn negates libsvm's value
    err = np.abs(dec - sk) / scale
    assert err.max() <= DEC_REL, err.max()


def test_spec_without_kernel_is_rbf():
    """a pickle written before SVC had other kernels carries no `kernel` attribute"""
    o = types.SimpleNamespace(support_vectors_=np.zeros((2, 3)), classes_=np.arange(2), dual_coef_=-np.ones((1, 2)),
                              _dual_coef_=np.ones((1, 2)), intercept_=np.zeros(1), _intercept_=np.zeros(1),
                              _n_support=np.array([1, 1]), _gamma=0.5, decision_function_shape="ovr")
    spec = modelio._spec_from_attrs("SVC", o)
    assert spec["kernel"] == "rbf"


@pytest.mark.parametrize("kernel", ["precomputed", "callable", "laplacian"])
def test_unsupported_kernels_raise(kernel):
    from sklearn.svm import SVC
    X, y = so.flows(80, seed=1)
    if kernel == "precomputed":
        est = SVC(kernel="precomputed").fit(X @ X.T, y)
    elif kernel == "callable":
        est = SVC(kernel=lambda a, b: a @ b.T).fit(X, y)
    else:
        est = types.SimpleNamespace(kernel="laplacian")
    with pytest.raises(modelio.SpecError):
        modelio._spec_from_attrs("SVC", est)
    if kernel == "precomputed":
        buf = io.BytesIO()
        pickle.dump(est, buf)
        with pytest.raises(modelio.SpecError):
            modelio.spec_from_pickle_bytes(buf.getvalue())


def _boundary_rows(spec, params, X, rng):
    """rows moved onto a pair's decision boundary: x - (dec / ||W||^2) W with W the pair's collapsed weights"""
    out = []
    for x in X:
        p = int(rng.integers(len(params)))
        W = np.asarray(params[p][0])
        dec = float(W @ x - params[p][2])
        out.append(x - (dec / float(W @ W)) * W)
    return np.asarray(out)


@pytest.mark.parametrize("n_classes,n", [(2, 200), (4, 300), (6, 400)])
def test_linear_certificate_bound_exact(n_classes, n):
    """|dec~ - dec_def| <= E on every pair, with dec~, E and dec_def the operations the kernels perform, compared exactly"""
    from fractions import Fraction
    est = so.fit("linear", {}, n=n, seed=n_classes, n_classes=n_classes)
    spec = modelio.spec_from_estimator(est)
    params = so.linear_params(spec)
    rng = np.random.default_rng(n_classes)
    X, _ = so.flows(12, seed=100 + n_classes)
    rows = np.vstack([X, _boundary_rows(spec, params, X, rng), 1e3 * X[:2]])
    uncertain = 0
    for x in rows:
        col = so.linear_collapsed(params, x)
        ref = so.linear_definition(spec, x)
        for (dv, E), r in zip(col, ref):
            assert abs(Fraction(dv) - Fraction(r)) <= Fraction(E), (dv, r, E)
            uncertain += abs(dv) <= E
    # the bound is not vacuous: random rows are certain, the boundary rows are not
    assert uncertain >= len(X) // 2
    col = [so.linear_collapsed(params, x) for x in X]
    assert sum(abs(dv) <= E for c in col for dv, E in c) == 0
