"""CPU: SVC(probability=True).  The CPU definition (tests/svc_proba_oracle.py) against scikit-learn's predict_proba on fitted
models of every kernel and on the golden rows (tests/golden/svc_proba.npz), the Platt parameters' import and round trips,
the availability rules of predict_proba / predict_log_proba (scikit-learn's available_if(_check_proba)), and the C ABI's
argument refusals that come before any device work."""
import ctypes as C
import functools
import pickle
import warnings

import numpy as np
import pytest

import svc_kernel_oracle as so
import svc_proba_oracle as po
from traffic_classifier_sdn_b200 import _lib, estimators, modelio

pytestmark = pytest.mark.filterwarnings("ignore::FutureWarning")   # scikit-learn 1.9 deprecates probability=True

KERNELS = ("linear", "poly", "rbf", "sigmoid")


@functools.lru_cache(maxsize=None)
def _fit(kernel, n_classes):
    return po.fit(kernel, n_classes, n=max(600, 80 * n_classes))


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("n_classes", [2, 3, 6, 9])
def test_definition_matches_sklearn(n_classes, kernel):
    sk = _fit(kernel, n_classes)
    X, _ = so.flows(3000, seed=11)
    dec = po.libsvm_dec(sk.decision_function(X), n_classes)
    p, rounds, margin = po.proba(dec, sk.probA_, sk.probB_)
    ref = sk.predict_proba(X)
    err = float(np.abs(p - ref).max())
    assert err <= 1e-15, err
    assert rounds.max() < 100 and np.all(np.abs(p.sum(axis=1) - 1) <= 1e-12)
    print(f"C={n_classes} {kernel}: max |p - sk| {err:.1e}, rows bit-identical {np.mean(np.all(p == ref, axis=1)):.3f}, "
          f"rounds {rounds.min()}-{rounds.max()}, smallest stopping margin {margin.min():.1e}")


def test_definition_matches_golden_rows():
    spec, dec, ref, version = po.load_fixture()
    assert version == "1.9.0" and dec.shape == (7653, 10) and ref.shape == (7653, 5)
    p, rounds, margin = po.proba(dec, spec["prob_a"], spec["prob_b"])
    assert float(np.abs(p - ref).max()) <= 1e-15
    assert margin.min() > 1e-9


def test_spec_carries_platt_parameters():
    sk = _fit("rbf", 3)
    spec = modelio.spec_from_estimator(sk)
    assert np.array_equal(spec["prob_a"], sk._probA) and np.array_equal(spec["prob_b"], sk._probB)
    assert spec["prob_a"].dtype == np.float64 and spec["prob_a"].shape == (3,)
    back = modelio.spec_from_pickle_bytes(pickle.dumps(sk))
    assert set(back) == set(spec)
    for k in ("prob_a", "prob_b", "sv", "dual_coef", "intercept"):
        assert np.array_equal(back[k], spec[k]), k
    with warnings.catch_warnings():
        warnings.simplefilter("error", FutureWarning)        # the import reads the private names: no deprecation warning
        modelio.spec_from_estimator(sk)


def test_probability_false_imports_as_before(specs):
    """empty Platt arrays (probability=False; the reference's SVC pickle) add no key: the spec is the one without them"""
    from sklearn.svm import SVC
    X, y = so.flows(300, seed=2)
    sk = SVC().fit(X, y)
    assert sk._probA.size == 0
    spec = modelio.spec_from_estimator(sk)
    assert "prob_a" not in spec and "prob_b" not in spec
    assert "prob_a" not in modelio.spec_from_pickle_bytes(pickle.dumps(sk))
    assert "prob_a" not in specs["svc"]


@pytest.mark.parametrize("a,b", [
    (np.zeros(2), np.zeros(3)), (np.zeros(3), np.zeros(0)), (np.zeros(4), np.zeros(4)),
    (np.array([0.0, np.nan, 1.0]), np.zeros(3)), (np.zeros(3), np.array([np.inf, 0.0, 0.0])),
], ids=["short-a", "empty-b", "long", "nan", "inf"])
def test_malformed_platt_parameters_raise(a, b):
    sk = _fit("rbf", 3)
    with pytest.raises(modelio.SpecError):
        modelio.svc_platt(a, b, 3)
    bad = pickle.loads(pickle.dumps(sk))
    bad._probA, bad._probB = a, b
    with pytest.raises(modelio.SpecError):
        modelio.spec_from_pickle_bytes(pickle.dumps(bad))


class _FakeLib:
    """stands in for libtcsdn.so: records which create call each handle came from"""

    def __init__(self):
        self.created = []

    def tcsdn_svc_create(self, *args):
        self.created.append("create")
        return _lib.OK

    def tcsdn_svc_create_kernel(self, *args):
        self.created.append("kernel")
        return _lib.OK

    def tcsdn_svc_create_proba(self, *args):
        self.created.append("proba")
        return _lib.OK

    def tcsdn_model_score_cols(self, h):
        return 3

    def tcsdn_destroy(self, h):
        pass


@pytest.fixture
def fake_lib(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    return fake


def test_from_spec_pickle_and_availability(fake_lib):
    sk = _fit("rbf", 3)
    spec = modelio.spec_from_estimator(sk)
    est = estimators.from_spec(spec)
    assert fake_lib.created == ["proba"]
    assert est.get_params()["probability"] is True and hasattr(est, "predict_proba") and hasattr(est, "predict_log_proba")
    assert np.array_equal(est.probA_, sk.probA_) and np.array_equal(est.probB_, sk.probB_)
    with pytest.raises(ValueError):
        est.probA_[0] = 1.0                                 # read-only, as in scikit-learn
    back = pickle.loads(pickle.dumps(est))
    assert fake_lib.created[-1] == "proba" and np.array_equal(back.probB_, sk.probB_)
    plain = {k: v for k, v in spec.items() if k not in ("prob_a", "prob_b")}
    est = estimators.from_spec(plain)
    assert fake_lib.created[-1] == "create" and "probability" not in est.get_params()
    assert not hasattr(est, "predict_proba") and not hasattr(est, "predict_log_proba")
    assert est.probA_.size == 0
    with pytest.raises(AttributeError, match="predict_proba is not available when probability=False"):
        est.predict_proba
    est.set_params(probability=True)                       # asked for, but the model has no Platt parameters
    assert hasattr(est, "predict_proba")
    with pytest.raises(estimators.NotFittedError, match="fitted with probability=False"):
        est.predict_proba(np.zeros((1, 12)))
    with pytest.raises(estimators.NotFittedError, match="fitted with probability=False"):
        est.predict_log_proba(np.zeros((1, 12)))
    poly = estimators.from_spec(modelio.spec_from_estimator(_fit("poly", 3)))
    assert fake_lib.created[-1] == "proba" and poly.kernel == "poly"


def test_unfitted_availability():
    assert not hasattr(estimators.SVC(), "predict_proba")
    est = estimators.SVC(probability=True)
    assert hasattr(est, "predict_proba")
    with pytest.raises(estimators.NotFittedError, match="not fitted yet"):
        est.predict_proba(np.zeros((1, 12)))


def test_abi_argument_refusals():
    """the Platt arguments are checked before any device work, so these answers come on any machine"""
    lib = _lib.load()
    sv = np.zeros((2, 3))
    dual = np.ones((2, 2))
    icpt = np.zeros(3)
    nsup = np.array([1, 1, 0], np.int32)
    good, nan = np.zeros(3), np.array([0.0, np.nan, 0.0])
    f = _lib._f64p
    h = C.c_void_p()
    base = (sv.ctypes.data_as(f), dual.ctypes.data_as(f), icpt.ctypes.data_as(f), nsup.ctypes.data_as(_lib._i32p), 2, 3, 3,
            _lib.SVC_RBF, 0.5, 0.0, 3)
    for a, b, what in ((good, None, "both"), (None, good, "both"), (nan, good, "non-finite"), (good, nan, "non-finite")):
        pa = None if a is None else a.ctypes.data_as(f)
        pb = None if b is None else b.ctypes.data_as(f)
        assert lib.tcsdn_svc_create_proba(*base, pa, pb, C.byref(h)) == _lib.EINVAL
        assert what in _lib.last_error() and h.value is None
    bad_c = base[:6] + (17,) + base[7:]
    assert lib.tcsdn_svc_create_proba(*bad_c, good.ctypes.data_as(f), good.ctypes.data_as(f), C.byref(h)) == _lib.EINVAL
    assert lib.tcsdn_svc_predict_proba(None, None, 0, 3, _lib.F64, _lib.HOST, None, None) == _lib.EINVAL
