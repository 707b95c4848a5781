"""KNeighborsClassifier(metric='manhattan' | 'chebyshev'), CPU side: the definition (tests/knn_metric_oracle.py) pinned to
scikit-learn, the metric's spellings in the model import, the estimator's plumbing and the C entry point's argument checks.
None of these needs a GPU; tests/test_knn_metric_gpu.py checks the kernels against the definition."""
import ctypes as C
import pickle

import numpy as np
import pytest

import knn_metric_oracle as kmo
import knn_weighted_oracle as kwo
import kneighbors_oracle as kno
from traffic_classifier_sdn_b200 import _lib, estimators, modelio


def _sk(k, metric, algorithm, weights="uniform"):
    from sklearn.neighbors import KNeighborsClassifier
    return KNeighborsClassifier(n_neighbors=k, metric=metric, algorithm=algorithm, weights=weights)


def _lattice(seed=5, nt=700, nq=2000):
    """integer lattice rows (every rdist exact), queries on lattice points and half-way between them: dense ties"""
    rng = np.random.default_rng(seed)
    tr = np.floor(rng.random((nt, 4)) * 4)
    y = rng.integers(0, 5, nt).astype(np.int32)
    q = np.floor(rng.random((nq, 4)) * 4)
    q[nq // 2:] += 0.5
    return dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(5), n_features=4), q


# ------------------------------------------------------------------ the definition against scikit-learn
def test_sequential_sum_is_not_numpys_row_sum():
    """rule 1 spells out the loop: numpy's pairwise row sum differs in the last bit on some rows"""
    rng = np.random.default_rng(0)
    X = rng.random((2000, 12)) * 10.0 ** rng.integers(-3, 6, (2000, 12))
    t = rng.random((1, 12)) * 1e4
    assert not np.array_equal(kmo.rdist("manhattan", X, t)[:, 0], np.abs(X - t).sum(axis=1))


@pytest.mark.parametrize("metric", kmo.METRICS)
@pytest.mark.parametrize("k", [1, 5, 8, 9])
def test_definition_equals_sklearn_brute_on_a_lattice(metric, k):
    """brute force runs the same heap in index order: kneighbors indices and distances, labels and predict_proba with both
    weightings are bit-identical on every row (lattice queries tie densely)"""
    spec, q = _lattice()
    from threadpoolctl import threadpool_limits
    dist, ind = kmo.kneighbors(spec, q, k, metric)
    with threadpool_limits(limits=1):
        sk = _sk(k, metric, "brute").fit(spec["fit_X"], spec["y"])
        sd, si = kno.canonical(*sk.kneighbors(q))
        lab_u, proba_u = sk.predict(q), sk.predict_proba(q)
        skw = _sk(k, metric, "brute", "distance").fit(spec["fit_X"], spec["y"])
        lab_w, proba_w = skw.predict(q), skw.predict_proba(q)
    assert np.array_equal(ind, si) and np.array_equal(dist, sd)
    d1, _ = kmo.kneighbors(spec, q, k + 1, metric)
    assert (d1[:, k] == d1[:, k - 1]).mean() > 0.3            # ties at the k-th distance are common
    lab, proba = kmo.predict(spec, q, k, metric)
    assert np.array_equal(lab, lab_u) and np.array_equal(proba, proba_u)
    lab, proba = kmo.predict(dict(spec, weights="distance"), q, k, metric)
    assert np.array_equal(lab, lab_w) and np.array_equal(proba, proba_w)


@pytest.mark.parametrize("metric", kmo.METRICS)
def test_definition_equals_sklearn_kd_tree_on_bundled_rows(golden, specs, metric):
    """the reference model's fit_X / y (12 features) with the metric, every bundled row: sorted distances bit-identical,
    indices equal wherever the (k+1)-th distance differs from the k-th, labels equal on rows without cross-class ties"""
    spec, X = specs["knn"], np.ascontiguousarray(golden["X"])
    k = int(spec["k"])
    dist, ind = kmo.kneighbors(spec, X, k + 1, metric)
    sk = _sk(k, metric, "kd_tree").fit(spec["fit_X"], spec["y"])
    sd, si = kno.canonical(*sk.kneighbors(X))
    assert np.array_equal(dist[:, :k], sd)
    clear = dist[:, k] != dist[:, k - 1]
    assert clear.sum() > 0.5 * len(X)
    assert np.array_equal(ind[clear, :k], si[clear])
    lab, _ = kmo.predict(spec, X, k, metric)
    ok = ~kmo.cross_class_ties(spec, X, k + 1, metric)
    assert ok.sum() > 0.5 * len(X)
    assert np.array_equal(lab[ok], sk.predict(X)[ok])


def test_distance_vote_reuses_the_weighted_definition():
    spec, q = _lattice()
    dist, ind = kmo.kneighbors(spec, q, 5, "manhattan")
    lab, proba = kmo.predict(dict(spec, weights="distance"), q, 5, "manhattan")
    l2, p2 = kwo.vote(kwo.weights(dist), np.asarray(spec["y"], np.int64)[ind], 5)
    assert np.array_equal(lab, l2) and np.array_equal(proba, p2)


# ------------------------------------------------------------------ model import
@pytest.mark.parametrize("metric,p,params,want", [
    ("manhattan", 2, None, "manhattan"), ("cityblock", 2, None, "manhattan"), ("l1", 2, None, "manhattan"),
    ("minkowski", 1, None, "manhattan"), ("minkowski", 2, {"p": 1}, "manhattan"),
    ("chebyshev", 2, None, "chebyshev"), ("infinity", 2, None, "chebyshev"), ("minkowski", np.inf, None, "chebyshev"),
    ("euclidean", 2, None, "euclidean"), ("l2", 2, None, "euclidean"), ("minkowski", 2, None, "euclidean"),
    ("minkowski", 3, {"p": 2}, "euclidean"),
])
def test_metric_spellings(metric, p, params, want):
    assert modelio.knn_metric(metric, p, params) == want


@pytest.mark.parametrize("metric,p,params", [
    ("minkowski", 3, None), ("minkowski", 1.5, None), ("minkowski", 2, {"p": 4}), ("minkowski", 1, {"w": np.ones(3)}),
    ("seuclidean", 2, {"V": np.ones(3)}), ("cosine", 2, None), ("haversine", 2, None), (lambda a, b: 0.0, 2, None),
    ("manhattan", 2, {"foo": 1}),
])
def test_refused_metrics_name_the_supported_ones(metric, p, params):
    with pytest.raises(modelio.SpecError, match="'euclidean', 'manhattan' and 'chebyshev'"):
        modelio.knn_metric(metric, p, params)


def test_spec_reads_the_fitted_metric():
    from sklearn.neighbors import KNeighborsClassifier
    rng = np.random.default_rng(1)
    X, y = rng.random((60, 3)), rng.integers(0, 3, 60)
    for kw, want in [(dict(metric="l1"), "manhattan"), (dict(p=1), "manhattan"), (dict(metric="infinity"), "chebyshev"),
                     (dict(p=np.inf), "chebyshev"), (dict(), "euclidean"), (dict(metric_params={"p": 1}), "manhattan")]:
        assert modelio.spec_from_estimator(KNeighborsClassifier(3, **kw).fit(X, y))["metric"] == want, kw
        spec = modelio.spec_from_pickle_bytes(pickle.dumps(KNeighborsClassifier(3, **kw).fit(X, y)))
        assert spec["metric"] == want and np.array_equal(spec["fit_X"], X)
    for kw in [dict(p=3), dict(metric="cosine"), dict(metric="minkowski", metric_params={"w": np.ones(3)})]:
        with pytest.raises(modelio.SpecError, match="supported metrics"):
            modelio.spec_from_estimator(KNeighborsClassifier(3, **kw).fit(X, y))


def test_golden_spec_without_the_key_is_euclidean(specs):
    assert "metric" not in specs["knn"]
    assert modelio.knn_metric(specs["knn"].get("metric", "euclidean")) == "euclidean"


# ------------------------------------------------------------------ the estimator's plumbing
class _FakeLib:
    """stands in for libtcsdn.so: records which create call each handle came from"""

    def __init__(self):
        self.created, self.destroyed = [], 0

    def tcsdn_knn_create_weighted(self, fx, y, n, d, n_classes, k, weights, out):
        self.created.append(("weighted", weights))
        return _lib.OK

    def tcsdn_knn_create_metric(self, fx, y, n, d, n_classes, k, weights, metric, out):
        self.created.append(("metric", weights, metric))
        return _lib.OK

    def tcsdn_model_score_cols(self, h):
        return 3

    def tcsdn_destroy(self, h):
        self.destroyed += 1


@pytest.fixture
def fake_lib(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    return fake


def _small_spec(**extra):
    rng = np.random.default_rng(3)
    return dict(kind="knn", fit_X=rng.random((20, 3)), y=rng.integers(0, 3, 20).astype(np.int32), k=3,
                classes=np.arange(3), n_features=3, **extra)


def test_from_spec_passes_the_metric(fake_lib):
    est = estimators.from_spec(_small_spec(metric="manhattan", weights="distance"))
    assert fake_lib.created == [("metric", _lib.KNN_DISTANCE, _lib.KNN_MANHATTAN)]
    assert est.get_params()["metric"] == "manhattan" and est.effective_metric_ == "manhattan"
    estimators.from_spec(_small_spec(metric="chebyshev"))
    assert fake_lib.created[-1] == ("metric", _lib.KNN_UNIFORM, _lib.KNN_CHEBYSHEV)
    est = estimators.from_spec(_small_spec())          # no key: euclidean, the weighted (euclidean) create call
    assert fake_lib.created[-1] == ("weighted", _lib.KNN_UNIFORM) and est.effective_metric_ == "euclidean"


def test_set_params_metric_keeps_the_fitted_handle(fake_lib):
    est = estimators.from_spec(_small_spec(metric="manhattan"))
    est.set_params(metric="chebyshev", p=1)
    assert len(fake_lib.created) == 1 and fake_lib.destroyed == 0
    assert est.effective_metric_ == "manhattan" and est._spec["metric"] == "manhattan"
    assert est.get_params()["metric"] == "chebyshev"
    est.set_params(weights="distance")                 # weights still re-create, in the fitted metric
    assert fake_lib.created[-1] == ("metric", _lib.KNN_DISTANCE, _lib.KNN_MANHATTAN)


def test_pickling_keeps_the_metric(fake_lib):
    est = estimators.from_spec(_small_spec(metric="chebyshev"))
    back = pickle.loads(pickle.dumps(est))
    assert fake_lib.created[-1] == ("metric", _lib.KNN_UNIFORM, _lib.KNN_CHEBYSHEV)
    assert back._spec["metric"] == "chebyshev" and back.effective_metric_ == "chebyshev"


def test_create_metric_argument_errors():
    """the metric is checked before any device work, so the call answers on any machine"""
    lib = _lib.load()
    fx = np.zeros((10, 3))
    y = np.zeros(10, np.int32)
    h = C.c_void_p()
    args = (fx.ctypes.data_as(_lib._f64p), y.ctypes.data_as(_lib._i32p), 10, 3, 2, 3, _lib.KNN_UNIFORM)
    for metric in (3, -1, 42):
        assert lib.tcsdn_knn_create_metric(*args, metric, C.byref(h)) == _lib.EINVAL
        assert "metric" in _lib.last_error() and h.value is None
    assert lib.tcsdn_knn_create_metric(*args, _lib.KNN_MANHATTAN, None) == _lib.EINVAL
    assert lib.tcsdn_knn_create_metric(*args[:6], 5, _lib.KNN_CHEBYSHEV, C.byref(h)) == _lib.EINVAL
    assert "weights" in _lib.last_error()
