"""KNeighborsClassifier(weights='distance'), CPU side: the definition (tests/knn_weighted_oracle.py) pinned to numpy and to
scikit-learn, the model import, the estimator's plumbing and the C entry point's argument checks.  None of these needs a GPU;
tests/test_knn_weighted_gpu.py checks the kernels against the definition."""
import ctypes as C
import pickle

import numpy as np
import pytest

import kneighbors_oracle as kno
import knn_weighted_oracle as kwo
from traffic_classifier_sdn_b200 import _lib, estimators, modelio


def _sk_distance(spec, k, algorithm):
    from sklearn.neighbors import KNeighborsClassifier
    classes = np.asarray(spec["classes"])
    return KNeighborsClassifier(n_neighbors=k, weights="distance", algorithm=algorithm).fit(spec["fit_X"], classes[spec["y"]])


def _lattice(seed=11, nt=700, nq=2000):
    """integer lattice rows (exact distances in every arithmetic), queries on lattice points and half-way between them"""
    rng = np.random.default_rng(seed)
    tr = np.floor(rng.random((nt, 4)) * 4)
    y = rng.integers(0, 5, nt).astype(np.int32)
    q = np.floor(rng.random((nq, 4)) * 4)
    q[nq // 2:] += 0.5
    return dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(5), n_features=4, weights="distance"), q


# ------------------------------------------------------------------ numpy's association, restated
def test_row_sum_restatement_equals_numpy_for_every_k():
    rng = np.random.default_rng(0)
    for k in range(1, 65):
        a = rng.random((3000, k)) * 10.0 ** rng.integers(-6, 7, (3000, k))
        a[rng.random(a.shape) < 0.4] = 0.0
        assert np.array_equal(kwo.row_sum(a), np.sum(a, axis=1)), k


@pytest.mark.parametrize("n_classes", [2, 6, 8, 17, 200])
def test_row_sum_restatement_equals_numpy_for_the_normaliser(n_classes):
    rng = np.random.default_rng(n_classes)
    P = rng.random((3000, n_classes)) * 10.0 ** rng.integers(-6, 7, (3000, n_classes))
    P[rng.random(P.shape) < 0.6] = 0.0
    assert np.array_equal(kwo.row_sum(P), np.sum(P, axis=1))


# ------------------------------------------------------------------ the definition against scikit-learn
@pytest.mark.parametrize("k,n_open", [(1, 8), (5, 0), (9, 0)])
def test_definition_equals_sklearn_kd_tree_on_bundled_rows(golden, specs, k, n_open):
    """the reference's model (12 features: sklearn picks kd_tree) with weights='distance', all 7 653 bundled rows: labels and
    predict_proba bit-identical on every row whose neighbour SET is defined -- where the k-th and (k+1)-th nearest rows are
    equally distant and of different classes, kd_tree and the index-order heap keep different rows (8 rows at k = 1, all of
    them duplicates of training rows with different labels; pinned).  Most rows are training rows, so the zero-distance
    rule is the common case."""
    spec, X = specs["knn"], np.ascontiguousarray(golden["X"])
    lab, proba = kwo.predict(spec, X, k)
    sk = _sk_distance(spec, k, "kd_tree")
    dist, ind = kno.kneighbors(spec, X, k + 1)
    yk = np.asarray(spec["y"])[ind]
    open_set = (dist[:, k] == dist[:, k - 1]) & (yk[:, k] != yk[:, k - 1])
    assert open_set.sum() == n_open
    ok = ~open_set
    assert np.array_equal(np.asarray(spec["classes"])[lab][ok], sk.predict(X)[ok])
    assert np.array_equal(proba[ok], sk.predict_proba(X)[ok])
    assert (dist[:, 0] == 0.0).sum() > len(X) // 2


@pytest.mark.parametrize("k,n_cross", [(16, 8), (33, 8)])
def test_definition_equals_sklearn_kd_tree_beyond_eight_neighbours(golden, specs, k, n_cross):
    """k >= 8: numpy's row sum is pairwise, so sklearn's label can hang on its undefined order among equally distant rows
    of different classes.  Rows without such a pair in the set: labels bit-identical; predict_proba (sequential class
    sums) bit-identical on every row.  The count of rows with such a pair is pinned."""
    spec, X = specs["knn"], np.ascontiguousarray(golden["X"])
    lab, proba = kwo.predict(spec, X, k)
    sk = _sk_distance(spec, k, "kd_tree")
    cross = kwo.cross_class_ties(spec, X, k)
    assert cross.sum() == n_cross
    clean = ~cross
    assert np.array_equal(np.asarray(spec["classes"])[lab][clean], sk.predict(X)[clean])
    assert np.array_equal(proba, sk.predict_proba(X))


@pytest.mark.parametrize("k", [1, 5, 8, 9])
def test_definition_equals_sklearn_brute_on_a_lattice(k):
    """integer lattice: the GEMM-expanded distances of brute are exact, and brute keeps the same index-order heap, so its
    neighbours and weights are the definition's; queries on lattice points (zero distances) and half-way between them.
    Nearly every row holds equally distant rows of different classes; for k >= 8 the label could hang on sklearn's order
    among them, but on this lattice it does not: labels and predict_proba are bit-identical on every row."""
    spec, q = _lattice()
    lab, proba = kwo.predict(spec, q, k)
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=1):
        sk = _sk_distance(spec, k, "brute")
        sl, sp = sk.predict(q), sk.predict_proba(q)
    dist, _ = kno.kneighbors(spec, q, k)
    assert (dist[:, 0] == 0.0).sum() > 0.3 * len(q) and (dist[:, 0] > 0.0).sum() > 0.3 * len(q)
    if k >= 5:
        assert kwo.cross_class_ties(spec, q, k).mean() > 0.99
    assert np.array_equal(lab, sl)
    assert np.array_equal(proba, sp)


# ------------------------------------------------------------------ model import and the estimator
def test_spec_records_the_weighting():
    from sklearn.neighbors import KNeighborsClassifier
    rng = np.random.default_rng(1)
    X, y = rng.random((60, 3)), rng.integers(0, 3, 60)
    assert modelio.spec_from_estimator(KNeighborsClassifier(3, weights="distance").fit(X, y))["weights"] == "distance"
    assert modelio.spec_from_estimator(KNeighborsClassifier(3).fit(X, y))["weights"] == "uniform"
    with pytest.raises(modelio.SpecError, match="callable"):
        modelio.spec_from_estimator(KNeighborsClassifier(3, weights=lambda d: d).fit(X, y))
    assert modelio.knn_weights(None) == "uniform"
    with pytest.raises(modelio.SpecError):
        modelio.knn_weights("inverse")


def test_spec_round_trips_through_a_pickle():
    """a pickled weights='distance' estimator read as data keeps its weighting"""
    from sklearn.neighbors import KNeighborsClassifier
    rng = np.random.default_rng(2)
    X, y = rng.random((50, 4)), rng.integers(0, 2, 50)
    spec = modelio.spec_from_pickle_bytes(pickle.dumps(KNeighborsClassifier(4, weights="distance").fit(X, y)))
    assert spec["weights"] == "distance" and spec["k"] == 4 and np.array_equal(spec["fit_X"], X)


class _FakeLib:
    """stands in for libtcsdn.so: records the weighting each handle is created with"""

    def __init__(self):
        self.created, self.destroyed = [], 0

    def tcsdn_knn_create_weighted(self, fx, y, n, d, n_classes, k, weights, out):
        self.created.append(weights)
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


def test_from_spec_passes_the_weighting(fake_lib):
    est = estimators.from_spec(_small_spec(weights="distance"))
    assert fake_lib.created == [_lib.KNN_DISTANCE]
    assert est.get_params()["weights"] == "distance" and est.weights == "distance"
    estimators.from_spec(_small_spec())        # no key: uniform, as in the golden specs
    assert fake_lib.created[-1] == _lib.KNN_UNIFORM


def test_set_params_weights_recreates_the_handle(fake_lib):
    est = estimators.from_spec(_small_spec())
    est.set_params(weights="distance")
    assert fake_lib.created == [_lib.KNN_UNIFORM, _lib.KNN_DISTANCE] and fake_lib.destroyed == 1
    assert est._spec["weights"] == "distance" and est.get_params()["weights"] == "distance"
    est.set_params(weights="distance")          # unchanged: the handle stays
    assert len(fake_lib.created) == 2
    est.set_params(weights=None)                # None is sklearn's older spelling of 'uniform'
    assert fake_lib.created[-1] == _lib.KNN_UNIFORM
    with pytest.raises(modelio.SpecError, match="callable"):
        est.set_params(weights=lambda d: d)
    unfitted = estimators.KNeighborsClassifier(3).set_params(weights="distance")
    assert unfitted.get_params()["weights"] == "distance" and len(fake_lib.created) == 3


def test_pickling_keeps_the_weighting(fake_lib):
    est = estimators.from_spec(_small_spec())
    est.set_params(weights="distance")
    back = pickle.loads(pickle.dumps(est))
    assert fake_lib.created[-1] == _lib.KNN_DISTANCE
    assert back._spec["weights"] == "distance" and back.get_params()["weights"] == "distance"


def test_create_weighted_argument_errors():
    """argument checks come before any device work, so they answer on any machine"""
    lib = _lib.load()
    fx = np.zeros((10, 3))
    y = np.zeros(10, np.int32)
    h = C.c_void_p()
    args = (fx.ctypes.data_as(_lib._f64p), y.ctypes.data_as(_lib._i32p), 10, 3, 2, 3)
    for w in (2, -1, 7):
        assert lib.tcsdn_knn_create_weighted(*args, w, C.byref(h)) == _lib.EINVAL
        assert "weights" in _lib.last_error() and h.value is None
    assert lib.tcsdn_knn_create_weighted(*args, _lib.KNN_DISTANCE, None) == _lib.EINVAL
    bad_k = args[:5] + (0,)
    assert lib.tcsdn_knn_create_weighted(*bad_k, _lib.KNN_DISTANCE, C.byref(h)) == _lib.EINVAL
    assert "k" in _lib.last_error()
