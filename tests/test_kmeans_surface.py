"""The CPU definition of KMeans.transform, KMeans.score and the k-means++ seeding (tests/kmeans_oracle.py) against
scikit-learn, and the argument checks of their C ABI, which return before any device work."""
import ctypes as C

import numpy as np
import pytest

import kmeans_oracle as ko
from traffic_classifier_sdn_b200 import _lib, synth


@pytest.mark.parametrize("d", range(1, 17))
def test_sqdist_is_sklearns_euclidean_dense_dense(d):
    from sklearn.cluster._k_means_common import _euclidean_dense_dense_wrapper
    rng = np.random.default_rng(d)
    X = rng.standard_normal((40, d)) * 10.0 ** rng.integers(-3, 4, (40, d))
    Cn = rng.standard_normal((5, d)) * 100
    got = ko.sqdist(X, Cn)
    for i in range(len(X)):
        for c in range(len(Cn)):
            want = _euclidean_dense_dense_wrapper(X[i], Cn[c], True)
            assert got[i, c] == want, (i, c, got[i, c], want)


def _lattice():
    rng = np.random.default_rng(4)
    return rng.integers(0, 3, (3000, 4)).astype(np.float64)    # 81 distinct rows, many duplicates


@pytest.mark.parametrize("case", [("flows", 5, 0), ("flows", 5, 3), ("flows", 5, 7), ("flows", 12, 5), ("lattice", 6, 0),
                                  ("lattice", 12, 2)])
def test_seeding_definition_is_sklearns(case):
    from sklearn.cluster import kmeans_plusplus
    name, k, seed = case
    X = synth.make_flows(40_000, seed=21, return_labels=False) if name == "flows" else _lattice()
    idx, draw_m, choice_m = ko.kmeans_plusplus(X, k, random_state=seed)
    _, sk_idx = kmeans_plusplus(X, k, random_state=seed)
    assert np.array_equal(X[idx], X[sk_idx])
    bound = ko.seeding_bound(len(X))
    assert (draw_m > bound).all() and (choice_m > bound).all(), (draw_m.min(), choice_m.min() if len(choice_m) else None)


def test_seeding_definition_is_sklearns_on_centred_flows():
    """KMeans.fit seeds on the mean-centred rows in scikit-learn, on the rows as given here: the same rows are chosen."""
    from sklearn.cluster import kmeans_plusplus
    X = synth.make_flows(40_000, seed=21, return_labels=False)
    for k, seed in ((5, 0), (5, 1), (5, 7), (12, 0)):
        idx, _, _ = ko.kmeans_plusplus(X, k, random_state=seed)
        _, sk_idx = kmeans_plusplus(X - X.mean(axis=0), k, random_state=seed)
        assert np.array_equal(X[idx], X[sk_idx]), (k, seed)


def test_score_and_transform_definitions_against_sklearn():
    from sklearn.cluster._k_means_common import _inertia_dense
    from sklearn.metrics.pairwise import euclidean_distances
    X = synth.make_flows(20_000, seed=3, return_labels=False)
    rng = np.random.default_rng(0)
    Cn = X[rng.choice(len(X), 7, replace=False)]
    labels = np.argmin(ko.sqdist(X, Cn), axis=1).astype(np.int32)
    terms = ko.inertia_terms(X, Cn, labels)
    exact = float(sum(Fraction_(t) for t in terms))
    sk = _inertia_dense(X, np.ones(len(X)), Cn, labels, n_threads=1)
    assert abs(sk - exact) <= ko.gamma(len(X)) * exact
    D = ko.transform(X, Cn)
    ref = euclidean_distances(X, Cn)
    d = X.shape[1]
    bound = 8 * (d + 2) * ko.U * ((X * X).sum(1)[:, None] + (Cn * Cn).sum(1)[None, :])
    assert (np.abs(D * D - ref * ref) <= bound).all()


def Fraction_(t):
    from fractions import Fraction
    return Fraction(float(t))


def test_abi_argument_errors_need_no_gpu():
    lib = _lib.load()
    x = np.zeros((4, 3))
    xp = x.ctypes.data_as(C.c_void_p)
    u = np.zeros(8)
    up = u.ctypes.data_as(_lib._f64p)
    ind = np.zeros(8, np.int64)
    ip = ind.ctypes.data_as(_lib._i64p)
    ctr = np.zeros(32)
    cp = ctr.ctypes.data_as(_lib._f64p)
    pp = lib.tcsdn_kmeans_plusplus
    assert pp(xp, 4, 3, 5, _lib.F64, _lib.HOST, 0, 1, up, ip, cp, None) == _lib.EINVAL      # k > n
    assert pp(xp, 4, 3, 0, _lib.F64, _lib.HOST, 0, 1, up, ip, cp, None) == _lib.EINVAL      # k < 1
    assert pp(xp, 4, 3, 2, _lib.F64, _lib.HOST, 0, 0, up, ip, cp, None) == _lib.EINVAL      # n_local_trials < 1
    assert pp(xp, 4, 3, 2, _lib.F64, _lib.HOST, 4, 1, up, ip, cp, None) == _lib.EINVAL      # first index out of range
    assert pp(None, 4, 3, 2, _lib.F64, _lib.HOST, 0, 1, up, ip, cp, None) == _lib.EINVAL
    assert pp(xp, 4, 3, 2, _lib.F64, _lib.HOST, 0, 1, None, ip, cp, None) == _lib.EINVAL    # uniforms needed for k > 1
    assert pp(xp, 4, 3, 2, _lib.F64, _lib.HOST, 0, 1, up, None, cp, None) == _lib.EINVAL
    assert pp(xp, 4, 3, 2, _lib.F64, _lib.HOST, 0, 1, up, ip, None, None) == _lib.EINVAL
    assert pp(xp, 4, 3, 2, 7, _lib.HOST, 0, 1, up, ip, cp, None) == _lib.EINVAL              # dtype
    out = np.zeros(8)
    inertia = C.c_double(0.0)
    assert lib.tcsdn_kmeans_transform(None, xp, 4, 3, _lib.F64, _lib.HOST, out.ctypes.data_as(C.c_void_p), None) == _lib.EINVAL
    assert lib.tcsdn_kmeans_score(None, xp, 4, 3, _lib.F64, _lib.HOST, C.byref(inertia), None) == _lib.EINVAL


def test_estimator_surface_without_gpu():
    import traffic_classifier_sdn_b200 as tc
    km = tc.KMeans(n_clusters=3)
    for name in ("transform", "fit_transform", "score"):
        assert callable(getattr(km, name))
    with pytest.raises(tc.NotFittedError):
        km.transform(np.zeros((2, 3)))
    with pytest.raises(tc.NotFittedError):
        km.score(np.zeros((2, 3)))
    assert callable(tc.kmeans_plusplus)
