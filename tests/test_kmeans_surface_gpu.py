"""KMeans.transform, KMeans.score and the k-means++ seeding on the GPU against their CPU definition
(tests/kmeans_oracle.py) and scikit-learn."""
import numpy as np
import pytest

import kmeans_oracle as ko
import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import _lib, synth

pytestmark = pytest.mark.gpu


def _model(d, k, seed=0):
    rng = np.random.default_rng(seed)
    X = synth.make_flows(4000, seed=seed + 1, return_labels=False)
    cols = rng.integers(0, X.shape[1], d)
    X = np.ascontiguousarray(X[:, cols])
    return tc.from_spec(dict(kind="kmeans", centers=X[rng.choice(len(X), k, replace=False)], classes=np.arange(k, dtype=np.int32),
                             n_features=d)), cols


def _rows(n, cols, dtype, seed=7):
    return np.ascontiguousarray(synth.make_flows(max(n, 1), seed=seed, return_labels=False)[:n][:, cols], dtype)


def _sk_bound(X, Cn):
    X = np.asarray(X, np.float64)
    return 8 * (X.shape[1] + 2) * ko.U * ((X * X).sum(1)[:, None] + (Cn * Cn).sum(1)[None, :])


def _check_transform(est, X, got, want=None):
    """got == the definition (bit for bit), and within the cancellation bound of scikit-learn's euclidean_distances"""
    from sklearn.metrics.pairwise import euclidean_distances
    Cn = est.cluster_centers_
    if want is None:
        want = ko.transform(X, Cn)
    assert got.shape == want.shape and got.dtype == np.float64
    assert np.array_equal(got, want)
    if len(X):
        ref = euclidean_distances(np.asarray(X, np.float64), Cn)
        assert (np.abs(want * want - ref * ref) <= _sk_bound(X, Cn)).all()
    return want


@pytest.mark.parametrize("d", [1, 4, 8, 12, 16, 20])
@pytest.mark.parametrize("k", [1, 3, 8, 9, 33])
def test_transform_is_the_definition(d, k):
    import torch
    est, cols = _model(d, k, seed=d * 100 + k)
    for dtype in (np.float64, np.float32):
        for n in (0, 1, 127, 128, 129, 5000):
            X = _rows(n, cols, dtype)
            _check_transform(est, X, est.transform(X))
        X = _rows(100_000, cols, dtype)
        want = _check_transform(est, X, est.transform(X))
        # every scorer CTA shape (TCSDN_OPT_SCORER_SHAPE 1..3, 0 = automatic) and the generic kernel (engine option 1)
        for shape in (0, 1, 2, 3):
            est.set_option(_lib.OPT_SCORER_SHAPE, shape)
            assert np.array_equal(est.transform(X), want)
        est.set_option(_lib.OPT_SCORER_SHAPE, 0)
        est.set_option(_lib.OPT_ENGINE, 1)
        assert np.array_equal(est.transform(X), want)
        est.set_option(_lib.OPT_ENGINE, 0)
        t = torch.from_numpy(X).cuda()
        got = est.transform(t)
        assert got.is_cuda
        est.sync_check()
        assert np.array_equal(got.cpu().numpy(), want)
        est.set_option(_lib.OPT_CHUNK_ROWS, 4097)   # ragged host chunks
        assert np.array_equal(est.transform(X), want)
        est.set_option(_lib.OPT_CHUNK_ROWS, 0)


@pytest.mark.parametrize("d,k", [(12, 5), (4, 8), (16, 2), (20, 33), (8, 12)])
def test_score_is_within_gamma_n_of_exact_and_repeatable(d, k):
    import torch
    from fractions import Fraction
    from sklearn.cluster._k_means_common import _inertia_dense
    est, cols = _model(d, k, seed=d + k)
    for dtype in (np.float64, np.float32):
        for n in (1, 129, 100_000):
            X = _rows(n, cols, dtype, seed=n)
            labels = est.predict(X)
            terms = ko.inertia_terms(X, est.cluster_centers_, labels)
            exact = sum(Fraction(float(t)) for t in terms)
            sk = _inertia_dense(np.asarray(X, np.float64), np.ones(n), est.cluster_centers_, labels.astype(np.int32), n_threads=1)
            runs = {}
            for shape in (0, 1, 2, 3):
                est.set_option(_lib.OPT_SCORER_SHAPE, shape)
                runs[f"shape{shape}"] = est.score(X)
            est.set_option(_lib.OPT_SCORER_SHAPE, 0)
            est.set_option(_lib.OPT_ENGINE, 1)
            runs["generic"] = est.score(X)
            est.set_option(_lib.OPT_ENGINE, 0)
            est.set_option(_lib.OPT_CHUNK_ROWS, 4097)
            runs["chunked"] = est.score(X)
            est.set_option(_lib.OPT_CHUNK_ROWS, 0)
            runs["device"] = est.score(torch.from_numpy(X).cuda())
            for name, s in runs.items():
                assert isinstance(s, float)
                assert abs(Fraction(-s) - exact) <= Fraction(ko.gamma(n)) * exact, name
                assert abs(-s - sk) <= 2 * ko.gamma(n) * float(exact), name
            assert est.score(X) == runs["shape0"] and est.score(X) == runs["shape0"]     # the same bits every call
    assert est.score(X[:0]) == 0.0


def test_surface_errors_and_fit_transform():
    import torch
    from sklearn.cluster import KMeans as SK
    est, cols = _model(12, 5)
    X = _rows(5000, cols, np.float64)
    bad = X.copy()
    bad[123, 4] = np.nan
    with pytest.raises(ValueError):
        est.transform(bad)
    with pytest.raises(ValueError):
        est.score(bad)
    bad[123, 4] = np.inf
    t = torch.from_numpy(bad).cuda()
    est.transform(t)
    with pytest.raises(ValueError):
        est.sync_check()
    with pytest.raises(ValueError):
        est.score(t)
    _check_transform(est, X, est.transform(X))     # the handle stays usable
    with pytest.raises(ValueError):
        est.score(X, sample_weight=np.ones(len(X)))
    with pytest.raises(ValueError):
        est.transform(X[:, :5])
    svc_like = tc.from_spec(dict(kind="linear", coef=np.ones((1, 12)), intercept=np.zeros(1), classes=np.arange(2), n_features=12))
    assert _lib.load().tcsdn_kmeans_transform(svc_like._handle, X.ctypes.data, 1, 12, _lib.F64, _lib.HOST,
                                              np.zeros(5).ctypes.data, None) == _lib.EINVAL
    Xf = synth.make_flows(30_000, seed=21, return_labels=False)
    ft = tc.KMeans(n_clusters=4, n_init=1, random_state=0).fit_transform(Xf)
    sk = SK(n_clusters=4, n_init=1, random_state=0).fit(Xf)
    assert ft.shape == (len(Xf), 4)
    np.testing.assert_allclose(ft, sk.transform(Xf), rtol=1e-6, atol=1e-6 * np.abs(sk.cluster_centers_).max())
    np.testing.assert_allclose(tc.KMeans(n_clusters=4, n_init=1, random_state=0).fit(Xf).score(Xf), sk.score(Xf), rtol=1e-9)


def _seed_cases(golden):
    flows = synth.make_flows(40_000, seed=21, return_labels=False)
    yield "golden", np.ascontiguousarray(golden["X"], np.float64), [(1, 0), (2, 1), (4, 0), (4, 1), (4, 7), (33, 0)]
    yield "flows", flows, [(1, 3), (5, 0), (5, 3), (5, 7), (12, 0), (12, 5), (33, 2)]


def test_seeding_is_the_definition_and_sklearns(golden):
    import torch
    from sklearn.cluster import kmeans_plusplus as sk_pp
    undecided = 0
    for name, X, cases in _seed_cases(golden):
        bound = ko.seeding_bound(len(X))
        Xd = torch.from_numpy(X).cuda()
        for k, seed in cases:
            idx_def, draw_m, choice_m = ko.kmeans_plusplus(X, k, random_state=seed)
            centers, idx = tc.kmeans_plusplus(X, k, random_state=seed)
            assert idx.dtype == np.int64 and centers.shape == (k, X.shape[1]) and centers.dtype == np.float64
            assert np.array_equal(centers, X[idx])
            if (draw_m > bound).all() and (choice_m > bound).all():
                assert np.array_equal(idx, idx_def), (name, k, seed)
            else:
                undecided += 1
            _, sk_idx = sk_pp(X, k, random_state=seed)
            assert np.array_equal(X[idx], X[sk_idx]), (name, k, seed)
            c2, i2 = tc.kmeans_plusplus(Xd, k, random_state=seed)            # device rows: the same seeding
            assert np.array_equal(i2, idx) and np.array_equal(c2, centers)
            c3, i3 = tc.kmeans_plusplus(X.astype(np.float32), k, random_state=seed)
            assert c3.dtype == np.float32 and np.array_equal(c3, X.astype(np.float32)[i3])
    assert undecided == 0


def test_seeding_edges():
    from sklearn.cluster import kmeans_plusplus as sk_pp
    rng = np.random.default_rng(4)
    lattice = rng.integers(0, 3, (3000, 4)).astype(np.float64)
    few = np.repeat(np.eye(3), 50, axis=0)                          # 3 distinct rows, k = 6: the potential reaches 0
    for X, k, L in ((lattice, 12, None), (lattice, 6, 1), (lattice, 5, 9), (few, 6, None), (few[:7], 7, 3)):
        centers, idx = tc.kmeans_plusplus(X, k, random_state=1, n_local_trials=L)
        _, sk_idx = sk_pp(X, k, random_state=1, n_local_trials=L)
        assert np.array_equal(X[idx], X[sk_idx]), (k, L)
        assert np.array_equal(idx, ko.kmeans_plusplus(X, k, random_state=1, n_local_trials=L)[0]), (k, L)
    with pytest.raises(ValueError):
        tc.kmeans_plusplus(lattice[:3], 4)
    bad = lattice.copy()
    bad[5, 1] = np.nan
    with pytest.raises(ValueError):
        tc.kmeans_plusplus(bad, 3, random_state=0)


def test_device_fit_copies_no_rows_to_the_host():
    import torch
    from sklearn.cluster import KMeans as SK
    X = synth.make_flows(40_000, seed=21, return_labels=False)
    for k, seed in ((5, 0), (5, 7), (12, 5)):
        sk = SK(n_clusters=k, n_init=1, random_state=seed).fit(X)
        t = torch.from_numpy(X).cuda()

        class NoHost(torch.Tensor):
            __module__ = "torch"   # a CUDA torch tensor to the estimator, whose host copies fail

            def cpu(self, *a, **kw):
                raise AssertionError("the rows were copied to the host")

            def numpy(self, *a, **kw):
                raise AssertionError("the rows were copied to the host")

        est = tc.KMeans(n_clusters=k, n_init=1, random_state=seed).fit(t.as_subclass(NoHost))
        scale = np.abs(sk.cluster_centers_).max()
        np.testing.assert_allclose(est.cluster_centers_, sk.cluster_centers_, rtol=1e-9, atol=1e-9 * scale)
        assert np.array_equal(est.labels_, sk.labels_) and est.n_iter_ == sk.n_iter_
