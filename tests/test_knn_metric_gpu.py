"""KNeighborsClassifier(metric='manhattan' | 'chebyshev') on the GPU: the pruned CUDA-core kernel (pruned and visiting every
tile), the fp64 kernel and the index-order tie kernel, bit-identical to the CPU definition (tests/knn_metric_oracle.py) in
labels, predict_proba and kneighbors, for float32 and float64 rows, host arrays and CUDA tensors."""
import numpy as np
import pytest

import kneighbors_oracle as kno
import knn_metric_oracle as kmo
from traffic_classifier_sdn_b200 import KNeighborsClassifier, _lib, from_spec, synth

pytestmark = pytest.mark.gpu

PRUNED, FP64 = 2, 1   # TCSDN_OPT_ENGINE values


def _spec(nt, metric, k=5, weights="uniform", d=12, seed=0, dup=True):
    X, y = synth.make_flows(nt, seed=seed)
    X = np.ascontiguousarray(X[:, :d]) if d <= 12 else np.hstack([X, X[:, :d - 12] * 0.5])
    if dup:
        X[10:20] = X[10]          # equal distances of different classes
    return dict(kind="knn", fit_X=X, y=y.astype(np.int32), k=k, classes=synth.CLASSES, n_features=X.shape[1],
                weights=weights, metric=metric)


def _queries(spec, n, seed):
    Xq = synth.make_flows(max(n, 1), seed=seed, return_labels=False)[:n]
    d = spec["fit_X"].shape[1]
    Xq = np.ascontiguousarray(Xq[:, :d]) if d <= 12 else np.hstack([Xq, Xq[:, :d - 12] * 0.5])
    m = min(n, 300)
    Xq[:m] = spec["fit_X"][:m]
    return Xq


def _model(spec, engine=0, prune=0):
    est = from_spec(spec)
    est.set_option(_lib.OPT_ENGINE, engine)
    est.set_option(_lib.OPT_KNN_PRUNE, prune)
    return est


def _check(est, spec, Xq, torch_in=False, rows=None):
    """labels, predict_proba and kneighbors (distances included) bit-identical to the definition on `rows` (all by default)"""
    rows = np.arange(len(Xq)) if rows is None else rows
    X = Xq
    if torch_in:
        import torch
        X = torch.from_numpy(Xq).cuda()
    lab = est.predict_indices(X)
    proba = est.predict_proba(X)
    dist, ind = est.kneighbors(X)
    if torch_in:
        est.sync_check()
        lab, dist, ind = lab.cpu().numpy(), dist.cpu().numpy(), ind.cpu().numpy()
    want_l, want_p = kmo.predict(spec, Xq[rows])
    wd, wi = kmo.kneighbors(spec, Xq[rows], spec["k"])
    assert np.array_equal(lab[rows], want_l)
    assert np.array_equal(proba[rows], want_p)
    assert np.array_equal(ind[rows], wi) and np.array_equal(dist[rows], wd)
    return est.stats()


@pytest.mark.parametrize("metric", kmo.METRICS)
@pytest.mark.parametrize("weights", ["uniform", "distance"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pruned_kernel_equals_definition(metric, weights, dtype):
    spec = _spec(4000, metric, weights=weights)
    Xq = _queries(spec, 6000, 1).astype(dtype)
    for prune in (0, 1):
        est = _model(spec, PRUNED, prune)
        st = _check(est, spec, Xq)
        assert st[1] == len(Xq) and st[2] == 0
    st = _check(_model(spec, PRUNED), spec, Xq, torch_in=True)
    assert st[1] == len(Xq)


@pytest.mark.parametrize("metric", kmo.METRICS)
@pytest.mark.parametrize("k", [1, 9, 32, 33, 64])
def test_k_range(metric, k):
    spec = _spec(3000, metric, k=k, weights="distance")
    Xq = _queries(spec, 5000, 2)
    est = _model(spec)
    st = _check(est, spec, Xq)
    assert (st[1] == len(Xq)) == (k <= 32)               # k > 32: the fp64 kernel
    if k <= 32:
        _check(_model(spec, FP64), spec, Xq)


@pytest.mark.parametrize("metric", kmo.METRICS)
def test_ties_go_to_the_index_order_kernel(metric):
    """integer lattice training rows and queries: dense ties at the k-th distance"""
    rng = np.random.default_rng(3)
    tr = np.floor(rng.random((5000, 4)) * 6)
    spec = dict(kind="knn", fit_X=tr, y=rng.integers(0, 5, 5000).astype(np.int32), k=5, classes=np.arange(5), n_features=4,
                metric=metric)
    q = np.floor(rng.random((8000, 4)) * 6)
    q[4000:] += 0.5
    st = _check(_model(spec), spec, q)
    assert st[1] == len(q) and st[7] > 0
    _check(_model(spec, 0, 1), spec, q)
    for w in ("distance",):
        s2 = dict(spec, weights=w)
        _check(_model(s2), s2, q)


@pytest.mark.parametrize("metric", kmo.METRICS)
@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 4095, 4096, 4097, 100_000])
def test_batch_sizes(metric, n):
    spec = _spec(2000, metric)
    Xq = _queries(spec, n, 4)
    est = _model(spec)
    if n == 0:
        assert est.predict_indices(Xq).shape == (0,)
        return
    rows = np.arange(n) if n < 10_000 else np.random.default_rng(0).choice(n, 2000, replace=False)
    st = _check(est, spec, Xq, rows=rows)
    assert st[1] == (n if n >= 1024 else 0)           # the dispatch crossover


@pytest.mark.parametrize("metric", kmo.METRICS)
@pytest.mark.parametrize("d", [1, 2, 7, 12, 13])
def test_feature_counts(metric, d):
    spec = _spec(3000, metric, d=d)
    Xq = _queries(spec, 5000, 5)
    st = _check(_model(spec), spec, Xq)
    assert st[1] == (len(Xq) if d <= 12 else 0)          # 13 features: the fp64 kernel
    if d > 12:
        est = _model(spec)
        with pytest.raises(ValueError, match="pruned kernel forced"):
            est.set_option(_lib.OPT_ENGINE, PRUNED).predict_indices(Xq)


@pytest.mark.parametrize("metric", kmo.METRICS)
def test_host_chunks_and_kneighbors_self(metric):
    spec = _spec(3000, metric, weights="distance")
    Xq = _queries(spec, 10_500, 6).astype(np.float32)
    est = _model(spec)
    est.set_option(_lib.OPT_CHUNK_ROWS, 4096)            # ragged last chunk of 2 308 rows
    _check(est, spec, Xq)
    d1, i1 = est.kneighbors()                            # X=None: the training rows, each without itself
    wd, wi = kno.exclude_self(*kmo.kneighbors(spec, spec["fit_X"], spec["k"] + 1))
    assert np.array_equal(i1, wi) and np.array_equal(d1, wd)


@pytest.mark.parametrize("metric", kmo.METRICS)
def test_large_model_without_neighbour_table(metric):
    """270k training rows: more than 4096 tiles, so the walk goes outwards in kd order"""
    spec = _spec(270_000, metric, dup=False)
    Xq = _queries(spec, 20_000, 7)
    rows = np.random.default_rng(1).choice(len(Xq), 500, replace=False)
    st = _check(_model(spec), spec, Xq, rows=rows)
    assert st[1] == len(Xq)


@pytest.mark.parametrize("metric", kmo.METRICS)
def test_bench_model_on_a_million_rows(metric):
    spec = _spec(50_000, metric, dup=False)
    Xq = synth.make_flows(1_000_000, seed=8, return_labels=False).astype(np.float32)
    rows = np.random.default_rng(2).choice(len(Xq), 2000, replace=False)
    st = _check(_model(spec), spec, Xq, rows=rows)
    assert st[1] == len(Xq)
    assert np.array_equal(_model(spec, FP64).predict_indices(Xq[rows]), _model(spec).predict_indices(Xq)[rows])


@pytest.mark.parametrize("metric", ["manhattan", "chebyshev", "l1", "cityblock", "infinity"])
def test_fit_predict_equals_sklearn(golden, metric):
    from sklearn.neighbors import KNeighborsClassifier as SK
    from traffic_classifier_sdn_b200 import modelio
    X, y = synth.make_flows(3000, seed=9)
    Xq = np.ascontiguousarray(golden["X"])
    ours = KNeighborsClassifier(5, metric=metric).fit(X, y)     # sklearn's own algorithm choice, then the import
    sk = SK(5, metric=modelio.knn_metric(metric), algorithm="brute").fit(X, y)   # brute does not take 'infinity'
    assert ours.effective_metric_ == sk.effective_metric_
    assert np.array_equal(ours.predict(Xq), sk.predict(Xq))
    sd, si = kno.canonical(*sk.kneighbors(Xq))
    dist, ind = ours.kneighbors(Xq)
    assert np.array_equal(dist, sd)


@pytest.mark.parametrize("metric", kmo.METRICS)
def test_nan_rows_are_reported(metric):
    spec = _spec(2000, metric)
    Xq = _queries(spec, 6000, 10)
    Xq[4500, 3] = np.nan
    for engine in (0, FP64):
        est = _model(spec, engine)
        with pytest.raises(ValueError, match="NaN"):
            est.predict(Xq)
        with pytest.raises(ValueError, match="NaN"):
            est.kneighbors(Xq)
        import torch
        est.predict_indices(torch.from_numpy(Xq).cuda())
        with pytest.raises(ValueError, match="NaN"):
            est.sync_check()


def test_engine_options(golden):
    spec = _spec(2000, "manhattan")
    est = from_spec(spec)
    for bad in (3, 4):
        with pytest.raises(ValueError, match="engine options 3 and 4"):
            est.set_option(_lib.OPT_ENGINE, bad)
    est.set_option(_lib.OPT_ENGINE, PRUNED)
    assert est.predict_indices(_queries(spec, 10, 11)).shape == (10,) and est.stats()[1] == 10
