"""KNeighborsClassifier(weights='distance') on the GPU: labels and predict_proba of the tensor-core engine (pruned and unpruned),
the fp64 kernel and the index-order tie kernel, bit-identical to the CPU definition (tests/knn_weighted_oracle.py) on every row
checked, for float32 and float64 rows, host arrays and CUDA tensors."""
import pickle

import numpy as np
import pytest

import knn_weighted_oracle as kwo
from traffic_classifier_sdn_b200 import _lib, from_spec, synth

pytestmark = pytest.mark.gpu


def _force(est, mode):
    est.set_option(_lib.OPT_ENGINE, mode)
    return est


def _flows_spec(nt, k=5, seed=0):
    """synthetic flows, weights='distance'; rows 10..19 are copies of row 10 with their own labels (equal zero distances
    of different classes for a query at that row)"""
    X, y = synth.make_flows(nt, seed=seed)
    X = X.copy()
    X[10:20] = X[10]
    return dict(kind="knn", fit_X=X, y=y.astype(np.int32), k=k, classes=synth.CLASSES, n_features=X.shape[1],
                weights="distance")


def _queries(spec, n, seed):
    """flows, the first 300 of them training rows (the zero-distance rule), five of them the duplicated row"""
    Xq = synth.make_flows(n, seed=seed, return_labels=False)
    Xq[:300] = spec["fit_X"][:300]
    Xq[300:305] = spec["fit_X"][10]
    return Xq


def _run(est, Xq, torch_in):
    if torch_in:
        import torch
        Xt = torch.from_numpy(Xq).cuda()
        lab = est.predict_indices(Xt)
        proba = est.predict_proba(Xt)
        return lab.cpu().numpy(), proba
    return est.predict_indices(Xq), est.predict_proba(Xq)


def _check(est, spec, Xq, path, torch_in=False):
    """predict_indices and predict_proba through `path` ('engine' = option 2, 'fp64' = option 1) equal the definition bit
    for bit; the rows went through that path"""
    _force(est, 2 if path == "engine" else 1)
    rl, rp = kwo.predict(spec, Xq)
    lab, proba = _run(est, Xq, torch_in)
    st = est.stats()
    assert st[1 if path == "engine" else 2] == len(Xq), (path, st.tolist())
    assert proba.shape == (len(Xq), len(spec["classes"])) and proba.dtype == np.float64
    assert np.array_equal(lab, rl), f"{path}: labels differ on {(lab != rl).sum()} rows"
    assert np.array_equal(proba, rp), f"{path}: predict_proba differs on {(proba != rp).any(1).sum()} rows"
    return lab, proba


@pytest.mark.parametrize("k", [1, 5, 8, 9, 32])
@pytest.mark.parametrize("path", ["engine", "fp64"])
def test_weighted_bit_exact_vs_definition(k, path):
    spec = _flows_spec(3000, k=k, seed=k)
    est = from_spec(spec)
    Xq = _queries(spec, 5000, seed=k + 100)
    _check(est, spec, Xq, path)
    _check(est, spec, Xq.astype(np.float32), path)
    _check(est, spec, Xq, path, torch_in=True)
    _check(est, spec, Xq.astype(np.float32), path, torch_in=True)


@pytest.mark.parametrize("k", [33, 64])
def test_weighted_beyond_engine_takes_fp64_kernel(k):
    """more than 32 neighbours: no engine for the model, every row goes to the fp64 kernel even on a large batch"""
    spec = _flows_spec(3000, k=k, seed=k)
    est = from_spec(spec)
    Xq = _queries(spec, 6000, seed=k + 7)
    for X in (Xq, Xq.astype(np.float32)):
        lab, proba = _run(est, X, torch_in=False)
        assert est.stats()[2] == len(X) and est.stats()[1] == 0
        rl, rp = kwo.predict(spec, X)
        assert np.array_equal(lab, rl) and np.array_equal(proba, rp)
    lab, proba = _run(est, Xq, torch_in=True)
    rl, rp = kwo.predict(spec, Xq)
    assert np.array_equal(lab, rl) and np.array_equal(proba, rp)


@pytest.mark.parametrize("k", [5, 9])
def test_weighted_pruned_equals_unpruned(k):
    spec = _flows_spec(20000, k=k, seed=k + 3)
    Xq = _queries(spec, 20000, seed=k + 70)
    rl, rp = kwo.predict(spec, Xq)
    for off in (0, 1):
        est = _force(from_spec(spec), 2)
        est.set_option(_lib.OPT_KNN_PRUNE, off)
        lab, proba = _run(est, Xq, torch_in=False)
        assert est.stats()[1] == len(Xq)
        assert np.array_equal(lab, rl) and np.array_equal(proba, rp), f"prune_off={off}"


@pytest.mark.parametrize("k", [1, 5, 9])
def test_weighted_lattice_ties_take_the_tie_kernel(k):
    """on a lattice most rows tie at the k-th distance across classes: the engine sends them to the index-order tie kernel
    (stats[7]), whose weighted vote must equal the definition too"""
    rng = np.random.default_rng(7)
    tr = np.floor(rng.random((900, 4)) * 3)
    y = rng.integers(0, 5, 900).astype(np.int32)
    q = np.floor(rng.random((5000, 4)) * 3)
    q[2500:] += 0.5
    spec = dict(kind="knn", fit_X=tr, y=y, k=k, classes=np.arange(5), n_features=4, weights="distance")
    est = _force(from_spec(spec), 2)
    before = est.stats()[7]
    lab, proba = _run(est, q, torch_in=False)
    assert est.stats()[7] > before
    rl, rp = kwo.predict(spec, q)
    assert np.array_equal(lab, rl) and np.array_equal(proba, rp)
    lab, proba = _run(est, q.astype(np.float32), torch_in=True)
    assert np.array_equal(lab, rl) and np.array_equal(proba, rp)


def test_weighted_reference_model(golden, specs):
    """the reference's model with weights='distance' on all 7 653 bundled rows (4 390 of them at distance 0 from a training
    row): engine and fp64 kernel equal the definition, and scikit-learn kd_tree on every row"""
    spec, X = dict(specs["knn"], weights="distance"), np.ascontiguousarray(golden["X"])
    est = from_spec(spec)
    lab, proba = _check(est, spec, X, "engine")
    _check(est, spec, X, "fp64")
    _check(est, spec, X.astype(np.float32), "engine", torch_in=True)
    from sklearn.neighbors import KNeighborsClassifier
    classes = np.asarray(spec["classes"])
    sk = KNeighborsClassifier(spec["k"], weights="distance", algorithm="kd_tree").fit(spec["fit_X"], classes[spec["y"]])
    assert np.array_equal(classes[lab], sk.predict(X))
    assert np.array_equal(proba, sk.predict_proba(X))


def test_weighted_training_rows_with_duplicates():
    """queries that are training rows, several of them duplicated under different labels: every row has a zero distance, so
    only the exact copies vote (weight 1 each)"""
    rng = np.random.default_rng(5)
    base = rng.normal(0, 50.0, (6000, 12))
    base[100:110] = base[100]
    base[200:203] = base[200]
    base[300:340] = base[300]          # more copies than neighbours
    y = rng.integers(0, 4, len(base)).astype(np.int32)
    y[100:110] = [0, 1, 1, 2, 3, 3, 3, 0, 1, 2]
    for k in (5, 9):
        spec = dict(kind="knn", fit_X=base, y=y, k=k, classes=np.arange(4), n_features=12, weights="distance")
        est = from_spec(spec)
        for path in ("engine", "fp64"):
            _, proba = _check(est, spec, base, path)
            assert np.all(np.isin(proba[:100], [0.0, 1.0]))   # a distinct row: its own class alone


def test_weighted_large_model_on_a_million_rows():
    """the bench model (50 000 training rows, k = 5) with weights='distance' on 1M device rows: a strided sample of 2 000
    rows equals the definition, labels and predict_proba"""
    import torch
    import bench
    w = bench.build_workload("knn")
    spec = dict(w["spec"], weights="distance")
    est = from_spec(spec)
    n = 1_000_000
    Xd = bench.synth_rows(n, w["d"], seed=5, device=torch.device("cuda", 0))
    lab = est.predict_indices(Xd)
    proba = est.predict_proba(Xd)
    assert est.stats()[1] == n
    sel = torch.from_numpy(np.arange(0, n, n // 2000)[:2000] + 11).cuda()
    Xs = Xd[sel].cpu().numpy()
    rl, rp = kwo.predict(spec, Xs)
    assert np.array_equal(lab[sel].cpu().numpy(), rl)
    assert np.array_equal(proba[sel.cpu().numpy()], rp)


def test_fit_predict_equals_sklearn_end_to_end(golden, specs):
    """tc.KNeighborsClassifier(weights='distance').fit(X, y).predict(X') is scikit-learn's on the bundled rows"""
    import traffic_classifier_sdn_b200 as tc
    from sklearn.neighbors import KNeighborsClassifier
    spec, X = specs["knn"], np.ascontiguousarray(golden["X"])
    Xt, yt = spec["fit_X"], np.asarray(spec["classes"])[spec["y"]]
    ours = tc.KNeighborsClassifier(weights="distance").fit(Xt, yt)
    theirs = KNeighborsClassifier(weights="distance").fit(Xt, yt)
    assert ours.get_params()["weights"] == "distance"
    assert np.array_equal(ours.predict(X), theirs.predict(X))
    assert np.array_equal(ours.predict_proba(X), theirs.predict_proba(X))


def test_set_params_and_pickle_switch_the_vote(golden, specs):
    """set_params(weights=...) on a fitted model changes what predict computes; a pickle keeps it"""
    import oracle
    spec, X = specs["knn"], np.ascontiguousarray(golden["X"])
    est = from_spec(spec)
    assert np.array_equal(est.predict_indices(X), oracle.knn(spec, X, want_scores=False)[0])
    est.set_params(weights="distance")
    rl, rp = kwo.predict(spec, X)
    assert np.array_equal(est.predict_indices(X), rl) and np.array_equal(est.predict_proba(X), rp)
    back = pickle.loads(pickle.dumps(est))
    assert np.array_equal(back.predict_indices(X), rl) and np.array_equal(back.predict_proba(X), rp)
    with pytest.raises(ValueError, match="audit"):
        _force(back, 3).predict_indices(X)
    est.set_params(weights="uniform")
    lab, sc = oracle.knn(spec, X)
    assert np.array_equal(est.predict_indices(X), lab) and np.array_equal(est.predict_proba(X), sc)
