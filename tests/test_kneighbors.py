"""KNeighborsClassifier.kneighbors: the neighbours predict votes on, in canonical (distance, index) order, with exact fp64
distances -- on the tensor-core engine and the fp64 kernel, bit-exact against the CPU definition (tests/kneighbors_oracle.py),
which is itself pinned to scikit-learn here.

Unmarked tests check the CPU definition against live scikit-learn; the ``gpu`` tests check the library against it."""
import numpy as np
import pytest

import kneighbors_oracle as kno
import oracle
from traffic_classifier_sdn_b200 import _lib, from_spec, synth


def _lattice(seed=7, nt=600, nq=3000):
    rng = np.random.default_rng(seed)
    tr = np.floor(rng.random((nt, 4)) * 3)   # tiny lattice: masses of exact distance ties, exact integer arithmetic
    y = rng.integers(0, 5, nt).astype(np.int32)
    q = np.floor(rng.random((nq, 4)) * 3)
    return dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(5), n_features=4), q


# ------------------------------------------------------------------ the CPU definition against scikit-learn
@pytest.mark.parametrize("k", [1, 5, 9])
def test_oracle_kneighbors_vs_sklearn_brute_lattice(k):
    """the heap set, sorted canonically, is sklearn brute's (sequential parallel_on_X reduction); distances are exact on a lattice"""
    spec, q = _lattice()
    dist, ind = kno.kneighbors(spec, q, k)
    from sklearn.neighbors import KNeighborsClassifier
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=1):
        sk = KNeighborsClassifier(k, algorithm="brute").fit(spec["fit_X"], spec["y"])
        sd, si = kno.canonical(*sk.kneighbors(q))
    assert np.array_equal(ind, si) and np.array_equal(dist, sd)


def test_oracle_kneighbors_vs_sklearn_kd_tree_bundled(golden, specs):
    """the reference's model runs kd_tree: identical sorted distances on every bundled row, identical neighbours wherever
    the k-th and (k+1)-th distances differ (elsewhere the two choose differently among equally distant rows)"""
    from sk_rebuild import sklearn_from_spec
    spec, X = specs["knn"], golden["X"]
    k = spec["k"]
    dist, ind = kno.kneighbors(spec, X, k + 1)
    sd, si = kno.canonical(*sklearn_from_spec(spec, knn_algorithm="kd_tree").kneighbors(X, k))
    assert np.array_equal(dist[:, :k], sd)
    clear = dist[:, k] != dist[:, k - 1]
    assert clear.sum() > 0.5 * len(X)
    d5, i5 = kno.kneighbors(spec, X, k)
    assert np.array_equal(d5, dist[:, :k])
    assert np.array_equal(i5[clear], si[clear])


def test_oracle_kneighbors_set_is_predicts(golden, specs):
    """with m == k the vote of y[ind] (first maximum) is the oracle's predict label"""
    spec, X = specs["knn"], golden["X"]
    _, ind = kno.kneighbors(spec, X, spec["k"])
    votes = np.stack([np.bincount(r, minlength=len(spec["classes"])) for r in spec["y"][ind]])
    assert np.array_equal(votes.argmax(1), oracle.knn(spec, X, want_scores=False)[0])


# ------------------------------------------------------------------ the library (GPU)
def _force(est, mode):
    est.set_option(_lib.OPT_ENGINE, mode)
    return est


def _flows_spec(nt, k=5, seed=0):
    X, y = synth.make_flows(nt, seed=seed)
    return dict(kind="knn", fit_X=X.copy(), y=y.astype(np.int32), k=k, classes=synth.CLASSES, n_features=X.shape[1])


def _vote(y, ind, n_classes):
    """first-maximum vote of y[ind] per row (numpy)"""
    cnt = np.zeros((ind.shape[0], n_classes), np.int64)
    np.add.at(cnt, (np.arange(ind.shape[0])[:, None], y[ind]), 1)
    return cnt.argmax(1)


def _check(est, spec, Xq, m, path, torch_in=False):
    """kneighbors through `path` ('engine' = option 2, 'fp64' = option 1) equals the CPU definition bit for bit"""
    _force(est, 2 if path == "engine" else 1)
    rd, ri = kno.kneighbors(spec, Xq, m)
    if torch_in:
        import torch
        Xt = torch.from_numpy(Xq).cuda()
        dist, ind = est.kneighbors(Xt, m)
        ind_only = est.kneighbors(Xt, m, return_distance=False)
        est.sync_check()
        assert ind.dtype == torch.int64 and dist.dtype == torch.float64 and ind.is_cuda
        dist, ind, ind_only = dist.cpu().numpy(), ind.cpu().numpy(), ind_only.cpu().numpy()
    else:
        dist, ind = est.kneighbors(Xq, m)
        ind_only = est.kneighbors(Xq, m, return_distance=False)
    st = est.stats()
    n = len(Xq)
    assert st[1 if path == "engine" else 2] == n, (path, st.tolist())
    assert ind.dtype == np.int64 and dist.dtype == np.float64 and ind.shape == (n, m)
    assert np.array_equal(ind, ri), f"{path} m={m}: indices differ on {(ind != ri).any(1).sum()} rows"
    assert np.array_equal(dist, rd), f"{path} m={m}: distances differ"
    assert np.array_equal(ind_only, ri)
    return ind


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 3, 5, 8, 9, 17, 32])
@pytest.mark.parametrize("path", ["engine", "fp64"])
def test_kneighbors_bit_exact_vs_oracle(m, path):
    """synthetic flows with exact duplicates of training rows (distance 0, ties with their twins); float64 and float32 rows,
    host arrays and CUDA tensors; with m == k the vote of y[ind] is predict's label"""
    spec = _flows_spec(3000, k=m, seed=m)
    est = from_spec(spec)
    Xq = synth.make_flows(5000, seed=m + 100, return_labels=False)
    Xq[:300] = spec["fit_X"][:300]
    ind = _check(est, spec, Xq, m, path)
    assert np.array_equal(_vote(spec["y"], ind, len(spec["classes"])), est.predict_indices(Xq))
    _check(est, spec, Xq.astype(np.float32), m, path)
    _check(est, spec, Xq, m, path, torch_in=True)
    _check(est, spec, Xq.astype(np.float32), m, path, torch_in=True)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [33, 64])
def test_kneighbors_beyond_engine_takes_fp64_kernel(m):
    """more than 32 neighbours: the engine keeps at most 32, so every row goes to the fp64 kernel even on a large batch"""
    spec = _flows_spec(3000, k=5, seed=1)
    est = from_spec(spec)
    Xq = synth.make_flows(6000, seed=7, return_labels=False)
    Xq[:200] = spec["fit_X"][:200]
    dist, ind = est.kneighbors(Xq, m)
    assert est.stats()[2] == len(Xq) and est.stats()[1] == 0
    rd, ri = kno.kneighbors(spec, Xq, m)
    assert np.array_equal(ind, ri) and np.array_equal(dist, rd)
    with pytest.raises(ValueError):   # the engine forced but not usable at this m
        _force(est, 2).kneighbors(Xq, m)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 5, 9])
def test_kneighbors_lattice_ties(m):
    """on a lattice most rows tie at the m-th distance: they are re-run by the index-order kernel (stats[7]), and the result
    equals both the CPU definition and sklearn brute (sorted canonically)"""
    spec, q = _lattice(nt=900, nq=5000)
    est = _force(from_spec(dict(spec, k=5)), 2)
    before = est.stats()[7]
    dist, ind = est.kneighbors(q, m)
    assert est.stats()[7] > before
    rd, ri = kno.kneighbors(spec, q, m)
    assert np.array_equal(ind, ri) and np.array_equal(dist, rd)
    from sklearn.neighbors import KNeighborsClassifier
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=1):
        sd, si = kno.canonical(*KNeighborsClassifier(m, algorithm="brute").fit(spec["fit_X"], spec["y"]).kneighbors(q))
    assert np.array_equal(ind, si) and np.array_equal(dist, sd)


@pytest.mark.gpu
@pytest.mark.parametrize("nt,nq,m", [(20000, 20000, 5), (5000, 9000, 17), (130, 5000, 3)])
def test_kneighbors_pruned_equals_unpruned(nt, nq, m):
    spec = _flows_spec(nt, k=5, seed=nt + 3)
    Xq = synth.make_flows(nq, seed=nq + 7, return_labels=False)
    Xq[:100] = spec["fit_X"][:100]
    rd, ri = kno.kneighbors(spec, Xq, m)
    for off in (0, 1):
        est = _force(from_spec(spec), 2)
        est.set_option(_lib.OPT_KNN_PRUNE, off)
        dist, ind = est.kneighbors(Xq, m)
        assert est.stats()[1] == nq
        assert np.array_equal(ind, ri) and np.array_equal(dist, rd), f"prune_off={off}"


@pytest.mark.gpu
def test_kneighbors_large_model_without_tile_table():
    """270 000 training rows: beyond the tile-by-tile neighbour table, the producer walks outwards in kd order"""
    nt, nq, m = 270_000, 4096, 7
    spec = _flows_spec(nt, k=5, seed=99)
    rng = np.random.default_rng(123)
    spots = spec["fit_X"][rng.choice(nt, 16, replace=False)]
    Xq = (spots[:, None, :] * (1.0 + 1e-3 * rng.standard_normal((16, 256, 12))) + 1e-2 * rng.standard_normal((16, 256, 12))).reshape(nq, 12)
    Xq[::256] = spots
    est = _force(from_spec(spec), 2)
    dist, ind = est.kneighbors(Xq, m)
    assert est.stats()[1] == nq
    rd, ri = kno.kneighbors(spec, Xq, m)
    assert np.array_equal(ind, ri) and np.array_equal(dist, rd)


@pytest.mark.gpu
def test_kneighbors_reference_model(golden, specs):
    """all 7 653 bundled rows through the engine: equal to the CPU definition, distances equal to sklearn kd_tree's on the
    rebuilt reference model, and the vote of y[ind] is predict's label (engine and fp64 kernel)"""
    from sk_rebuild import sklearn_from_spec
    spec, X = specs["knn"], np.ascontiguousarray(golden["X"])
    k = spec["k"]
    est = _force(from_spec(spec), 2)
    dist, ind = est.kneighbors(X)
    assert est.stats()[1] == len(X)
    rd, ri = kno.kneighbors(spec, X, k)
    assert np.array_equal(ind, ri) and np.array_equal(dist, rd)
    sd, _ = kno.canonical(*sklearn_from_spec(spec, knn_algorithm="kd_tree").kneighbors(X))
    assert np.array_equal(dist, sd)
    lab = est.predict_indices(X)
    assert np.array_equal(_vote(spec["y"], ind, len(spec["classes"])), lab)
    assert np.array_equal(lab, golden["knn.expected_label"])
    d1, i1 = _force(est, 1).kneighbors(X)
    assert est.stats()[2] == len(X)
    assert np.array_equal(i1, ind) and np.array_equal(d1, dist)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 4, 5])
def test_kneighbors_without_X_excludes_self(m):
    """X=None: sklearn's rule on the (m + 1)-neighbour result of fit_X -- including rows with more exact duplicates than
    neighbours, where the row's own index is not kept and the first column goes instead"""
    rng = np.random.default_rng(m)
    base = rng.normal(0, 50.0, (5000, 12))
    base[100:110] = base[100]          # ten copies of one row
    base[200:203] = base[200]          # three copies
    y = rng.integers(0, 4, len(base)).astype(np.int32)
    spec = dict(kind="knn", fit_X=base, y=y, k=5, classes=np.arange(4), n_features=12)
    est = from_spec(spec)
    rd, ri = kno.exclude_self(*kno.kneighbors(spec, base, m + 1))
    for path in ("engine", "fp64"):
        dist, ind = _force(est, 2 if path == "engine" else 1).kneighbors(n_neighbors=m)
        assert ind.shape == (len(base), m)
        assert np.array_equal(ind, ri) and np.array_equal(dist, rd), path
        assert np.array_equal(_force(est, 0).kneighbors(return_distance=False, n_neighbors=m), ri)
    assert not (ri[100:110] == np.arange(100, 110)[:, None]).any()


@pytest.mark.gpu
def test_kneighbors_full_size_bench_workload():
    """the bench KNN workload (50k training rows, k = 5) on 10M device rows: a strided sample of 2 000 rows equals the CPU
    definition, and the vote of y[ind] equals predict on every row"""
    import torch
    import bench
    w = bench.build_workload("knn")
    spec = w["spec"]
    est = from_spec(spec)
    n = w["rows"]
    Xd = bench.synth_rows(n, w["d"], seed=3, device=torch.device("cuda", 0))
    dist, ind = est.kneighbors(Xd)
    lab = est.predict_indices(Xd)
    est.sync_check()
    y = torch.from_numpy(np.ascontiguousarray(spec["y"], np.int64)).cuda()
    cnt = torch.zeros((n, len(spec["classes"])), dtype=torch.int32, device="cuda")
    cnt.scatter_add_(1, y[ind], torch.ones_like(ind, dtype=torch.int32))
    assert torch.equal(cnt.argmax(1).to(torch.int32), lab)   # torch's argmax returns the first maximum
    sel = np.arange(0, n, n // 2000)[:2000] + 17
    Xs = Xd[torch.from_numpy(sel).cuda()].cpu().numpy()
    rd, ri = kno.kneighbors(spec, Xs, spec["k"])
    assert np.array_equal(ind[torch.from_numpy(sel).cuda()].cpu().numpy(), ri)
    assert np.array_equal(dist[torch.from_numpy(sel).cuda()].cpu().numpy(), rd)


@pytest.mark.gpu
def test_kneighbors_errors():
    from traffic_classifier_sdn_b200 import KNeighborsClassifier, NotFittedError
    spec = _flows_spec(100, k=5, seed=3)
    est = from_spec(spec)
    X = synth.make_flows(10, seed=4, return_labels=False)
    with pytest.raises(ValueError, match="Expected n_neighbors > 0"):
        est.kneighbors(X, 0)
    with pytest.raises(ValueError, match="n_neighbors <= n_samples_fit"):
        est.kneighbors(X, 101)
    with pytest.raises(ValueError, match="n_neighbors < n_samples_fit"):
        est.kneighbors(None, 100)
    big = from_spec(_flows_spec(200, k=5, seed=3))
    with pytest.raises(ValueError, match="at most 64"):
        big.kneighbors(X, 65)
    with pytest.raises(ValueError, match="at most 64"):
        big.kneighbors(None, 64)
    with pytest.raises(TypeError):
        est.kneighbors(X, 3.0)
    bad = X.copy()
    bad[3, 2] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        est.kneighbors(bad, 3)
    with pytest.raises(ValueError, match="features"):
        est.kneighbors(X[:, :5], 3)
    with pytest.raises(NotFittedError):
        KNeighborsClassifier(5).kneighbors(X)
