"""GPU parity tests (run on an H100): the CUDA path, called through the C ABI, against
  (a) tests/golden/bundled.*.npz -- sklearn's answers for the reference's six pickles on its bundled rows,
  (b) the CPU oracle (oracle/tcsdn_oracle.c) on seeded inputs and edge cases,
  (c) live scikit-learn (installed on the box; the library the reference calls) on fresh fits,
  (d) size-independent properties at BASELINE sizes.
Bars: class indices bit-exact everywhere; RandomForest probabilities and KNN votes bit-exact; LR / NB /
KMeans scores <= 1e-11 of the row's largest score (fp64, FMA vs
numpy association); SVC decision values <= 1e-9 absolute with the fp64 kernel.
"""

import numpy as np
import pytest

import oracle
from conftest import KINDS
from sk_rebuild import quiet
from traffic_classifier_sdn_b200 import _lib, from_sklearn, from_spec, synth

pytestmark = pytest.mark.gpu

SCORE_TOL = {"linear": 1e-12, "gnb": 1e-11, "kmeans": 1e-11, "knn": 0.0, "svc": 1e-9, "forest": 0.0}


def rel_err(a, b):
    """max |a-b| relative to the largest score of the same row (scores of one row share their cancellation scale)"""
    if not a.size:
        return 0.0
    scale = np.maximum(1.0, np.max(np.abs(b), axis=1, keepdims=True))
    return float(np.max(np.abs(a - b) / scale))


@pytest.fixture(scope="module")
def models(specs):
    """this module pins the fp64 CUDA-core kernels (engine option 1); tests/test_engine_gpu.py covers the
    tensor-core engine that large KNN / SVC batches take by default"""
    out = {k: from_spec(specs[k]) for k in KINDS}
    for k in ("knn", "svc"):
        out[k].set_option(_lib.OPT_ENGINE, 1)
    return out


# ------------------------------------------------------------------ (a) golden vectors
@pytest.mark.parametrize("kind", KINDS)
def test_golden_labels_and_scores_f64_host(golden, specs, models, kind):
    X = golden["X"]
    idx, sc = models[kind]._run(X, True)
    assert np.array_equal(idx, golden[f"{kind}.expected_label"])
    exp = golden[f"{kind}.expected_score"]
    if kind == "knn":
        assert np.array_equal(np.rint(sc * 5).astype(np.uint8), exp)
    elif kind == "forest":
        assert np.array_equal(sc, exp)
    elif kind == "kmeans":
        d2 = sc + np.einsum("ij,ij->i", X, X)[:, None]
        assert np.max(np.abs(d2 - exp ** 2) / np.maximum(1.0, exp ** 2)) < 1e-6
    elif kind == "svc":
        assert np.max(np.abs(sc - exp)) < 1e-9
    else:
        assert rel_err(sc, exp) < SCORE_TOL[kind]
    # and the public sklearn-like surface
    pred = models[kind].predict(X[:50])
    if kind == "kmeans":
        assert pred.dtype == np.int32 and np.array_equal(pred, idx[:50])
    else:
        assert np.array_equal(pred, np.asarray(specs[kind]["classes"])[idx[:50]])


def test_svc_decision_function_ovr(golden, models):
    ovr = models["svc"].decision_function(golden["X"])
    assert np.max(np.abs(ovr - golden["svc.expected_ovr"])) < 1e-9


def test_reference_call_pattern_one_row_list(golden, specs, models):
    """traffic_classifier.py:106 -- predict(features.tolist()) with a single 1x12 row of Python floats."""
    for kind in KINDS:
        for i in (0, 1234, 7652):
            row = golden["X"][i].reshape(1, -1).tolist()
            lab = models[kind].predict(row)
            exp = golden[f"{kind}.expected_label"][i]
            assert lab.shape == (1,)
            assert lab[0] == (exp if kind == "kmeans" else specs[kind]["classes"][exp])


# ------------------------------------------------------------------ (b) oracle, dtypes, locations, edges
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [1, 31, 255, 256, 257, 1024, 1025, 3000])
def test_ragged_sizes_f32_host_vs_oracle(specs, models, kind, n):
    X32 = synth.make_flows(n, seed=100 + n, dtype=np.float32, return_labels=False)
    idx, sc = models[kind]._run(X32, True)
    ref_idx, ref_sc = oracle.predict(specs[kind], X32.astype(np.float64))
    assert np.array_equal(idx, ref_idx)
    if SCORE_TOL[kind] == 0.0:
        assert np.array_equal(sc, ref_sc)
    elif kind == "svc":
        assert np.max(np.abs(sc - ref_sc)) < 1e-9
    else:
        assert rel_err(sc, ref_sc) < SCORE_TOL[kind]


@pytest.mark.parametrize("kind", KINDS)
def test_device_pointers_match_host_pointers(specs, models, kind):
    import torch
    X = synth.make_flows(5000, seed=5, return_labels=False)
    for dt in (np.float32, np.float64):
        Xh = X.astype(dt)
        idx_h, sc_h = models[kind]._run(Xh, True)
        idx_d, sc_d = models[kind]._run(torch.from_numpy(Xh).cuda(), True)
        models[kind].sync_check()
        assert idx_d.is_cuda and np.array_equal(idx_d.cpu().numpy(), idx_h)
        assert np.array_equal(sc_d.cpu().numpy(), sc_h)


def test_empty_batch(models):
    for kind in KINDS:
        out = models[kind].predict(np.empty((0, 12)))
        assert out.shape == (0,)


def test_wrong_feature_count_and_nonfinite_raise(models):
    for kind in KINDS:
        with pytest.raises(ValueError, match="features"):
            models[kind].predict(np.zeros((3, 11)))
        bad = np.ones((700, 12))
        bad[513, 4] = np.nan
        with pytest.raises(ValueError, match="NaN|infinity"):
            models[kind].predict(bad)
        bad[513, 4] = np.inf
        with pytest.raises(ValueError, match="NaN|infinity"):
            models[kind].predict(bad.astype(np.float32))
        # -inf in every feature position: in the forest a -inf used to satisfy `v <= -inf` at a leaf / halt node and run the
        # walk out of its group (sticky illegal address or an endless spin); it must raise like the others, in both dtypes,
        # on the shared-memory walker and -- huge float64 values overflow to -inf in the float32 cast -- through the cast
        for col in (0, 6, 11):
            bad = np.ones((1500, 12))
            bad[1027, col] = -np.inf
            with pytest.raises(ValueError, match="NaN|infinity"):
                models[kind].predict(bad)
            with pytest.raises(ValueError, match="NaN|infinity"):
                models[kind].predict(bad.astype(np.float32))
        if kind == "forest":
            bad = np.ones((300, 12))
            bad[7, 3] = -1e300                    # finite float64, -inf after sklearn's cast to float32: sklearn raises too
            with pytest.raises(ValueError, match="NaN|infinity"):
                models[kind].predict(bad)
        with pytest.raises(ValueError, match="2D"):
            models[kind].predict(np.zeros(12))
        assert models[kind].predict(np.ones((2, 12))).shape == (2,)  # still usable afterwards


def test_unaligned_host_pointer_and_chunked_pipeline(specs, models):
    X = synth.make_flows(20000, seed=9, dtype=np.float32, return_labels=False)
    buf = np.empty(X.size + 1, np.float32)
    view = buf[1:].reshape(X.shape)   # 4-byte aligned only
    view[:] = X
    for kind in ("linear", "gnb", "forest"):
        ref = models[kind]._run(X, False)[0]
        assert np.array_equal(models[kind]._run(view, False)[0], ref)
        models[kind].set_option(_lib.OPT_CHUNK_ROWS, 3000)   # 7 chunks through the double-buffered pipeline
        assert np.array_equal(models[kind]._run(X, False)[0], ref)
        models[kind].set_option(_lib.OPT_CHUNK_ROWS, 0)


def test_inputs_not_modified_and_outputs_fresh(models):
    X = synth.make_flows(300, seed=2, return_labels=False)
    X0 = X.copy()
    a = models["forest"].predict(X)
    b = models["forest"].predict(X)
    assert np.array_equal(X, X0) and a is not b and np.array_equal(a, b)


def test_not_fitted_raises():
    from traffic_classifier_sdn_b200 import GaussianNB, NotFittedError
    with pytest.raises(NotFittedError):
        GaussianNB().predict(np.zeros((1, 12)))


# ------------------------------------------------------------------ generic shapes (d, classes outside the fast path)
def test_scorers_generic_shapes_vs_oracle():
    rng = np.random.default_rng(0)
    for d, R in ((5, 3), (12, 11), (20, 4), (8, 1), (12, 1), (16, 8), (4, 2)):
        X = rng.normal(0, 30, (2000, d))
        lin = dict(kind="linear", coef=rng.normal(0, 1, (R, d)), intercept=rng.normal(0, 1, R),
                   classes=np.arange(max(R, 2)), n_features=d)
        nb = dict(kind="gnb", theta=rng.normal(0, 20, (max(R, 2), d)), var=rng.random((max(R, 2), d)) * 50 + 0.1,
                  class_prior=np.full(max(R, 2), 1.0 / max(R, 2)), classes=np.arange(max(R, 2)), n_features=d)
        km = dict(kind="kmeans", centers=rng.normal(0, 30, (max(R, 2), d)), classes=np.arange(max(R, 2)), n_features=d)
        for spec in (lin, nb, km):
            est = from_spec(spec)
            for Xi in (X, X.astype(np.float32)):
                idx, sc = est._run(Xi, True)
                ridx, rsc = oracle.predict(spec, Xi.astype(np.float64))
                assert np.array_equal(idx, ridx), (spec["kind"], d, R)
                assert rel_err(sc, rsc) < 1e-11


# ------------------------------------------------------------------ forest: groups, oversize trees, impure leaves, fp32 rounding
@pytest.mark.parametrize("cfg", [dict(n_trees=40, depth=11, full=True), dict(n_trees=3, depth=15, full=True),
                                 dict(n_trees=100, depth=16, full=False), dict(n_trees=7, depth=3, full=True)])
def test_forest_synthetic_vs_oracle(cfg):
    spec = synth.random_forest_spec(seed=4, impure=0.2, **cfg)
    est = from_spec(spec)
    X = synth.make_flows(6000, seed=8, return_labels=False)
    X[::7] += 1e-6   # values that are not fp32-representable: exercises the float32 cast + floor32 thresholds
    idx, pr = est._run(X, True)
    ridx, rpr = oracle.forest(spec, X)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)
    idx32, pr32 = est._run(X.astype(np.float32), True)
    assert np.array_equal(pr32, rpr)
    # non-finite rows on every walker (shared-memory groups, trees walked in L2/HBM, both CTA shapes): the call raises
    # and the handle stays usable
    for bad_value in (-np.inf, np.inf, np.nan):
        Xb = X[:3000].copy()
        Xb[1234, 5] = bad_value
        with pytest.raises(ValueError, match="NaN|infinity"):
            est.predict(Xb)
    assert np.array_equal(est.predict_indices(X), ridx)


def test_forest_threshold_boundary_values():
    """rows sitting exactly on thresholds and one ulp either side (in fp32) go the way sklearn sends them"""
    spec = synth.random_forest_spec(n_trees=5, depth=6, seed=1, full=True, impure=0.3)
    thr = spec["threshold"][spec["left"] >= 0]
    f = spec["feature"][spec["left"] >= 0]
    rows = []
    for t, j in zip(thr[:150], f[:150]):
        for v in (np.float32(t), np.nextafter(np.float32(t), np.float32(np.inf)), np.nextafter(np.float32(t), np.float32(-np.inf)), t):
            r = np.zeros(12)
            r[j] = v
            rows.append(r)
    X = np.asarray(rows)
    est = from_spec(spec)
    idx, pr = est._run(X, True)
    ridx, rpr = oracle.forest(spec, X)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)


# ------------------------------------------------------------------ knn: ties
def test_knn_lattice_ties_match_sklearn_heap_semantics():
    rng = np.random.default_rng(7)
    tr = np.floor(rng.random((900, 4)) * 3)
    y = rng.integers(0, 5, 900).astype(np.int32)
    q = np.floor(rng.random((3000, 4)) * 3)
    spec = dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(5), n_features=4)
    est = from_spec(spec)
    idx, pr = est._run(q, True)
    ridx, rpr = oracle.knn(spec, q)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)
    from sklearn.neighbors import KNeighborsClassifier
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=1):
        sk = KNeighborsClassifier(5, algorithm="brute").fit(tr, y)
        assert np.array_equal(pr, sk.predict_proba(q))


@pytest.mark.parametrize("k", [1, 3, 5, 17])
def test_knn_k_values_vs_oracle(k):
    Xt, yt = synth.make_flows(3000, seed=21)
    Xq = synth.make_flows(1500, seed=22, return_labels=False)
    Xq[:200] = Xt[:200]  # exact duplicates of training rows
    spec = dict(kind="knn", fit_X=Xt, y=yt, k=k, classes=synth.CLASSES, n_features=12)
    est = from_spec(spec)
    idx, pr = est._run(Xq, True)
    ridx, rpr = oracle.knn(spec, Xq)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)


# ------------------------------------------------------------------ (c) fresh fits vs live scikit-learn
def test_fresh_fits_on_bundled_rows_vs_sklearn(golden):
    """notebook recipe (SURVEY 8c): train_test_split(test_size=0.5, random_state=101), default constructors"""
    from sklearn.cluster import KMeans
    from sklearn.ensemble import RandomForestClassifier
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import train_test_split
    from sklearn.naive_bayes import GaussianNB
    from sklearn.neighbors import KNeighborsClassifier
    from sklearn.svm import SVC
    from threadpoolctl import threadpool_limits
    X, y = golden["X"], golden["y"]
    Xtr, Xte, ytr, yte = train_test_split(X, y, test_size=0.5, random_state=101)
    fits = [quiet(LogisticRegression().fit, Xtr, ytr), GaussianNB().fit(Xtr, ytr),
            KMeans(5, n_init=3, random_state=0).fit(Xtr), KNeighborsClassifier(algorithm="brute").fit(Xtr, ytr),
            SVC().fit(Xtr, ytr), RandomForestClassifier(random_state=0).fit(Xtr, ytr)]
    for sk in fits:
        est = from_sklearn(sk)
        with threadpool_limits(limits=1):
            exp = quiet(sk.predict, X)
        got = est.predict(X)
        assert np.array_equal(got, exp), type(sk).__name__
        if hasattr(sk, "predict_proba") and type(sk).__name__ in ("RandomForestClassifier", "KNeighborsClassifier"):
            with threadpool_limits(limits=1):
                assert np.array_equal(est.predict_proba(X), quiet(sk.predict_proba, X))
    assert est.score(Xte, yte) > 0.99  # the forest, like notebook cell 17


def test_estimator_fit_route(golden):
    from traffic_classifier_sdn_b200 import GaussianNB, RandomForestClassifier
    X, y = golden["X"], golden["y"]
    nb = GaussianNB().fit(X, y)
    assert nb.score(X, y) > 0.95 and list(nb.classes_) == sorted(set(y))
    rf = RandomForestClassifier(n_estimators=10, random_state=0).fit(X, y)
    assert rf.predict_proba(X[:10]).shape == (10, 5)


# ------------------------------------------------------------------ (d) BASELINE-size properties
def test_large_batch_properties_scorers_and_forest(specs, models):
    """2M rows: permutation equivariance, agreement between one big launch and 16 slices, oracle on a sample."""
    import torch
    n = 2_000_000
    base = synth.make_flows(250_000, seed=77, dtype=np.float32, return_labels=False)
    g = torch.Generator(device="cpu").manual_seed(1)
    pick = torch.randint(0, len(base), (n,), generator=g)
    X = torch.from_numpy(base)[pick].cuda()
    perm = torch.randperm(n, generator=g).cuda()
    for kind in ("linear", "gnb", "kmeans", "forest"):
        full = models[kind].predict_indices(X)
        permuted = models[kind].predict_indices(X[perm].contiguous())
        assert torch.equal(full[perm], permuted)
        parts = torch.cat([models[kind].predict_indices(c.contiguous()) for c in X.chunk(16)])
        assert torch.equal(full, parts)
        models[kind].sync_check()
        s = slice(0, n, 997)
        ref = oracle.predict(specs[kind], X[s].cpu().numpy().astype(np.float64), want_scores=False)[0]
        assert np.array_equal(full[s].cpu().numpy(), ref)
        # label histogram is a checksum of checksums: equal to the histogram of the base rows weighted by picks
        base_lab = oracle.predict(specs[kind], base.astype(np.float64), want_scores=False)[0]
        exp_hist = np.bincount(base_lab[pick.numpy()], minlength=8)
        assert np.array_equal(np.bincount(full.cpu().numpy(), minlength=8), exp_hist)


# ------------------------------------------------------------------ N1: feature derivation on device
def test_flow_update_kernel_matches_oracle():
    """tcsdn_flow_update against the ORACLE's restatement of Flow.updateforward/updatereverse (traffic_classifier.py:63-96),
    sample by sample over six polls with repeated timestamps (the `!=` guards) and idle directions"""
    import torch
    from traffic_classifier_sdn_b200 import flows
    rng = np.random.default_rng(5)
    n = 3000
    state = np.zeros((n, flows.STATE))
    t0 = rng.integers(1000, 2000, n).astype(float)
    state[:, flows.T0] = t0
    state[:, flows.FWD + 8] = t0
    state[:, flows.REV + 8] = t0
    state[:, flows.FWD + 0] = rng.integers(0, 50, n)
    state[:, flows.FWD + 1] = state[:, flows.FWD + 0] * 100
    ref = state.copy()
    dstate = torch.from_numpy(state).cuda()
    lib = _lib.load()
    now = t0.copy()
    for step in range(6):
        now = now + rng.integers(0, 3, n)   # repeated timestamps hit the `!=` guards
        direction = rng.integers(0, 3, n).astype(np.uint8)
        dp = rng.integers(0, 40, n) * (rng.random(n) < 0.7)
        cum_p = np.where(direction == 0, ref[:, flows.FWD], ref[:, flows.REV]) + dp
        cum_b = np.where(direction == 0, ref[:, flows.FWD + 1], ref[:, flows.REV + 1]) + dp * rng.integers(60, 1500, n)
        for i in range(n):
            if direction[i] < 2:
                o = flows.REV if direction[i] else flows.FWD
                ref[i, o:o + 9] = oracle.flow_update(ref[i, o:o + 9], ref[i, flows.T0], cum_p[i], cum_b[i], now[i])
        feats = torch.empty((n, 12), dtype=torch.float64, device="cuda")
        args = [torch.from_numpy(a.astype(np.float64)).cuda() for a in (cum_p, cum_b, now)]
        dd = torch.from_numpy(direction).cuda()
        _lib.check(lib.tcsdn_flow_update(dstate.data_ptr(), args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(),
                                         dd.data_ptr(), n, feats.data_ptr(), _lib.F64,
                                         torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert np.array_equal(dstate.cpu().numpy(), ref)
        assert np.array_equal(feats.cpu().numpy(), ref[:, flows.FEATURE_COLUMNS])


def test_device_flow_table_equals_host_table(specs):
    """the CLI's default table (state in HBM, features derived by tcsdn_flow_update) against the host mirror of the
    reference's run_ryu / Flow (tests/test_host.py checks that mirror against the reference's formulas): state, features
    and ACTIVE/INACTIVE columns identical after every line, and predict on the device features equals predict on the
    host features"""
    from test_host import _monitor_log
    from traffic_classifier_sdn_b200 import flows
    host, dev = flows.FlowTable(), flows.DeviceFlowTable()
    est = from_spec(specs["forest"])
    for k, line in enumerate(_monitor_log(np.random.default_rng(2), n_flows=40, polls=12)):
        rec = flows.parse_monitor_line(line)
        if rec is None:
            continue
        host.ingest(rec); dev.ingest(rec)
        if k % 37 == 0 or k < 5:
            assert np.array_equal(dev.state, host.state)
            assert np.array_equal(dev.features(), host.features())
            assert list(dev.rows()) == list(host.rows())
    assert np.array_equal(dev.state, host.state) and list(dev.rows()) == list(host.rows())
    a = est.predict_indices(dev.features_device()).cpu().numpy()
    assert np.array_equal(a, est.predict_indices(host.features()))
    assert np.array_equal(a, oracle.predict(specs["forest"], host.features(), want_scores=False)[0])


def test_synthetic_rows_through_the_flow_kernel_equal_the_closed_form():
    """synth.make_flows_device pushes cumulative counters through tcsdn_flow_update poll by poll (SURVEY 8d); the rows must
    be bit-identical to the closed form the CPU tests use"""
    from traffic_classifier_sdn_b200 import synth
    for d, dt in ((12, np.float64), (8, np.float32), (12, np.float32)):
        ref = synth.make_flows(20_000, seed=11, d=d, dtype=dt, return_labels=False)
        got = synth.make_flows_device(20_000, seed=11, d=d, dtype="float32" if dt == np.float32 else "float64").cpu().numpy()
        assert got.dtype == ref.dtype and np.array_equal(got, ref)


# ------------------------------------------------------------------ the CLI shim end to end (reference argv words)
def test_cli_replays_a_monitor_log_through_the_gpu(tmp_path, golden, specs, capsys):
    """`python -m ...cli gaussiannb --monitor-cmd 'cat log' --models DIR`: model files are read exactly like the reference
    reads models/<Name> (pickles), the monitor's stdout lines are parsed like run_ryu does, every report classifies all
    flows with one GPU predict.  (Ryu itself is not needed: the monitor command is replaced by a recorded log.)"""
    import pickle
    from sk_rebuild import sklearn_from_spec
    from test_host import _monitor_log
    from traffic_classifier_sdn_b200 import cli, flows, modelio
    models = tmp_path / "models"
    models.mkdir()
    for word, fname in modelio.MODEL_FILES.items():
        kind = {"logistic": "linear", "kmeans": "kmeans", "svm": "svc", "kneighbors": "knn", "Randomforest": "forest",
                "gaussiannb": "gnb"}[word]
        with open(models / fname, "wb") as fh:
            pickle.dump(sklearn_from_spec(specs[kind], knn_algorithm="kd_tree"), fh)
    log = tmp_path / "monitor.log"
    lines = _monitor_log(np.random.default_rng(5), n_flows=7, polls=21)
    log.write_bytes(b"".join(lines))
    table = flows.FlowTable()
    for ln in lines:
        rec = flows.parse_monitor_line(ln)
        if rec is not None:
            table.ingest(rec)
    for word in ("gaussiannb", "Randomforest", "kmeans", "knearest", "supervised", "svm"):
        assert cli.main([word, "--monitor-cmd", f"cat {log}", "--models", str(models), "--every", "1"]) == 0
        out = capsys.readouterr().out
        assert out.count("Flow ID") >= 2 and "Traffic Type" in out
        kind = {"gaussiannb": "gnb", "Randomforest": "forest", "kmeans": "kmeans", "knearest": "knn", "supervised": "linear",
                "svm": "svc"}[word]
        exp_idx = oracle.predict(specs[kind], table.features(), want_scores=False)[0]
        exp = [cli.INT_LABELS[int(i)] if kind == "kmeans" else str(np.asarray(specs[kind]["classes"])[i]) for i in exp_idx]
        final_table = out[out.rstrip().rfind("Flow ID"):]
        got = [row.split("|")[4].strip() for row in final_table.splitlines() if row.startswith("|") and "Flow ID" not in row]
        assert got == exp, (word, got, exp)   # --every 1: the last report is printed at the last data line = final state


# ------------------------------------------------------------------ GaussianNB: certified fp32 pre-pass
def test_gnb_fp32_prepass_is_certified_or_refined(specs, models):
    """float32 rows, labels only: the kernel evaluates in fp32 with an error bound and re-runs uncertified rows in fp64.
    Labels must equal the fp64 kernel's on every row -- bulk rows, exact ties and near-ties -- and the counter of
    refined rows (stats[6]) must show that both routes were taken."""
    import torch
    from traffic_classifier_sdn_b200 import _lib
    n = 1_000_000
    X = torch.from_numpy(synth.make_flows(n, seed=123, dtype=np.float32, return_labels=False)).cuda()
    fast = from_spec(specs["gnb"])
    slow = from_spec(specs["gnb"])
    slow.set_option(_lib.OPT_ENGINE, 1)                       # fp64 only
    a, b = fast.predict_indices(X), slow.predict_indices(X)
    assert torch.equal(a, b)
    refined = int(fast.stats()[6])
    assert int(slow.stats()[6]) == 0 and refined < 0.05 * n   # the pre-pass certifies the bulk
    print(f"gnb pre-pass: {refined} of {n} rows refined in fp64")
    # exact ties (two identical classes) and near ties (class 2 = class 0 shifted by a few ulps of fp32)
    d, rng = 8, np.random.default_rng(5)
    theta = rng.uniform(1.0, 1e4, (3, d))
    theta[1] = theta[0]
    theta[2] = theta[0] * (1.0 + 3e-8)
    var = np.tile(rng.uniform(1.0, 1e3, (1, d)), (3, 1))
    spec = dict(kind="gnb", theta=theta, var=var, class_prior=np.full(3, 1 / 3), classes=np.arange(3), n_features=d)
    Xt = (theta[0] + rng.normal(0, 30.0, (200_000, d))).astype(np.float32)
    est = from_spec(spec)
    got = est.predict_indices(torch.from_numpy(Xt).cuda()).cpu().numpy()
    ref = oracle.predict(spec, Xt.astype(np.float64), want_scores=False)[0]
    assert np.array_equal(got, ref)
    assert int(est.stats()[6]) > 0.5 * len(Xt)                # nothing here can be certified in fp32
    assert set(np.unique(ref)) <= {0, 2}                      # class 1 never beats its identical twin (first maximum)
