"""GPU: every kernel instantiation and launch option a real call can reach, against the CPU oracle.

The other GPU modules pin the answers of each estimator; this one walks the launch configurations underneath them, because
a kernel can be right in one template instantiation and wrong in its neighbour:
  1. the streaming scorers: dtype x D in {4, 8, 12, 16} x R in 1..8 x kind x CTA shape (OPT_SCORER_SHAPE 1 / 2 / 3) x with /
     without scores, with an exact tie designed into every model (first-max / first-min rule) and batches that wrap the
     mbarrier ring and end in a ragged tile;
  2. the GaussianNB fp32 pre-pass at the edge of its error bound, at every D;
  3. the bench models just above the batch size where the default CTA shapes take over from the small-batch shape;
  4. the forest walkers: every CTA shape, coherence sort on / off, shared-memory ceilings, padded feature rows, one-leaf trees;
  5. the distance engine: KNN flush cadence, shared / local heap boundary, feature counts other than 4 and 12;
  6. the host pipeline's chunk loop, device rows aligned to 4 bytes only, concurrent host-pointer predicts on one handle;
  7. two GPUs in one process.
Batch sizes follow the device (SM count, shared memory), not a fixed GPU.
"""
import ctypes as C
import threading

import numpy as np
import pytest

import kneighbors_oracle as kno
import oracle
from conftest import KINDS
from test_engine_gpu import _check_svc, _libsvm_signs, _svc_spec
from traffic_classifier_sdn_b200 import _lib, from_spec, synth

pytestmark = pytest.mark.gpu

SCORER_SHAPES = {1: (128, 4), 2: (256, 2), 3: (128, 2)}   # OPT_SCORER_SHAPE -> threads x rows per thread (csrc/scorers.cu)
SCORER_STAGES = 3                                          # csrc/scorers.cu kStages
SCORE_TOL = 1e-11                                          # of the row's largest score, as in test_parity_gpu.py


def _sm_count():
    n = C.c_int32(0)
    _lib.check(_lib.load().tcsdn_device_sm_count(C.byref(n)))
    return int(n.value)


def _scorer_per_sm(dtype):
    """CTAs per SM of scorer shapes 1 and 2 (shape 3 runs one more), as launch_tiled chooses them"""
    return 3 if np.dtype(dtype) == np.float32 else 2


def _scorer_n(dtype):
    """every CTA of every shape runs at least kStages + 2 tiles (the mbarrier parity wraps) and the last tile is ragged"""
    sms, p = _sm_count(), _scorer_per_sm(dtype)
    most = max(sms * (p + (s == 3)) * t * r for s, (t, r) in SCORER_SHAPES.items())
    return (SCORER_STAGES + 2) * most + 137


def _small_batch_limit(dtype):
    """the smallest batch launch_tiled no longer sends to the small-batch shape 3: 16 tiles of 512 rows per CTA"""
    return 16 * _sm_count() * _scorer_per_sm(dtype) * 512


def _force(est, mode):
    est.set_option(_lib.OPT_ENGINE, mode)
    return est


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------ 1. scorer instantiation matrix
def _scorer_rows_host(n, D, seed):
    """Gaussian rows, a quarter of them on the integer lattice [-8, 8]^D (exact scores for integer models, exact zeros in
    the last feature for the designed ties) and a few scaled by 1e3"""
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 30.0, (n, D))
    lat = rng.random(n) < 0.25
    X[lat] = rng.integers(-8, 9, (int(lat.sum()), D))
    X[lat & (rng.random(n) < 0.4), D - 1] = 0.0
    X[rng.random(n) < 0.03] *= 1e3
    return X


def _scorer_spec(kind, R, D, rng):
    """-> (spec, tied class pairs).  R = 1: linear is a binary LR with integer coefficients (scores on lattice rows are
    integers, exactly 0 on many); gnb / kmeans have one class.  R >= 2: class a is made to win near the origin, where the
    lattice rows are, and class b is its mirror image in the last feature (the same score, exactly, where x[D-1] == 0);
    R >= 3: one more class e is an exact copy of a (a tie wherever a wins)."""
    if kind == "linear" and R == 1:
        spec = dict(kind="linear", coef=rng.integers(-3, 4, (1, D)).astype(float), intercept=rng.integers(-2, 3, 1).astype(float),
                    classes=np.arange(2), n_features=D)
        return spec, []
    if kind == "linear":
        P = dict(coef=rng.normal(0.0, 1.0, (R, D)), intercept=rng.normal(0.0, 1.0, R))
    elif kind == "gnb":
        prior = rng.random(R) + 0.5
        P = dict(theta=rng.normal(0.0, 20.0, (R, D)), var=rng.random((R, D)) * 50 + 0.1, class_prior=prior / prior.sum())
    else:
        P = dict(centers=rng.normal(0.0, 30.0, (R, D)))
    if R == 1:
        return dict(kind=kind, classes=np.arange(R), n_features=D, **P), []
    a, b = (int(v) for v in rng.choice(R, 2, replace=False))
    if kind == "linear":
        P["coef"][a] = rng.normal(0.0, 4.0, D)
        P["intercept"][a] = 20.0
        first = "coef"
    elif kind == "gnb":
        P["theta"][a] = rng.integers(-3, 4, D)
        P["var"][a] = 30.0 + 10.0 * rng.random(D)
        P["class_prior"][a] = P["class_prior"].max()
        first = "theta"
    else:
        P["centers"][a] = rng.integers(-3, 4, D)
        first = "centers"
    if kind != "linear":
        P[first][a, D - 1] = 2.5
    for v in P.values():
        v[b] = v[a]
    P[first][b, D - 1] = -P[first][a, D - 1]     # coef / theta / centre: opposite signs in the last feature
    pairs = [(a, b)]
    if R >= 3:
        e = int(rng.choice([r for r in range(R) if r not in (a, b)]))
        for v in P.values():
            v[e] = v[a]
        pairs.append((a, e))
    return dict(kind=kind, classes=np.arange(R), n_features=D, **P), pairs


@pytest.fixture(scope="module")
def scorer_rows():
    """(device rows, the same rows as float64 on the host) per (dtype, D); one (dtype, D) is kept at a time"""
    cache = {}

    def get(dtype, D):
        if (dtype, D) not in cache:
            cache.clear()
            X = _scorer_rows_host(_scorer_n(dtype), D, seed=D).astype(dtype)
            cache[(dtype, D)] = (_cuda(X), X.astype(np.float64))
        return cache[(dtype, D)]

    yield get
    cache.clear()


@pytest.mark.parametrize("kind", ["linear", "gnb", "kmeans"])
@pytest.mark.parametrize("R", list(range(1, 9)))
@pytest.mark.parametrize("D", [4, 8, 12, 16])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_scorer_instantiation_matrix(scorer_rows, dtype, D, R, kind):
    """every (dtype, D, R, kind) tiled instantiation in all three CTA shapes, with scores and labels only (float32 GaussianNB
    labels only = the certified fp32 pre-pass): labels equal the oracle on every row, scores within 1e-11 of the row's
    largest score"""
    import torch
    Xd, X64 = scorer_rows(dtype, D)
    rng = np.random.default_rng(10_000 * D + 100 * R + ("linear", "gnb", "kmeans").index(kind) + (dtype == np.float64) * 7)
    spec, pairs = _scorer_spec(kind, R, D, rng)
    ref_lab, ref_sc = oracle.predict(spec, X64)
    # the designed ties are real: on some rows the tied classes share the best score, so the first-max / first-min rule decides
    best = ref_sc.min(1) if kind == "kmeans" else ref_sc.max(1)
    for a, b in pairs:
        assert np.count_nonzero((ref_sc[:, a] == best) & (ref_sc[:, b] == best)) > 0, (a, b)
    if kind == "linear" and R == 1:
        assert np.count_nonzero(ref_sc[:, 0] == 0.0) > 0 and 0 < ref_lab.sum() < len(ref_lab)
    lab_ref_d, sc_ref_d = _cuda(ref_lab), _cuda(ref_sc)
    scale = sc_ref_d.abs().amax(1, keepdim=True).clamp_min(1.0)
    if R == 1 and kind != "gnb":
        # a single affine score has no other score to set its row's scale and can cancel to near 0 (x.c ~ ||c||^2 / 2):
        # there the two fp64 association orders differ relative to the terms they sum
        A, c0 = (spec["coef"][0], spec["intercept"][0]) if kind == "linear" else (-2.0 * spec["centers"][0], (spec["centers"][0] ** 2).sum())
        terms = Xd.double().abs() @ _cuda(np.abs(A)) + abs(float(c0))
        scale = torch.maximum(scale, terms[:, None])
    est = from_spec(spec)
    for shape in SCORER_SHAPES:
        est.set_option(_lib.OPT_SCORER_SHAPE, shape)
        lab, sc = est._run(Xd, True)
        only = est.predict_indices(Xd)
        est.sync_check()
        assert torch.equal(lab, lab_ref_d), f"shape {shape}: {int((lab != lab_ref_d).sum())} labels differ (with scores)"
        assert torch.equal(only, lab_ref_d), f"shape {shape}: {int((only != lab_ref_d).sum())} labels differ (labels only)"
        err = float(((sc - sc_ref_d).abs() / scale).max())
        assert err < SCORE_TOL, f"shape {shape}: score error {err:.3e}"


# ------------------------------------------------------------------ 2. GaussianNB fp32 pre-pass at its bound
def _flow_columns(X12, D):
    if D == 4:
        return X12[:, :4]
    if D == 8:
        return X12[:, list(synth.COLUMNS_8)]
    if D == 12:
        return X12
    return np.hstack([X12, X12[:, [1, 4, 7, 10]] * 0.5 + 1.0])


def _adversarial_gnb(D, R, rng):
    """class 0 and classes built against it, in turn: near twins theta0 (1 + k 2^-23) with k = 4, 4^2, ... (top-2 margins from
    far inside the pre-pass's error bound to outside it); a sharp class (large |theta / sigma|); a near twin with a prior of
    1e-300 (|log prior| ~ 690).  R >= 3: the last class is an exact twin of class 1 (exact ties wherever class 1 wins)."""
    theta0 = rng.uniform(1.0, 1e4, D)
    var0 = rng.uniform(1.0, 1e3, D)
    theta, var, prior = np.tile(theta0, (R, 1)), np.tile(var0, (R, 1)), np.ones(R)
    for r in range(1, R):
        kind = (r - 1) % 3
        if kind == 0:
            theta[r] = theta0 * (1.0 + 4.0 ** r * 2.0 ** -23)
        elif kind == 1:
            theta[r] = theta0 + rng.normal(0.0, 30.0, D)
            var[r] = var0 * 1e-4
        else:
            theta[r] = theta0 * (1.0 + 2.0 * 2.0 ** -23)
            prior[r] = 1e-300
    if R >= 3:
        theta[R - 1], var[R - 1], prior[R - 1] = theta[1], var[1], prior[1]
    return dict(kind="gnb", theta=theta, var=var, class_prior=prior / prior.sum(), classes=np.arange(R), n_features=D), theta0


def _flow_gnb(D, R):
    """a GaussianNB fitted on flow rows with R classes (flow classes folded modulo R; R = 8 splits two classes by a feature)"""
    from sklearn.naive_bayes import GaussianNB
    X12, y = synth.make_flows(60_000, seed=500 + D)
    X = _flow_columns(X12, D)
    if R == 8:
        y = np.where((y < 2) & (X[:, 0] > np.median(X[:, 0])), y + 6, y)
    else:
        y = y % R
    from traffic_classifier_sdn_b200.modelio import spec_from_estimator
    return spec_from_estimator(GaussianNB().fit(X, y))


@pytest.mark.parametrize("R", [2, 5, 8])
@pytest.mark.parametrize("D", [4, 8, 12, 16])
def test_gnb_prepass_at_its_bound(D, R):
    """float32 rows, labels only, shapes 1 (128 x 4) and 3 (128 x 2): labels equal the fp64 kernel and the oracle on every
    row of an adversarial model (some rows refined in fp64), and the pre-pass certifies all but < 5 % of plain flow rows"""
    rng = np.random.default_rng(70 * D + R)
    spec, theta0 = _adversarial_gnb(D, R, rng)
    n = 200_003
    X = (theta0 + rng.normal(0.0, 30.0, (n, D))).astype(np.float32)
    X[:1000] = theta0.astype(np.float32)
    flow = _flow_gnb(D, R)
    Xf = _flow_columns(synth.make_flows(400_001, seed=600 + D, dtype=np.float32, return_labels=False), D)
    Xf = np.ascontiguousarray(Xf, np.float32)
    for s, rows in ((spec, X), (flow, Xf)):
        ref = oracle.predict(s, rows.astype(np.float64), want_scores=False)[0]
        slow = _force(from_spec(s), 1).predict_indices(rows)
        assert np.array_equal(slow, ref)
        for shape in (1, 3):
            est = from_spec(s)
            est.set_option(_lib.OPT_SCORER_SHAPE, shape)
            got = est.predict_indices(_cuda(rows)).cpu().numpy()
            refined = int(est.stats()[6])
            assert np.array_equal(got, ref), f"shape {shape}: {int((got != ref).sum())} labels differ"
            assert refined <= len(rows)
            if s is spec:
                assert refined > 0, "the adversarial model must leave rows to the fp64 re-evaluation"
            else:
                assert refined < 0.05 * len(rows), f"{refined} of {len(rows)} flow rows refined"
            print(f"gnb pre-pass D={D} R={R} {'adversarial' if s is spec else 'flows'} shape {shape}: "
                  f"{refined} of {len(rows)} rows refined in fp64")


# ------------------------------------------------------------------ 3. the bench scorers just above the small-batch shape
@pytest.mark.parametrize("name", ["gnb", "logistic", "kmeans"])
def test_bench_scorers_above_the_small_batch_limit(name):
    """bench models in auto mode on batches just large enough for the default shapes (GaussianNB 128 x 4 -- float32 rows:
    the pre-pass --, LR / KMeans 256 x 2): labels equal the oracle on every row and the forced small-batch shape"""
    import torch
    import bench
    w = bench.build_workload(name)
    for dtype in (np.float32, np.float64):
        n = _small_batch_limit(dtype) + 4099
        X = bench.synth_rows(n, w["d"], seed=4243, device=torch.device("cuda", 0))
        if dtype == np.float64:
            X = X.double()
        est = from_spec(w["spec"])
        auto = est.predict_indices(X)
        est.set_option(_lib.OPT_SCORER_SHAPE, 3)
        small = est.predict_indices(X)
        est.sync_check()
        ref = oracle.predict(w["spec"], X.cpu().numpy().astype(np.float64), want_scores=False)[0]
        got = auto.cpu().numpy()
        assert np.array_equal(got, ref), f"{np.dtype(dtype).name}: {int((got != ref).sum())} of {n} labels differ"
        assert torch.equal(auto, small)


# ------------------------------------------------------------------ 4. forest walkers
FOREST_SHAPES = (1, 2, 3)   # OPT_FOREST_SHAPE: 512 x 2, 256 x 4, 1024 x 1
FORESTS = {"one_group": dict(n_trees=6, depth=10, full=True),          # 12 282 nodes: one shared-memory group
           "many_groups": dict(n_trees=100, depth=16, full=False),
           "oversize": dict(n_trees=3, depth=15, full=True)}            # 65 535-node trees, walked in L2 / HBM


def _forest_runs(spec, X64):
    """every shape x sort x dtype against the oracle, bit for bit (labels and predict_proba)"""
    import torch
    rlab, rpr = oracle.forest(spec, X64)
    rlab_d, rpr_d = _cuda(rlab), _cuda(rpr)
    est = from_spec(spec)
    for dtype in (np.float32, np.float64):
        Xd = _cuda(X64.astype(dtype))
        for shape in FOREST_SHAPES:
            for sort in (1, 0):
                est.set_option(_lib.OPT_FOREST_SHAPE, shape)
                est.set_option(_lib.OPT_FOREST_SORT, sort)
                lab, pr = est._run(Xd, True)
                est.sync_check()
                where = f"{np.dtype(dtype).name} shape {shape} sort {sort}"
                assert torch.equal(lab, rlab_d), f"{where}: {int((lab != rlab_d).sum())} labels differ"
                assert torch.equal(pr, rpr_d), f"{where}: probabilities differ"


@pytest.mark.parametrize("forest", list(FORESTS))
def test_forest_walkers_bit_exact(forest):
    n = 3 * 2 * _sm_count() * 1024 + 5      # three 1024-row tiles per CTA at two CTAs per SM
    X = synth.make_flows(n, seed=31, return_labels=False)
    X[::7] += 1e-6                          # not representable in float32: the cast and the rounded-down thresholds matter
    spec = synth.random_forest_spec(seed=17, impure=0.2, **FORESTS[forest])
    _forest_runs(spec, X)


def _smem_optin():
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


def _forest_smem(d, C):
    """shared memory forest_pack requires before any tree: staged rows, accumulators, sort buffers, a 64-node tree buffer"""
    return max(d, C + 1) * 4096 + (C + 1) * 8192 + 7744


def _ceilings():
    """(most classes at d = 12, most features at C = 6) that forest_pack admits on this device"""
    optin = _smem_optin()
    cmax = max(c for c in range(1, 128) if _forest_smem(12, c) <= optin)
    dmax = max(d for d in range(1, 128) if _forest_smem(d, 6) <= optin)
    if optin == 232_448:   # H100: 227 KB per block
        assert (cmax, dmax) == (17, 40)
    return cmax, dmax


def _concat_forests(parts):
    out = {k: [] for k in ("left", "right", "feature", "threshold", "value")}
    offs = [0]
    for p in parts:
        o = np.asarray(p["tree_offsets"])
        offs.extend((o[1:] + offs[-1]).tolist())
        for k in out:
            out[k].append(np.asarray(p[k]))
    spec = dict(parts[0], tree_offsets=np.asarray(offs, np.int64), **{k: np.concatenate(v) for k, v in out.items()})
    spec["value"] = np.ascontiguousarray(spec["value"])
    return spec


def _leaf_tree(C, cls=None, d=12):
    v = np.zeros((1, C))
    if cls is None:
        v[0, :] = 1.0 / C            # an impure root
    else:
        v[0, cls] = 1.0
    return dict(kind="forest", tree_offsets=np.array([0, 1]), left=np.array([-1], np.int32), right=np.array([-1], np.int32),
                feature=np.array([-2], np.int32), threshold=np.array([-2.0]), value=v, n_features=d)


def _wide_rows(n, d, seed):
    X = synth.make_flows(n, seed=seed, return_labels=False)
    X = np.hstack([X] * (d // 12 + 1))[:, :d] if d > 12 else X[:, :d]
    X = np.ascontiguousarray(X)
    X[::5] += 1e-6
    return X


def _scale(d):
    base = np.array([24, 2076, 24, 122, 2069, 9651, 27, 2977, 27, 17, 2974, 2441], float)
    return np.tile(base, d // 12 + 1)[:d]


@pytest.mark.parametrize("case", ["d1", "d3", "d20", "d4_C10", "C_ceiling_d12", "d_ceiling_C6", "single_leaf_trees"])
def test_forest_edges_bit_exact(case):
    """feature and class counts at the edges: tiny d, d > 12, d < C + 1 (zero-padded rows of xs that leaves read), the
    shared-memory ceilings (a few hundred tree nodes left: one tree per group, plus a tree too large for the buffer), and
    forests that mix one-leaf trees in (also as tree 0, which the coherence sort walks)"""
    cmax, dmax = _ceilings()
    rf = synth.random_forest_spec
    if case == "d1":
        spec = rf(n_trees=8, depth=6, d=1, seed=1, impure=0.2)
    elif case == "d3":
        spec = rf(n_trees=12, depth=9, d=3, seed=2, impure=0.2, full=False)
    elif case == "d20":
        spec = rf(n_trees=16, depth=10, d=20, seed=3, impure=0.2, scale=_scale(20), full=False)
    elif case == "d4_C10":
        spec = rf(n_trees=20, depth=8, d=4, n_classes=10, seed=4, impure=0.2)
    elif case == "C_ceiling_d12":
        spec = _concat_forests([rf(n_trees=10, depth=7, n_classes=cmax, seed=5, impure=0.2),
                                rf(n_trees=1, depth=9, n_classes=cmax, seed=6, impure=0.2),
                                rf(n_trees=6, depth=6, n_classes=cmax, seed=7, impure=0.2, full=False)])
    elif case == "d_ceiling_C6":
        spec = _concat_forests([rf(n_trees=10, depth=7, d=dmax, seed=8, impure=0.2, scale=_scale(dmax)),
                                rf(n_trees=1, depth=9, d=dmax, seed=9, impure=0.2, scale=_scale(dmax)),
                                rf(n_trees=6, depth=6, d=dmax, seed=10, impure=0.2, scale=_scale(dmax), full=False)])
    else:
        trees = rf(n_trees=5, depth=7, seed=11, impure=0.2, full=False)
        spec = _concat_forests([_leaf_tree(6, 2), trees, _leaf_tree(6, 0), _leaf_tree(6, None), _leaf_tree(6, 5),
                                rf(n_trees=3, depth=9, seed=12, impure=0.2), _leaf_tree(6, 2)])
        spec["classes"] = trees["classes"]
    d = int(spec["n_features"])
    _forest_runs(spec, _wide_rows(50_003, d, seed=40 + d))


def test_forest_one_step_past_the_shared_memory_ceiling():
    """one class or one feature more than the ceilings above: from_spec refuses with a shared-memory error"""
    cmax, dmax = _ceilings()
    for d, C in ((12, cmax + 1), (dmax + 1, 6)):
        spec = synth.random_forest_spec(n_trees=2, depth=3, d=d, n_classes=C, seed=1, scale=_scale(d))
        with pytest.raises(ValueError, match="shared memory"):
            from_spec(spec)


# ------------------------------------------------------------------ 5. distance engine
@pytest.fixture(scope="module")
def knn_sets():
    """flows: 3 000 training rows, 100 of them duplicated, queries with exact copies of training rows; lattice: 3^4"""
    Xt, yt = synth.make_flows(3000, seed=41)
    Xt[2900:] = Xt[:100]
    Xq = synth.make_flows(5000, seed=42, return_labels=False)
    Xq[:300] = Xt[:300]
    rng = np.random.default_rng(7)
    tr = np.floor(rng.random((900, 4)) * 3)
    y = rng.integers(0, 5, 900).astype(np.int32)
    q = np.floor(rng.random((5000, 4)) * 3)
    return {"flows": (dict(kind="knn", fit_X=Xt, y=yt.astype(np.int32), classes=synth.CLASSES, n_features=12), Xq),
            "lattice": (dict(kind="knn", fit_X=tr, y=y, classes=np.arange(5), n_features=4), q)}


@pytest.mark.parametrize("k", [8, 9, 32])
@pytest.mark.parametrize("data", ["flows", "lattice"])
def test_knn_engine_flush_cadence_and_heap_kinds(knn_sets, data, k):
    """k = 8 / 9: the shared-memory / local-memory heap boundary, k = 32: the engine's largest heap; evaluation rounds every
    1, 2 and 31 tiles; pruned and unpruned: labels and probabilities equal the oracle"""
    base, Xq = knn_sets[data]
    spec = dict(base, k=k)
    ridx, rpr = oracle.knn(spec, Xq)
    for flush in (1, 2, 31):
        for prune_off in (0, 1):
            est = _force(from_spec(spec), 2)
            est.set_option(_lib.OPT_KNN_FLUSH_TILES, flush)
            est.set_option(_lib.OPT_KNN_PRUNE, prune_off)
            idx, pr = est._run(Xq, True)
            st = est.stats()
            assert st[1] == len(Xq) and st[2] == 0, "rows did not go through the tensor-core engine"
            assert np.array_equal(idx, ridx) and np.array_equal(pr, rpr), f"flush {flush} prune_off {prune_off}"


@pytest.mark.parametrize("m", [8, 9, 32])
def test_kneighbors_engine_flush_one(knn_sets, m):
    for data in ("flows", "lattice"):
        base, Xq = knn_sets[data]
        spec = dict(base, k=5)
        est = _force(from_spec(spec), 2)
        est.set_option(_lib.OPT_KNN_FLUSH_TILES, 1)
        dist, ind = est.kneighbors(Xq, m)
        assert est.stats()[1] == len(Xq)
        rd, ri = kno.kneighbors(spec, Xq, m)
        assert np.array_equal(ind, ri), f"{data}: indices differ on {int((ind != ri).any(1).sum())} rows"
        assert np.array_equal(dist, rd), f"{data}: distances differ"


FLOW_COLUMNS = {7: [0, 1, 3, 5, 6, 7, 9], 11: [0, 1, 3, 4, 5, 6, 7, 8, 9, 10, 11], 2: [5, 7]}


@pytest.mark.parametrize("d", [1, 2, 7, 11])
def test_knn_engine_feature_counts(d):
    """K-slot packing and kd tree at d = 1, 2 (integer lattices: masses of equal distances), 7 and 11 (flow columns)"""
    rng = np.random.default_rng(d)
    if d <= 2:
        tr = rng.integers(0, 12 if d == 1 else 7, (2000, d)).astype(float)
        y = rng.integers(0, 4, 2000).astype(np.int32)
        q = rng.integers(-1, 13 if d == 1 else 8, (6000, d)).astype(float)
        spec = dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(4), n_features=d)
    else:
        X, y = synth.make_flows(4000, seed=80 + d)
        tr = np.ascontiguousarray(X[:, FLOW_COLUMNS[d]])
        q = np.ascontiguousarray(synth.make_flows(6000, seed=90 + d, return_labels=False)[:, FLOW_COLUMNS[d]])
        q[:200] = tr[:200]
        spec = dict(kind="knn", fit_X=tr, y=y.astype(np.int32), k=5, classes=synth.CLASSES, n_features=d)
    for rows in (q, q.astype(np.float32)):
        ridx, rpr = oracle.knn(spec, rows.astype(np.float64))
        est = _force(from_spec(spec), 2)
        idx, pr = est._run(rows, True)
        st = est.stats()
        assert st[1] == len(rows) and st[2] == 0
        assert np.array_equal(idx, ridx) and np.array_equal(pr, rpr), f"{int((idx != ridx).sum())} labels differ"
        dist, ind = est.kneighbors(rows, 7)
        rd, ri = kno.kneighbors(spec, rows, 7)
        assert np.array_equal(ind, ri) and np.array_equal(dist, rd)
        print(f"knn engine d={d} {rows.dtype}: {st[7]} tie rows re-run in index order of {len(rows)}")
        if d <= 2:
            assert st[7] > 0


@pytest.mark.parametrize("d", [2, 7, 11])
def test_svc_engine_feature_counts(d):
    """SVC through the engine on a column subset of a libsvm-signed model: the full certificate bar of test_engine_gpu"""
    spec = _svc_spec(3000, 6, seed=200 + d)
    cols = FLOW_COLUMNS[d]
    sv = np.ascontiguousarray(spec["sv"][:, cols])
    spec.update(sv=sv, n_features=d, gamma=float(1.0 / (d * sv.var())))
    assert np.array_equal(np.sign(spec["dual_coef"][spec["dual_coef"] != 0]),
                          _libsvm_signs(6, spec["n_support"])[spec["dual_coef"] != 0])
    X = np.ascontiguousarray(synth.make_flows(5000, seed=300 + d, return_labels=False)[:, cols])
    _check_svc(spec, X, f"d={d} f64 rows")
    _check_svc(spec, X.astype(np.float32), f"d={d} f32 rows")


# ------------------------------------------------------------------ 6. host pipeline, alignment, concurrency
@pytest.mark.parametrize("kind", ["knn", "svc", "kneighbors"])
def test_chunked_host_calls_equal_one_device_call(specs, kind):
    """host rows in chunks of 1 000 / 4 096 / 5 000 (256-row passes split, ragged last chunk) through the engine: bit for bit
    the single device-pointer call; for KNN the index-order tie rows of the chunks add up to the single call's"""
    n = 12_345
    X = synth.make_flows(n, seed=61, return_labels=False)
    X[:200] = X[5000:5200]
    spec = specs["svc" if kind == "svc" else "knn"]
    one = _force(from_spec(spec), 2)
    Xd = _cuda(X)
    if kind == "kneighbors":
        ref = [t.cpu().numpy() for t in one.kneighbors(Xd, 5)]
    else:
        ref = [one.predict_indices(Xd).cpu().numpy()] + [t.cpu().numpy() for t in one._run(Xd, True)]
    one.sync_check()
    ties = int(one.stats()[7])
    for chunk in (1000, 4096, 5000):
        est = _force(from_spec(spec), 2)
        est.set_option(_lib.OPT_CHUNK_ROWS, chunk)
        if kind == "kneighbors":
            got = list(est.kneighbors(X, 5))
        else:
            got = [est.predict_indices(X)] + list(est._run(X, True))
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), f"chunk {chunk}"
        if kind == "knn":
            assert int(est.stats()[7]) == ties, (chunk, int(est.stats()[7]), ties)


@pytest.mark.parametrize("kind", KINDS)
def test_misaligned_device_rows(specs, kind):
    """float32 device rows that are 4-byte aligned only (a view 4 bytes into a buffer): the same labels and scores as the
    aligned rows (scorers: the generic kernel instead of the bulk-copy tiles; the others read rows with scalar loads)"""
    import torch
    X = synth.make_flows(5000, seed=71, dtype=np.float32, return_labels=False)
    Xd = _cuda(X)
    buf = torch.empty(X.size + 1, dtype=torch.float32, device="cuda")
    view = buf[1:1 + X.size].view(X.shape)
    view.copy_(Xd)
    assert view.data_ptr() % 16 == 4
    est = from_spec(specs[kind])
    lab_a, sc_a = est._run(Xd, True)
    lab_b, sc_b = est._run(view, True)
    only_a, only_b = est.predict_indices(Xd), est.predict_indices(view)
    est.sync_check()
    assert torch.equal(lab_a, lab_b) and torch.equal(only_a, only_b) and torch.equal(only_a, lab_a)
    assert torch.equal(sc_a, sc_b)


@pytest.mark.parametrize("kind", KINDS)
def test_concurrent_host_predicts_on_one_handle(specs, kind):
    """four host threads predict on one handle at once (ctypes releases the GIL), three rounds each, labels only and with
    scores, in 5 000-row chunks: each result equals the single-threaded one, only the thread whose rows hold a NaN gets a
    ValueError, and the handle keeps working"""
    est = from_spec(specs[kind])
    est.set_option(_lib.OPT_CHUNK_ROWS, 5000)
    rows = [synth.make_flows(12_000 + 1000 * i, seed=80 + i, return_labels=False) for i in range(4)]
    bad = 2
    rows[bad][7777, 5] = np.nan
    expect = {i: [est._run(rows[i], s) for s in (False, True)] for i in range(4) if i != bad}
    results, errors = {}, {}
    start = threading.Barrier(4)

    def work(i):
        start.wait()
        out = []
        try:
            for rep in range(3):
                out.append(est._run(rows[i], rep % 2 == 1))
        except Exception as e:   # noqa: BLE001 -- recorded and checked below
            errors[i] = e
        results[i] = out

    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert set(errors) == {bad} and isinstance(errors[bad], ValueError), errors
    assert "NaN" in str(errors[bad]) or "infinity" in str(errors[bad])
    for i, exp in expect.items():
        assert len(results[i]) == 3
        for rep, (idx, sc) in enumerate(results[i]):
            e_idx, e_sc = exp[rep % 2]
            assert np.array_equal(idx, e_idx), (i, rep)
            assert (sc is None) == (e_sc is None) and (sc is None or np.array_equal(sc, e_sc)), (i, rep)
    idx, sc = est._run(rows[0], True)
    assert np.array_equal(idx, expect[0][1][0]) and np.array_equal(sc, expect[0][1][1])


# ------------------------------------------------------------------ 7. two devices in one process
def test_scorers_on_two_devices_in_one_process():
    """one handle per device; shapes 1 and 2 need more than 48 KB of dynamic shared memory (73 728 B for float32 rows at
    d = 12), an opt-in each device needs for itself: predicting on GPU 0 first must not leave GPU 1 without it"""
    import torch
    if _lib.device_count() < 2:
        pytest.skip("needs two GPUs")
    lib = _lib.load()
    rng = np.random.default_rng(3)
    specs_ = [_scorer_spec("gnb", 6, 12, rng)[0], _scorer_spec("linear", 5, 8, rng)[0]]
    models = {}
    try:
        for dev in (0, 1):
            _lib.check(lib.tcsdn_set_device(dev))
            models[dev] = [from_spec(s) for s in specs_]
    finally:
        _lib.check(lib.tcsdn_set_device(0))
    for s, dev_models in zip(specs_, zip(models[0], models[1])):
        X = _scorer_rows_host(_scorer_n(np.float32), s["n_features"], seed=9).astype(np.float32)
        ref = oracle.predict(s, X.astype(np.float64), want_scores=False)[0]
        for dev, est in zip((0, 1), dev_models):
            Xd = torch.from_numpy(X).to(torch.device("cuda", dev))
            for shape in (1, 2):
                est.set_option(_lib.OPT_SCORER_SHAPE, shape)
                got = est.predict_indices(Xd)
                with torch.cuda.device(dev):
                    est.sync_check()
                assert np.array_equal(got.cpu().numpy(), ref), (s["kind"], dev, shape)
