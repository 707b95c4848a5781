"""GPU: the tensor-core (wgmma) distance engine against the oracle.

KNN through the engine must be bit-identical to the fp64 kernel / oracle / sklearn's sequential heap: the
tensor-core distances only FILTER candidates, every survivor is re-evaluated in fp64 in index order.
SVC through the engine evaluates exp() and the one-vs-one sums in fp32 next to a per-pair error bound; rows whose
vote the bound cannot certify are re-evaluated by the fp64 kernel in the same call, so LABELS equal libsvm's fp64
vote on every row (no tolerance, no mask).  Decision VALUES never come from the engine: `decision_function` is the
fp64 kernel at every batch size (SVC_DEC_TOL).  The engine's own values and bounds are visible to the tests
through the audit options 3 / 4: |engine value - fp64 value| <= bound must hold on every pair.
"""
import numpy as np
import pytest

import oracle
from traffic_classifier_sdn_b200 import _lib, from_spec, synth

pytestmark = pytest.mark.gpu

SVC_DEC_TOL = 1e-9      # absolute: decision values (fp64 kernel) against libsvm's fp64 (SURVEY 8d policy: <= 1e-5)
SVC_EPS_MMA = 2.0 ** -19  # csrc/svc_engine.cu kSvcEpsMma
KAPPA = 2.0 ** -18      # csrc/knn_engine.cu kKappa


def _force(est, mode):
    est.set_option(_lib.OPT_ENGINE, mode)
    return est


def _knn_spec(nt, k=5, seed=0, d=12):
    X, y = synth.make_flows(nt, seed=seed)
    return dict(kind="knn", fit_X=X[:, :d].copy(), y=y.astype(np.int32), k=k, classes=synth.CLASSES, n_features=d)


@pytest.mark.parametrize("nt,nq,k", [(5000, 6000, 5), (777, 4100, 1), (20000, 9000, 5), (3000, 5000, 17), (64, 4096, 3)])
def test_knn_engine_bit_exact_vs_oracle(nt, nq, k):
    spec = _knn_spec(nt, k=k, seed=nt)
    est = _force(from_spec(spec), 2)
    Xq = synth.make_flows(nq, seed=nq + 1, return_labels=False)
    dup = min(300, nt)
    Xq[:dup] = spec["fit_X"][:dup]           # exact duplicates of training rows (distance 0, ties with their twins)
    idx, pr = est._run(Xq, True)
    ridx, rpr = oracle.knn(spec, Xq)
    st = est.stats()
    assert st[1] == nq and st[2] == 0, "rows did not go through the tensor-core engine"
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)
    # the filter must actually filter: far fewer exact evaluations than pairs
    assert st[3] < 0.05 * nq * nt + 64 * nq, (st[3], nq * nt)
    print(f"knn nt={nt} nq={nq} k={k}: {st[3] / nq:.1f} exact re-evaluations per query of {nt} candidates")
    idx32, pr32 = est._run(Xq.astype(np.float32), True)
    r32 = oracle.knn(spec, Xq.astype(np.float32).astype(np.float64))
    assert np.array_equal(pr32, r32[1]) and np.array_equal(idx32, r32[0])


@pytest.mark.parametrize("case", ["flows", "positive_large", "offset_4e5", "heavy_tail"])
def test_knn_filter_slack_audit_all_pairs(case):
    """audit mode re-evaluates EVERY pair exactly and records max |tensor-core value - exact| / (||x||^2 + max ||t||^2):
    the filter slack kappa = 2^-18 must dominate it with a wide margin on adversarial magnitudes."""
    rng = np.random.default_rng(11)
    nt, nq = 2048, 4096
    if case == "flows":
        tr = synth.make_flows(nt, seed=1, return_labels=False); q = synth.make_flows(nq, seed=2, return_labels=False)
    elif case == "positive_large":   # no sign cancellation inside the dot products, every term near 4e5^2
        tr = rng.uniform(1e5, 4e5, (nt, 12)); q = rng.uniform(1e5, 4e5, (nq, 12))
    elif case == "offset_4e5":
        tr = 4e5 + rng.normal(0, 50.0, (nt, 12)); q = 4e5 + rng.normal(0, 50.0, (nq, 12))
    else:
        tr = rng.standard_cauchy((nt, 12)) * 100; q = rng.standard_cauchy((nq, 12)) * 100
        tr = np.clip(tr, -1e6, 1e6); q = np.clip(q, -1e6, 1e6)
    y = rng.integers(0, 3, nt).astype(np.int32)
    spec = dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(3), n_features=12)
    est = _force(from_spec(spec), 3)
    idx, pr = est._run(q, True)
    st = est.stats()
    assert st[3] == nq * nt, "audit mode must re-evaluate every pair"
    ratio = st[5] / 2.0 ** 40
    print(f"audit[{case}]: max error ratio {ratio:.3e} = 2^{np.log2(ratio):.1f} (kappa = 2^-18)")
    assert 0 < ratio < KAPPA / 4
    ridx, rpr = oracle.knn(spec, q)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)


def test_knn_engine_lattice_ties_heap_order():
    rng = np.random.default_rng(7)
    tr = np.floor(rng.random((900, 4)) * 3)
    y = rng.integers(0, 5, 900).astype(np.int32)
    q = np.floor(rng.random((5000, 4)) * 3)
    spec = dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(5), n_features=4)
    est = _force(from_spec(spec), 2)
    idx, pr = est._run(q, True)
    ridx, rpr = oracle.knn(spec, q)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)
    # the engine visits tiles nearest-first; rows whose class counts depend on WHICH of several equally distant rows sklearn's
    # index-order heap keeps are handed to the index-order kernel (stats[7]) -- on a 3^4 lattice that is most of them
    assert est.stats()[7] > 0
    from sklearn.neighbors import KNeighborsClassifier
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=1):
        sk = KNeighborsClassifier(5, algorithm="brute").fit(tr, y)
        assert np.array_equal(pr, sk.predict_proba(q))


@pytest.mark.parametrize("nt,nq,k", [(20000, 40000, 5), (5000, 9000, 3), (130, 5000, 7)])
def test_knn_engine_pruned_equals_unpruned_and_oracle(nt, nq, k):
    """queries sorted by home tile + far tiles left out (the default) against every-tile-for-every-query (option 8 = 1) and the
    oracle: identical labels and probabilities; the pruned run multiplies fewer tiles per pass and evaluates no more pairs"""
    spec = _knn_spec(nt, k=k, seed=nt + 3)
    Xq = synth.make_flows(nq, seed=nq + 7, return_labels=False)
    Xq[:100] = spec["fit_X"][:100]
    ridx, rpr = oracle.knn(spec, Xq)
    n_tiles = -(-nt // 64)
    seen = {}
    for off in (0, 1):
        est = _force(from_spec(spec), 2)
        est.set_option(_lib.OPT_KNN_PRUNE, off)
        idx, pr = est._run(Xq, True)
        st = est.stats()
        assert st[1] == nq and st[2] == 0
        assert np.array_equal(idx, ridx) and np.array_equal(pr, rpr), f"prune_off={off}"
        seen[off] = (st[4] / 1000.0, st[3] / nq, st[7])
    print(f"knn nt={nt} k={k}: tiles per pass pruned {seen[0][0]:.1f} / unpruned {seen[1][0]:.1f} of {n_tiles}; "
          f"exact evaluations per query {seen[0][1]:.1f} / {seen[1][1]:.1f}; tie rows {seen[0][2]} / {seen[1][2]}")
    assert abs(seen[1][0] - n_tiles) < 1e-6
    assert seen[0][0] <= n_tiles
    if nt >= 20000:
        assert seen[0][0] < 0.9 * n_tiles, "clustered flow rows, dense queries: the pruned pass should leave tiles out"


def test_knn_engine_large_model_without_tile_table():
    """beyond 4 096 tiles (262 144 training rows) there is no tile-by-tile neighbour table: the producer walks outwards from the
    home tile in kd order and tests every tile -- same answers, still far fewer tiles than all of them"""
    nt, nq, k = 270_000, 4096, 5
    spec = _knn_spec(nt, k=k, seed=99)
    # 16 spots x 256 queries around them: with 4 219 kd cells, 4 096 queries spread over the whole feature space would put one
    # query in each cell and leave a pass nothing to leave out
    rng = np.random.default_rng(123)
    spots = spec["fit_X"][rng.choice(nt, 16, replace=False)]
    Xq = (spots[:, None, :] * (1.0 + 1e-3 * rng.standard_normal((16, 256, 12))) + 1e-2 * rng.standard_normal((16, 256, 12))).reshape(nq, 12)
    Xq[::256] = spots                                        # the spots themselves: distance 0 to a training row
    est = _force(from_spec(spec), 2)
    idx, pr = est._run(Xq, True)
    ridx, rpr = oracle.knn(spec, Xq)
    st = est.stats()
    assert st[1] == nq and np.array_equal(idx, ridx) and np.array_equal(pr, rpr)
    n_tiles = -(-nt // 64)
    print(f"knn nt={nt}: {st[4] / 1000:.1f} of {n_tiles} tiles per pass, {st[3] / nq:.1f} exact evaluations per query, {st[7]} tie rows")
    assert st[4] / 1000.0 < 0.75 * n_tiles


def test_knn_engine_class_relevant_ties_go_to_index_order_kernel():
    """twin training rows with DIFFERENT classes and k = 1: the label is whichever twin sklearn's heap keeps (the first); twins
    with the SAME class need no second opinion"""
    rng = np.random.default_rng(5)
    base = rng.normal(0, 100.0, (3000, 12))
    tr = np.concatenate([base, base[:500]])                  # 500 rows have an exact twin (index + 3000)
    y = rng.integers(0, 4, len(tr)).astype(np.int32)
    y[3000:3250] = y[:250]                                   # ... half of the twins agree on the class
    y[3250:3500] = (y[250:500] + 1) % 4                      # ... half do not
    q = np.concatenate([base[:500], rng.normal(0, 100.0, (4000, 12))])
    spec = dict(kind="knn", fit_X=tr, y=y, k=1, classes=np.arange(4), n_features=12)
    est = _force(from_spec(spec), 2)
    idx, pr = est._run(q, True)
    ridx, rpr = oracle.knn(spec, q)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)
    # expected: queries whose nearest distance is shared by rows of different classes (the 250 disagreeing twins themselves,
    # and every other query whose nearest neighbour happens to be such a pair)
    d2 = ((q[:, None, :] - tr[None, :, :]) ** 2).sum(2)
    near = d2 == d2.min(1, keepdims=True)
    expect = sum(len(set(y[np.flatnonzero(r)])) > 1 for r in near)
    assert expect >= 250 and est.stats()[7] == expect, (expect, est.stats())


def test_knn_engine_equals_fp64_kernel_on_golden(golden, specs):
    X = golden["X"]
    a = _force(from_spec(specs["knn"]), 2)._run(X, True)
    b = _force(from_spec(specs["knn"]), 1)._run(X, True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert np.array_equal(a[0], golden["knn.expected_label"])


def test_knn_engine_huge_magnitudes_and_offsets():
    """features around 4e5 with tiny relative differences: the filter must still keep every true neighbour"""
    rng = np.random.default_rng(3)
    tr = 4e5 + rng.normal(0, 3.0, (4000, 12))
    y = rng.integers(0, 4, 4000).astype(np.int32)
    q = 4e5 + rng.normal(0, 3.0, (4500, 12))
    spec = dict(kind="knn", fit_X=tr, y=y, k=5, classes=np.arange(4), n_features=12)
    est = _force(from_spec(spec), 2)
    idx, pr = est._run(q, True)
    ridx, rpr = oracle.knn(spec, q)
    assert np.array_equal(pr, rpr) and np.array_equal(idx, ridx)


def _libsvm_signs(C, nsup):
    """sign[m, s] of libsvm's dual coefficients: row m of a class-c vector faces opponent o = m if m < c else m + 1 and is
    +alpha when c < o, -alpha when c > o (sk:svm/src/libsvm/svm.cpp:2093-2118)."""
    cls = np.repeat(np.arange(C), nsup)
    m = np.arange(C - 1)[:, None]
    opp = np.where(m < cls[None, :], m, m + 1)
    return np.where(cls[None, :] < opp, 1.0, -1.0)


def _svc_spec(nsv, C=6, seed=0, gamma=None, signed=True):
    """A synthetic SVC model: support vectors from the flow generator, dual coefficients with libsvm's sign pattern
    (many at the box bound 1.0, as C=1 fits have) -- or with random signs (`signed=False`: not a libsvm model)."""
    rng = np.random.default_rng(seed)
    Xs, ys = synth.make_flows(nsv, seed=seed + 1, class_weights=np.r_[np.ones(C), np.zeros(6 - C)] if C < 6 else None)
    order = np.argsort(ys, kind="stable")
    Xs, ys = Xs[order], ys[order]
    nsup = np.bincount(ys, minlength=C)[:C].astype(np.int32)
    g = gamma if gamma is not None else 1.0 / (12 * Xs.var())
    mag = np.minimum(1.0, rng.uniform(0.0, 1.6, (C - 1, nsv))) * (rng.random((C - 1, nsv)) < 0.6)
    dual = mag * (_libsvm_signs(C, nsup) if signed else rng.choice([-1.0, 1.0], (C - 1, nsv)))
    return dict(kind="svc", sv=Xs, dual_coef=dual, intercept=rng.normal(0, 0.5, C * (C - 1) // 2), n_support=nsup,
                gamma=float(g), classes=synth.CLASSES[:C], n_features=12, decision_function_shape="ovr", break_ties=False,
                n_classes=C)


def _check_svc(spec, X, name="", max_refined=0.05):
    """labels through the engine == libsvm fp64 labels on EVERY row; decision values (fp64 kernel) to SVC_DEC_TOL; the
    certificate holds on every pair (audit options) and is not vacuous (few rows need the fp64 re-evaluation)."""
    ridx, rdec = oracle.svc(spec, X.astype(np.float64))
    est = _force(from_spec(spec), 2)
    idx = est.predict_indices(X)
    st = est.stats()
    assert st[1] == len(X) and st[2] == 0, "rows did not go through the tensor-core engine"
    refined = int(st[6])
    assert np.array_equal(idx, ridx), f"{int((idx != ridx).sum())} labels differ from libsvm's fp64 vote"
    assert idx.min() >= 0
    # decision values: always the fp64 kernel, whatever the batch size
    idx2, dec = from_spec(spec)._run(X, True)
    assert np.array_equal(idx2, ridx)
    err = float(np.max(np.abs(dec - rdec)))
    assert err < SVC_DEC_TOL, f"max |dec - libsvm fp64| = {err:.3e}"
    # the engine's own values against its own bounds
    a3 = _force(from_spec(spec), 3)
    raw_idx, raw = a3._run(X, True)
    ratio = a3.stats()[5] / 2.0 ** 40
    _, bound = _force(from_spec(spec), 4)._run(X, True)
    viol = np.abs(raw - rdec) > bound
    assert not viol.any(), f"certificate violated on {int(viol.sum())} pairs: worst {np.max(np.abs(raw - rdec) / bound):.2f}x the bound"
    assert 0 < ratio < SVC_EPS_MMA / 2, f"tensor-core error ratio 2^{np.log2(ratio):.1f} too close to eps_mma = 2^-19"
    tight = float(np.max(np.abs(raw - rdec) / bound))
    print(f"svc {name}: {len(X)} rows, refined {refined} ({100.0 * refined / len(X):.3f} %), raw engine labels wrong on "
          f"{int((raw_idx != ridx).sum())}, max |raw - fp64| {np.max(np.abs(raw - rdec)):.2e}, worst error/bound {tight:.3f}, "
          f"mma error ratio 2^{np.log2(ratio):.1f}, fp64 kernel err {err:.1e}")
    assert refined <= max(max_refined * len(X), 50), "the certificate rejects too many rows to be useful"
    return refined


def test_svc_engine_golden(golden, specs):
    _check_svc(specs["svc"], golden["X"], "golden")
    est = from_spec(specs["svc"])            # auto mode: 7 653 rows take the engine
    assert np.array_equal(est.predict_indices(golden["X"]), golden["svc.expected_label"])
    assert est.stats()[1] == len(golden["X"])


@pytest.mark.parametrize("nsv,C,nq", [(3000, 6, 5000), (513, 3, 4200), (20000, 6, 4608), (130, 2, 4096)])
def test_svc_engine_synthetic(nsv, C, nq):
    spec = _svc_spec(nsv, C, seed=nsv)
    X = synth.make_flows(nq, seed=nsv + 5, return_labels=False)
    _check_svc(spec, X, f"nsv={nsv} C={C} f64 rows")
    _check_svc(spec, X.astype(np.float32), f"nsv={nsv} C={C} f32 rows")


@pytest.mark.parametrize("kw", [dict(), dict(C=10.0), dict(gamma=1e-6)])
def test_svc_engine_sklearn_fitted(kw):
    """a real libsvm fit (class overlap, many bounded vectors): labels equal sklearn's own predict on fresh rows"""
    from sklearn.svm import SVC
    Xtr, ytr = synth.make_flows(6000, seed=77)
    sk = SVC(**kw).fit(Xtr, ytr)
    from traffic_classifier_sdn_b200.modelio import spec_from_estimator
    spec = spec_from_estimator(sk)
    X = synth.make_flows(8192, seed=78, return_labels=False)
    _check_svc(spec, X, f"sklearn fit {kw} nSV={len(spec['sv'])}")
    est = from_spec(spec)
    assert np.array_equal(est.predict(X), sk.predict(X))
    assert np.max(np.abs(est.decision_function(X) - sk.decision_function(X))) < 1e-8


def test_svc_engine_adversarial_magnitudes():
    """offset data (every feature near 4e5 with unit spread) and heavy tails: the bound must still hold"""
    rng = np.random.default_rng(5)
    for case in ("offset", "tails"):
        if case == "offset":
            sv = 4e5 + rng.normal(0, 40.0, (2000, 12)); X = 4e5 + rng.normal(0, 40.0, (4500, 12)); g = 1.0 / (12 * 1600.0)
        else:
            sv = np.clip(rng.standard_cauchy((2000, 12)) * 50, -1e6, 1e6); X = np.clip(rng.standard_cauchy((4500, 12)) * 50, -1e6, 1e6)
            g = 1e-5
        C = 4
        nsup = np.array([500, 500, 500, 500], np.int32)
        dual = np.minimum(1.0, rng.uniform(0, 1.6, (C - 1, 2000))) * _libsvm_signs(C, nsup)
        spec = dict(kind="svc", sv=sv, dual_coef=dual, intercept=rng.normal(0, 0.5, 6), n_support=nsup, gamma=float(g),
                    classes=np.arange(C), n_features=12, decision_function_shape="ovr", break_ties=False, n_classes=C)
        _check_svc(spec, X, case, max_refined=1.0)   # heavy tails: most rows are far from c0, the bound is wide; still exact


def test_svc_uncertifiable_model_stays_on_fp64():
    """dual coefficients without libsvm's sign pattern: the certificate does not apply, so the engine is not used"""
    spec = _svc_spec(1500, 5, seed=3, signed=False)
    X = synth.make_flows(5000, seed=9, return_labels=False)
    est = from_spec(spec)
    idx, dec = est._run(X, True)
    ridx, rdec = oracle.svc(spec, X)
    assert np.array_equal(idx, ridx) and np.max(np.abs(dec - rdec)) < SVC_DEC_TOL
    assert np.array_equal(est.predict_indices(X), ridx)
    st = est.stats()
    assert st[1] == 0 and st[2] == len(X)
    with pytest.raises(ValueError, match="forced"):
        _force(from_spec(spec), 2).predict_indices(X)


def test_svc_decision_function_same_either_side_of_engine_threshold(golden, specs):
    """the engine threshold (4 096 rows) must not change decision values: both sides are the fp64 kernel"""
    X = golden["X"]
    est = from_spec(specs["svc"])
    big = est._run(X[:5000], True)[1]
    small = np.vstack([est._run(X[i:i + 1000], True)[1] for i in range(0, 5000, 1000)])
    assert np.array_equal(big, small)
    assert np.max(np.abs(big - golden["svc.expected_score"][:5000])) < SVC_DEC_TOL


def test_engine_ragged_and_auto_dispatch(specs):
    """n not a multiple of 512; small batches stay on the fp64 kernels, large ones take the engine"""
    for kind in ("knn", "svc"):
        est = from_spec(specs[kind])
        for n in (100, 4095, 4096, 4097, 5000):
            X = synth.make_flows(n, seed=n, return_labels=False)
            idx = est.predict_indices(X)
            st = est.stats()
            assert (st[1] == n) == (n >= 4096) and (st[2] == n) == (n < 4096)
            ridx, rsc = oracle.predict(specs[kind], X)
            assert np.array_equal(idx, ridx)
            idx, sc = est._run(X, True)
            assert np.array_equal(idx, ridx)
            if kind == "knn":
                assert np.array_equal(sc, rsc)
            else:
                assert est.stats()[2] == n and np.max(np.abs(sc - rsc)) < SVC_DEC_TOL


def test_engine_nonfinite_rows_raise(specs):
    X = synth.make_flows(5000, seed=1, return_labels=False)
    X[4321, 7] = np.inf
    for kind in ("knn", "svc"):
        with pytest.raises(ValueError, match="NaN|infinity"):
            from_spec(specs[kind]).predict(X)


# ------------------------------------------------------------------ BASELINE sizes: 10M query rows (configs[2], configs[3])
@pytest.mark.parametrize("name", ["knn", "svc"])
def test_engine_full_size_properties(name):
    """The bench workloads at their full size (10M rows x 50k training rows / 20k support vectors), checked through
    properties that do not need a 10M-row oracle: a permutation of the rows permutes the labels, one launch equals
    eight slices, a strided sample equals the CPU oracle and the fp64 CUDA-core kernel EXACTLY (KNN and SVC), and the
    exact-evaluation / refinement counters stay sane."""
    import os
    import sys
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    w = bench.build_workload(name)
    n = w["full_rows"]
    est = from_spec(w["spec"])
    X = bench.synth_rows(n, w["d"], seed=4242, device=torch.device("cuda", 0))
    full = est.predict_indices(X)
    st = est.stats()
    assert st[1] == n and st[2] == 0                       # every row went through the tensor-core engine
    g = torch.Generator(device="cpu").manual_seed(3)
    perm = torch.randperm(n, generator=g).cuda()
    assert torch.equal(full[perm], est.predict_indices(X[perm].contiguous()))
    assert torch.equal(full, torch.cat([est.predict_indices(c.contiguous()) for c in X.chunk(8)]))
    est.sync_check()
    hist = np.bincount(full.cpu().numpy(), minlength=8)
    assert hist.sum() == n and (hist > 0).sum() >= 2       # not a constant answer
    # strided sample against the oracle (fp64 restatement of sklearn) and the fp64 kernel
    s = slice(0, n, 20_011)
    xs = X[s].cpu().numpy().astype(np.float64)
    lab_o, sc_o = oracle.predict(w["spec"], xs, want_scores=True)
    lab_e = full[s].cpu().numpy()
    est64 = _force(from_spec(w["spec"]), 1)
    lab_k = est64.predict_indices(xs)
    assert np.array_equal(lab_k, lab_o)
    if name == "knn":
        assert np.array_equal(lab_e, lab_o)
        evals_per_query = (est.stats()[3]) / (3.0 * n)     # three full passes so far
        assert 5 <= evals_per_query < 400
    else:
        assert np.array_equal(lab_e, lab_o)
        refined = est.stats()[6] / (3.0 * n)               # three full passes so far
        print(f"svc 10M x {len(w['spec']['sv'])}: {100 * refined:.3f} % of rows re-evaluated in fp64")
        assert refined < 0.10
