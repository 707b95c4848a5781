"""RandomForestClassifier.fit(X, y, backend="gpu") (csrc/forest_fit.cu) against scikit-learn 1.9 and the CPU definition
(tests/forest_fit_oracle.py): the same trees, np.array_equal on all eight node arrays and on feature_importances_."""
import numpy as np
import pytest

import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import synth
from traffic_classifier_sdn_b200.estimators import forest_feature_importances, forest_fit
from forest_fit_oracle import fit_forest, forest_diff, sklearn_forest
from test_forest_fit import CASES, tricky_rows

pytestmark = pytest.mark.gpu


def _gpu_forest(est):
    return dict(est.tree_arrays_, feature_importances=est.feature_importances_)


def _check(X, y, oracle=True, **p):
    from sklearn.ensemble import RandomForestClassifier as SK
    sk = SK(**p).fit(X, y)
    est = tc.RandomForestClassifier(**p).fit(X, y, backend="gpu")
    assert np.array_equal(est.classes_, sk.classes_)
    mine = _gpu_forest(est)
    assert forest_diff(mine, sklearn_forest(sk)) == []
    if oracle:
        assert forest_diff(mine, fit_forest(X, y, **p)[1]) == []
    assert est.n_estimators_ == len(sk.estimators_) and est.n_classes_ == sk.n_classes_
    return est, sk


@pytest.mark.parametrize("p", CASES, ids=[str(c) for c in CASES])
def test_gpu_trees_are_sklearns_on_flows(p):
    X, y = synth.make_flows(2500, seed=3)
    est, sk = _check(X, y, n_estimators=3, random_state=11, **p)
    Xh, _ = synth.make_flows(3000, seed=99)
    assert np.array_equal(est.predict(Xh), sk.predict(Xh))
    assert np.array_equal(est.predict_proba(Xh), sk.predict_proba(Xh))


def test_gpu_trees_on_golden_rows_ties_and_labels(golden):
    from sklearn.ensemble import RandomForestClassifier as SK
    _check(golden["X"], golden["y"], n_estimators=4, random_state=0)
    X, y = tricky_rows()
    _check(X, y, n_estimators=4, random_state=2)
    _check(X, y, n_estimators=2, random_state=2, max_features=None)
    X, y = synth.make_flows(2000, seed=4)
    _check(X.astype(np.float32), y, n_estimators=2, random_state=1)
    _check(X, y % 2, n_estimators=2, random_state=1)
    # 20 classes on 12 features need more shared memory than the predict walker (tcsdn_forest_create) has, so these trees
    # are compared as the fit returns them, without building a predict handle
    y20 = np.random.default_rng(5).integers(0, 20, len(X))
    p20 = dict(n_estimators=2, random_state=1, max_depth=8)
    classes, a = forest_fit(X, y20, p20)
    mine = dict(a, feature_importances=forest_feature_importances(a["tree_offsets"], a["left"], a["right"], a["feature"],
                                                                  a["impurity"], a["weighted_n_node_samples"], 12))
    assert forest_diff(mine, sklearn_forest(SK(**p20).fit(X, y20))) == []
    assert forest_diff(mine, fit_forest(X, y20, **p20)[1]) == []
    _check(X, np.array(["dns", "ping", "voice", "game"])[y % 4], n_estimators=2, random_state=1)
    _check(X[:1], y[:1], n_estimators=2, random_state=0)
    _check(X[:50], np.zeros(50, np.int64), n_estimators=2, random_state=0)


def test_gpu_fit_is_repeatable_and_device_rows_stay_on_device():
    import torch
    X, y = synth.make_flows(20_000, seed=8)
    X32 = X.astype(np.float32)
    a = tc.RandomForestClassifier(n_estimators=6, random_state=3).fit(X32, y, backend="gpu")
    b = tc.RandomForestClassifier(n_estimators=6, random_state=3).fit(X32, y, backend="gpu")
    assert forest_diff(_gpu_forest(a), _gpu_forest(b)) == []

    class NoHostCopy(torch.Tensor):
        __module__ = "torch"   # a CUDA torch tensor to the estimator, whose host copies fail

        def cpu(self, *a, **k):
            raise AssertionError("rows copied to the host")

        def numpy(self, *a, **k):
            raise AssertionError("rows copied to the host")

    Xd = torch.from_numpy(X32).cuda().as_subclass(NoHostCopy)
    yd = torch.from_numpy(y).cuda()
    c = tc.RandomForestClassifier(n_estimators=6, random_state=3).fit(Xd, yd, backend="gpu")
    assert forest_diff(_gpu_forest(a), _gpu_forest(c)) == []


def test_gpu_large_root_takes_the_global_sort_and_matches_sklearn():
    from sklearn.ensemble import RandomForestClassifier as SK
    X, y = synth.make_flows(200_000, seed=12)
    p = dict(n_estimators=20, random_state=4, max_depth=12)
    sk = SK(n_jobs=-1, **p).fit(X, y)
    est = tc.RandomForestClassifier(**p).fit(X, y, backend="gpu")
    assert forest_diff(_gpu_forest(est), sklearn_forest(sk)) == []


def test_gpu_tree_that_outgrows_its_first_capacity_is_grown_again():
    X, y = synth.make_flows(3000, seed=13)
    p = dict(n_estimators=3, random_state=6)
    ref = tc.RandomForestClassifier(**p).fit(X, y, backend="gpu")
    small = tc.RandomForestClassifier(**p)
    assert small._fit_gpu(X, y, True, node_capacity=7)
    assert forest_diff(_gpu_forest(small), _gpu_forest(ref)) == []
    assert np.diff(ref.tree_arrays_["tree_offsets"]).min() > 7


def test_gpu_fit_errors_and_auto_route():
    X, y = synth.make_flows(500, seed=14)
    bad = X.copy()
    bad[17, 3] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        tc.RandomForestClassifier(n_estimators=2).fit(bad, y, backend="gpu")
    with pytest.raises(ValueError, match="inconsistent"):
        tc.RandomForestClassifier(n_estimators=2).fit(X, y[:-1], backend="gpu")
    for p in (dict(criterion="entropy"), dict(class_weight="balanced"), dict(max_leaf_nodes=8),
              dict(min_weight_fraction_leaf=0.1), dict(oob_score=True), dict(warm_start=True), dict(ccp_alpha=0.1)):
        with pytest.raises(ValueError, match=next(iter(p))):
            tc.RandomForestClassifier(n_estimators=2, **p).fit(X, y, backend="gpu")
    est = tc.RandomForestClassifier(n_estimators=2, random_state=0).fit(X, y)   # auto: scikit-learn on the host
    assert not hasattr(est, "tree_arrays_") and est.feature_importances_.shape == (12,)
