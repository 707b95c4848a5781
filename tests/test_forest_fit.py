"""RandomForestClassifier.fit's definition (tests/forest_fit_oracle.py) against scikit-learn 1.9: the oracle's trees must
be scikit-learn's, np.array_equal on all eight node arrays of every tree and on feature_importances_.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import _lib, synth
from traffic_classifier_sdn_b200.estimators import forest_fit_plan
from forest_fit_oracle import fit_forest, forest_diff, sklearn_forest

CASES = [dict(), dict(max_depth=4), dict(min_samples_leaf=5), dict(min_samples_split=10), dict(min_samples_split=0.01),
         dict(max_features=None), dict(max_features="log2"), dict(max_features=2), dict(max_features=0.5),
         dict(bootstrap=False), dict(max_samples=0.5), dict(min_impurity_decrease=1e-3)]


def tricky_rows(seed=0, n=1500):
    """Constant columns, duplicated rows and neighbouring values closer than FEATURE_THRESHOLD (1e-7)."""
    rng = np.random.default_rng(seed)
    X = np.round(rng.normal(size=(n, 5)), 1)
    X[:, 1] = 3.0
    X[:, 2] = 1.0 + rng.integers(0, 4, n) * 6e-8
    X[:, 3] = 1.0 + rng.integers(0, 5, n) * 1.2e-7
    X = np.vstack([X, X[:200]])
    y = rng.integers(0, 3, len(X))
    y[:500] = (X[:500, 2] > 1.0000001).astype(int)
    return X, y


def _check(X, y, **p):
    from sklearn.ensemble import RandomForestClassifier as SK
    sk = SK(**p).fit(X, y)
    classes, mine = fit_forest(X, y, **p)
    assert np.array_equal(classes, sk.classes_)
    assert forest_diff(mine, sklearn_forest(sk)) == []
    return mine


@pytest.mark.parametrize("p", CASES, ids=[str(c) for c in CASES])
def test_oracle_is_sklearn_on_flows(p):
    X, y = synth.make_flows(2500, seed=3)
    _check(X, y, n_estimators=3, random_state=11, **p)


def test_oracle_is_sklearn_on_golden_rows(golden):
    _check(golden["X"], golden["y"], n_estimators=2, random_state=0)


@pytest.mark.parametrize("p", [dict(), dict(max_features=None)], ids=["default", "all-features"])
def test_oracle_is_sklearn_on_ties_and_constants(p):
    X, y = tricky_rows()
    _check(X, y, n_estimators=4, random_state=2, **p)


def test_oracle_float32_two_twenty_and_string_classes():
    X, y = synth.make_flows(2000, seed=4)
    _check(X.astype(np.float32), y, n_estimators=2, random_state=1)
    _check(X, y % 2, n_estimators=2, random_state=1)
    rng = np.random.default_rng(5)
    _check(X, rng.integers(0, 20, len(X)), n_estimators=2, random_state=1, max_depth=8)
    _check(X, np.array(["dns", "ping", "voice", "game"])[y % 4], n_estimators=2, random_state=1)


def test_oracle_single_row_and_single_class():
    X, y = synth.make_flows(50, seed=6)
    _check(X[:1], y[:1], n_estimators=2, random_state=0)
    _check(X, np.zeros(len(X), np.int64), n_estimators=2, random_state=0)


def test_plan_refuses_what_it_does_not_support():
    for bad in (dict(criterion="entropy"), dict(criterion="log_loss"), dict(class_weight="balanced"),
                dict(max_leaf_nodes=10), dict(min_weight_fraction_leaf=0.1), dict(monotonic_cst=[1] * 12),
                dict(oob_score=True), dict(warm_start=True), dict(ccp_alpha=0.01)):
        name = next(iter(bad))
        with pytest.raises(ValueError, match=name):
            forest_fit_plan(bad, 100, 12)
        with pytest.raises(ValueError, match=name):   # refused before any library call
            tc.RandomForestClassifier(**bad)._fit_gpu(np.zeros((100, 12)), np.zeros(100), True)
    for bad in (dict(n_estimators=0), dict(max_depth=0), dict(min_samples_leaf=0), dict(min_samples_split=1),
                dict(max_features=13), dict(max_features="auto"), dict(bootstrap=False, max_samples=0.5),
                dict(max_samples=1.5), dict(min_impurity_decrease=-1.0)):
        with pytest.raises(ValueError):
            forest_fit_plan(bad, 100, 12)
    plan = forest_fit_plan(dict(n_jobs=-1, verbose=1, min_samples_leaf=0.05, min_samples_split=0.01), 1000, 12)
    assert plan["min_samples_leaf"] == 50 and plan["min_samples_split"] == 100 and plan["max_features"] == 3


def test_forest_fit_argument_errors_need_no_gpu():
    lib = _lib.load()
    out = C.c_void_p()
    seeds = np.zeros(2, np.uint32)
    x = np.zeros((4, 3))
    y = np.zeros(4, np.int32)
    args = lambda **k: dict(dict(x=x.ctypes.data_as(C.c_void_p), y=y.ctypes.data_as(C.c_void_p), n=4, d=3, C=2, dt=1, loc=0,
                                 T=2, boot=None, nb=0, seeds=seeds.ctypes.data_as(C.c_void_p), mf=1, md=10, mss=2, msl=1,
                                 mid=0.0, cap=0), **k)
    for bad in (dict(x=None), dict(y=None), dict(seeds=None), dict(d=0), dict(d=256), dict(C=33), dict(T=0),
                dict(mf=4), dict(mss=1), dict(msl=0), dict(mid=-1.0), dict(cap=-1), dict(loc=5)):
        a = args(**bad)
        assert lib.tcsdn_forest_fit(a["x"], a["y"], a["n"], a["d"], a["C"], a["dt"], a["loc"], a["T"], a["boot"], a["nb"],
                                    a["seeds"], a["mf"], a["md"], a["mss"], a["msl"], a["mid"], a["cap"], C.byref(out),
                                    None) == _lib.EINVAL, bad
