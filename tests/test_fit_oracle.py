"""tests/fit_oracle.py (the CPU definition of GaussianNB.fit and KMeans.fit that csrc/fit.cu computes) against
scikit-learn 1.9.0 on float64 rows.  Needs no GPU.

scikit-learn's own sums are rounded (numpy's pairwise order), so parameters are compared with a relative tolerance: theta
and the KMeans centres within 1e-12; variances and epsilon_ within 1e-12, because np.var on the flow columns, whose
squares reach 1e20, is itself about 1e-13 off the exact value.  KMeans labels and n_iter_ must be identical."""
import warnings

import numpy as np
import pytest

import fit_oracle as fo
from traffic_classifier_sdn_b200 import synth


def _sk_gnb(X, y):
    from sklearn.naive_bayes import GaussianNB
    return GaussianNB().fit(X, y)


def _sk_kmeans(X, init, **kw):
    from sklearn.cluster import KMeans
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")        # "Number of distinct clusters found smaller than n_clusters"
        return KMeans(n_clusters=len(init), init=init, n_init=1, algorithm="lloyd", **kw).fit(X)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), np.finfo(np.float64).tiny)))


def gnb_cases(golden):
    rng = np.random.default_rng(2)
    yield "golden", golden["X"], golden["y"]
    yield "flows", *synth.make_flows(20_000, seed=9)
    X, y = synth.make_flows(5_000, seed=4, d=8)
    y = y.copy()
    y[17] = 99                                     # a class with one row: var_ == epsilon_
    X = X.copy()
    X[:, 3] = 7.25                                 # a constant column
    yield "one_row_class_constant_column", X, y
    yield "offset_1e9", 1e9 + rng.standard_normal((3_000, 4)), rng.integers(0, 3, 3_000)
    yield "all_constant", np.full((50, 3), 2.5), np.arange(50) % 2


@pytest.mark.parametrize("case", ["golden", "flows", "one_row_class_constant_column", "offset_1e9", "all_constant"])
def test_gnb_definition_matches_sklearn(golden, case):
    name, X, y = next(c for c in gnb_cases(golden) if c[0] == case)
    ref = fo.gnb_fit(X, y)
    sk = _sk_gnb(X, y)
    assert np.array_equal(ref["classes"], sk.classes_)
    assert np.array_equal(ref["class_count"], sk.class_count_)
    assert np.array_equal(ref["class_prior"], sk.class_prior_)
    theta_ok = np.abs(ref["theta"] - sk.theta_) <= 1e-13 * np.abs(sk.theta_)
    assert theta_ok.all(), _rel(ref["theta"], sk.theta_)
    # np.var squares the error of its own rounded mean (up to gamma_n * |theta| on same-sign columns): at a 1e9 offset
    # that alone is ~1e-12 of a unit variance
    var_tol = 1e-12 * sk.var_ + (fo.gamma(len(X)) * np.abs(sk.theta_)) ** 2
    assert np.all(np.abs(ref["var"] - sk.var_) <= var_tol), _rel(ref["var"], sk.var_)
    assert abs(ref["epsilon"] - sk.epsilon_) <= 1e-12 * abs(sk.epsilon_)
    if case == "one_row_class_constant_column":
        c = list(ref["classes"]).index(99)
        assert np.all(ref["var"][c] == ref["epsilon"])                  # one row: variance 0, plus epsilon
        assert np.all(ref["var"][:, 3] == ref["epsilon"])
    if case == "all_constant":
        assert ref["epsilon"] == 0.0 and np.all(ref["var"] == 0.0)


def kmeans_cases(golden):
    """(name, X, init, kwargs, relocations expected)"""
    Xg = golden["X"]
    yield "golden", Xg, Xg[np.random.default_rng(3).choice(len(Xg), 4, replace=False)], {}, False
    X = synth.make_flows(20_000, seed=9, return_labels=False)
    init = X[np.random.default_rng(3).choice(len(X), 5, replace=False)].copy()
    init[2] = X.max(axis=0) * 3                    # nearest to no row
    yield "one_empty", X, init, {}, True
    init = init.copy()
    init[4] = X.max(axis=0) * 5
    yield "two_empty", X, init, {}, True
    # every row a duplicate, more clusters than distinct rows: nothing is relocated (all distances 0); the empty
    # clusters take the largest cluster's entry, before (averaged) or after (its centred sum) it in sklearn's loop
    D = np.array([[1.0, 2.0]] * 2 + [[5.0, 7.0]] * 3)
    yield "duplicates_largest_first", D, np.array([[1.0, 2.0], [5.0, 7.0], [0.0, 0.0], [100.0, 100.0]]), {}, False
    yield "duplicates_largest_last", D, np.array([[0.0, 0.0], [100.0, 100.0], [1.0, 2.0], [5.0, 7.0]]), {}, False
    # cluster 1's only row is the farthest row, so it moves to empty cluster 2 and leaves cluster 1 empty
    L = np.zeros((40, 2))
    L[:, 1] = np.arange(40) % 4
    L[-1] = [100.0, 1.0]
    yield "donor_loses_only_row", L, np.array([[0.0, 1.5], [60.0, 1.0], [1000.0, 1000.0]]), {}, True
    # exact ties on a lattice (centring on the mean 5 is exact): row x0 = 6 is equidistant from 3 and 9 in every
    # iteration and must go to cluster 0
    T = np.array([[a, b] for a in (0.0, 2.0, 4.0, 6.0, 8.0, 10.0) for b in (0.0, 1.0)] * 3)
    yield "lattice_ties", T, np.array([[3.0, 0.5], [9.0, 0.5]]), {}, False
    yield "max_iter_1", X, X[:6].copy(), {"max_iter": 1}, False
    yield "tol_0", Xg, Xg[np.random.default_rng(5).choice(len(Xg), 3, replace=False)], {"tol": 0.0}, False


KM_CASES = ["golden", "one_empty", "two_empty", "duplicates_largest_first", "duplicates_largest_last",
            "donor_loses_only_row", "lattice_ties", "max_iter_1", "tol_0"]


@pytest.mark.parametrize("case", KM_CASES)
def test_kmeans_definition_matches_sklearn(golden, case):
    name, X, init, kw, relocates = next(c for c in kmeans_cases(golden) if c[0] == case)
    ref = fo.kmeans_fit(X, init, **kw)
    sk = _sk_kmeans(X, init, **kw)
    assert np.array_equal(ref["labels"], sk.labels_)
    assert ref["n_iter"] == sk.n_iter_
    scale = np.abs(sk.cluster_centers_).max()
    assert np.all(np.abs(ref["centers"] - sk.cluster_centers_) <= 1e-12 * scale)
    assert abs(ref["inertia"] - sk.inertia_) <= 1e-12 * max(sk.inertia_, scale ** 2 * 1e-300)
    assert (ref["n_relocated"] > 0) == relocates
    if case == "lattice_ties":
        assert np.all(ref["labels"][X[:, 0] == 6.0] == 0)


def test_gnb_definition_is_exact_before_rounding():
    """theta_exact / var_exact are the exact rational moments: a class of two rows 1 and 2**-60 has mean
    (1 + 2**-60) / 2 exactly, which fp64 cannot hold"""
    from fractions import Fraction
    X = np.array([[1.0], [2.0 ** -60], [3.0]])
    ref = fo.gnb_fit(X, np.array([0, 0, 1]), var_smoothing=0.0)
    assert ref["theta_exact"][0][0] == (1 + Fraction(1, 2 ** 60)) / 2
    assert ref["var_exact"][0][0] == ((1 - Fraction(1, 2 ** 60)) / 2) ** 2
    assert ref["theta"][0, 0] == 0.5 and ref["var"][1, 0] == 0.0
