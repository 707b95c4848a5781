"""GaussianNB.fit and KMeans.fit on the GPU (csrc/fit.cu) at the shapes and cases where the fit kernels could go wrong,
held to the exact CPU definition in tests/fit_oracle.py.

Bars.  A sum of m fp64 terms, added in any order (per lane, then over lanes, then over blocks), is within
gamma_m * sum|term| of the exact sum (gamma_m = m u / (1 - m u), u = 2^-53), whatever the launch shape.  So:
* theta (and a KMeans centre) = fl(sum / cnt) is within gamma_{n+2} * sum|x| / cnt of the exact mean;
* var = fl(fl(sum (x - theta~)^2) / cnt) + epsilon: the exact variance plus (theta~ - theta)^2, each square carrying two
  roundings, so within gamma_{n+4} * sum (x - theta~)^2 / cnt + (theta tolerance)^2 + (epsilon tolerance) + 2u var;
* counts exact, class_prior_ == fl(count / n);
* KMeans labels_, n_iter_ and predict() identical to the definition.  The GPU E-step forms ||c||^2 - 2 x.c in d + d
  roundings, so on rows whose exact gap between nearest and second-nearest centre exceeds
  gamma_{2d+1} * (||c1||^2 + ||c2||^2 + 2 |x|.(|c1| + |c2|)) it cannot pick another centre; `_assert_margins` checks
  that the final centres give every row that gap (the lattice cases instead tie exactly, in exact arithmetic).
A float32 accumulator, or a dropped or doubled row or lane, breaks these bars by orders of magnitude."""
import ctypes as C

import numpy as np
import pytest

import fit_oracle as fo
import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import _lib, synth

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- GaussianNB ---------------------------------------------------------------------------------------------------

def _gnb_tolerances(X, yi, C, theta):
    """per-class (theta_tol [C][d], Q [C][d] >= sum (x - theta~)^2, cnt [C]) for rows X (float64) and labels yi"""
    n, d = X.shape
    A, Q, cnt = np.zeros((C, d)), np.zeros((C, d)), np.bincount(yi, minlength=C).astype(np.float64)
    for c in range(C):
        Xc = X[yi == c]
        A[c] = np.abs(Xc).sum(axis=0)
        Q[c] = ((Xc - theta[c]) ** 2).sum(axis=0)
    slack = 1.0 + 1e-6                                   # the numpy sums above are themselves rounded
    return fo.gamma(n + 2) * A * slack / cnt[:, None], Q * slack, cnt


def _check_gnb(est, X, y, var_smoothing=1e-9):
    """est (a GPU fit on X, y) against fo.gnb_fit within the bars in the module docstring"""
    X = np.asarray(X, np.float64)
    ref = fo.gnb_fit(X, y, var_smoothing)
    n, d = X.shape
    yi = np.searchsorted(ref["classes"], y)
    Cn = len(ref["classes"])
    assert np.array_equal(est.classes_, ref["classes"])
    assert np.array_equal(est.class_count_, ref["class_count"])
    assert np.array_equal(est.class_prior_, ref["class_prior"])
    th_tol, Q, cnt = _gnb_tolerances(X, yi, Cn, est.theta_)
    th_err = np.abs(est.theta_ - _exact(ref["theta_exact"]))
    assert np.all(th_err <= th_tol), f"theta off by {np.max(th_err / np.maximum(th_tol, 1e-300)):.3g} x its bound"
    at_tol, Qa, _ = _gnb_tolerances(X, np.zeros(n, np.int64), 1, X.mean(axis=0, keepdims=True))
    eps_tol = var_smoothing * float(np.max(fo.gamma(n + 4) * Qa[0] / n + at_tol[0] ** 2)) + 2 * U * ref["epsilon"]
    assert abs(est.epsilon_ - ref["epsilon"]) <= eps_tol + abs(float(ref["epsilon_exact"]) - ref["epsilon"])
    v_exact = _exact(ref["var_exact"]) + float(ref["epsilon_exact"])
    v_tol = fo.gamma(n + 4) * Q / cnt[:, None] + th_tol ** 2 + eps_tol + 2 * U * v_exact
    v_err = np.abs(est.var_ - v_exact)
    assert np.all(v_err <= v_tol), f"var off by {np.max(v_err / np.maximum(v_tol, 1e-300)):.3g} x its bound"
    return ref


def _exact(F):
    """Fractions -> float64, each correctly rounded (only used next to tolerances far above one rounding)"""
    return np.array([[float(v) for v in row] for row in F])


def _gnb_rows(n, d, C, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    scale = np.exp(rng.uniform(-3, 6, d))
    X = offset + rng.standard_normal((n, d)) * scale + rng.uniform(-50, 50, d) * scale
    y = np.arange(n) % C if n < 4 * C else rng.integers(0, C, n)
    y[:C] = np.arange(min(C, n))                        # every class present
    return X, y


@pytest.mark.parametrize("d", [1, 2, 12, 16, 17, 127, 128, 255])
def test_gnb_every_lane_split(d):
    """lanes = 256 // (d + 1): 128, 85, 19, 15, 14, 2, 1, 1 row lanes per block"""
    X, y = _gnb_rows(3_001, d, 3, seed=d)
    _check_gnb(tc.GaussianNB().fit(X, y, backend="gpu"), X, y)


def _block_edges():
    lanes = 256 // 13
    two_waves = 2 * _sms() * 1024
    return [1, 2, lanes - 1, lanes, lanes + 1, 1023, 1024, 1025, two_waves - 1, two_waves + 1]


def _abi_gnb_fit(X, y):
    """tcsdn_gnb_fit called directly (a model with a zero variance cannot be created, so the estimator cannot hold it)"""
    from types import SimpleNamespace
    classes, yi = np.unique(y, return_inverse=True)
    Cn, (n, d) = len(classes), X.shape
    yi = np.ascontiguousarray(yi, np.int32)
    th, var, pr, cnt, eps = np.empty((Cn, d)), np.empty((Cn, d)), np.empty(Cn), np.empty(Cn), C.c_double(0.0)
    f = _lib._f64p
    _lib.check(_lib.load().tcsdn_gnb_fit(X.ctypes.data_as(C.c_void_p), yi.ctypes.data_as(C.c_void_p), n, d, Cn, _lib.F64,
                                         _lib.HOST, 1e-9, th.ctypes.data_as(f), var.ctypes.data_as(f),
                                         pr.ctypes.data_as(f), cnt.ctypes.data_as(f), C.byref(eps), None))
    return SimpleNamespace(classes_=classes, theta_=th, var_=var, class_prior_=pr, class_count_=cnt, epsilon_=eps.value)


@pytest.mark.parametrize("which", range(10))
def test_gnb_every_block_split(which):
    """n around the lane count (d = 12: 19 lanes), one block (1024 rows) and the 2 x SMs block cap"""
    n = _block_edges()[which]
    d = 12 if n < 100_000 else 2
    X, y = _gnb_rows(n, d, 1 if n == 1 else 2, seed=n)
    _check_gnb(_abi_gnb_fit(X, y), X, y)


@pytest.mark.parametrize("C", [1, 2, 8, 32])
def test_gnb_class_counts(C):
    X, y = _gnb_rows(4_000, 12, C, seed=C)
    _check_gnb(tc.GaussianNB().fit(X, y, backend="gpu"), X, y)


@pytest.mark.parametrize("C,d", [(33, 12), (64, 12), (3, 256)])
def test_gnb_beyond_the_kernel_limits_is_sklearns_fit(C, d):
    """33+ classes or 256+ features: backend='auto' falls back to scikit-learn, backend='gpu' names the limit"""
    from sklearn.naive_bayes import GaussianNB as SK
    X, y = _gnb_rows(3_000, d, C, seed=C + d)
    sk = SK().fit(X, y)
    est = tc.GaussianNB().fit(X, y)
    assert np.array_equal(est.theta_, sk.theta_) and np.array_equal(est.var_, sk.var_)
    assert np.array_equal(est.predict(X), sk.predict(X))
    with pytest.raises(ValueError, match="at most 32 classes and 255 features"):
        tc.GaussianNB().fit(X, y, backend="gpu")


def test_gnb_content_edges():
    X, y = _gnb_rows(5_000, 6, 4, seed=7)
    y[123] = 9                                           # a class with one row
    X[:, 2] = 3.0                                        # a constant column
    est = tc.GaussianNB().fit(X, y, backend="gpu")
    _check_gnb(est, X, y)
    assert np.all(est.var_[-1] == est.epsilon_)          # one row: variance 0 + epsilon, exactly
    assert np.all(est.var_[:, 2] == est.epsilon_)
    # every column constant: epsilon 0 and variances 0, exactly.  Such a model cannot predict (tcsdn_gnb_create needs
    # var_ > 0), so the fit is read through the ABI and the estimator raises
    Z = np.full((300, 3), -1.75)
    yz = np.ascontiguousarray(np.arange(300) % 3, np.int32)
    th, var, pr, cnt, eps = np.empty((3, 3)), np.ones((3, 3)), np.empty(3), np.empty(3), C.c_double(1.0)
    f = _lib._f64p
    assert _lib.load().tcsdn_gnb_fit(Z.ctypes.data_as(C.c_void_p), yz.ctypes.data_as(C.c_void_p), 300, 3, 3, _lib.F64,
                                     _lib.HOST, 1e-9, th.ctypes.data_as(f), var.ctypes.data_as(f), pr.ctypes.data_as(f),
                                     cnt.ctypes.data_as(f), C.byref(eps), None) == _lib.OK
    assert eps.value == 0.0 and np.all(var == 0.0) and np.all(th == -1.75) and np.all(cnt == 100)
    with pytest.raises(ValueError):
        tc.GaussianNB().fit(Z, yz, backend="gpu")


def test_gnb_large_offset_needs_two_passes():
    """rows at 1e9 + N(0, 1): a one-pass E[x^2] - E[x]^2 variance would be off by ~1e2, the bound here is ~1e-5"""
    rng = np.random.default_rng(11)
    X = 1e9 + rng.standard_normal((40_000, 5))
    y = rng.integers(0, 3, 40_000)
    _check_gnb(tc.GaussianNB().fit(X, y, backend="gpu"), X, y)


def test_gnb_float32_and_device_rows():
    import torch
    X, y = _gnb_rows(20_000, 12, 5, seed=3)
    X32 = X.astype(np.float32)
    est = tc.GaussianNB().fit(X32, y, backend="gpu")
    _check_gnb(est, X32.astype(np.float64), y)           # float32 rows are fitted in fp64: the widened rows' fit
    dev = tc.GaussianNB().fit(torch.from_numpy(X32).cuda(), torch.from_numpy(y).cuda(), backend="gpu")
    for a in ("theta_", "var_", "class_prior_", "class_count_"):
        assert np.array_equal(getattr(dev, a), getattr(est, a)), a
    assert dev.epsilon_ == est.epsilon_


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
def test_gnb_nonfinite_rows_raise(bad):
    X, y = _gnb_rows(2_000, 4, 2, seed=1)
    X[1500, 1] = bad
    with pytest.raises(ValueError):
        tc.GaussianNB().fit(X, y, backend="gpu")


@pytest.mark.parametrize("bad", [-1, 3])
def test_gnb_abi_rejects_y_out_of_range(bad):
    X, y = _gnb_rows(2_000, 4, 3, seed=2)
    yi = np.ascontiguousarray(y, np.int32)
    yi[777] = bad
    out = [np.empty((3, 4)), np.empty((3, 4)), np.empty(3), np.empty(3)]
    f = _lib._f64p
    rc = _lib.load().tcsdn_gnb_fit(X.ctypes.data_as(C.c_void_p), yi.ctypes.data_as(C.c_void_p), len(X), 4, 3, _lib.F64,
                                   _lib.HOST, 1e-9, *[o.ctypes.data_as(f) for o in out], None, None)
    assert rc == _lib.EINVAL


def test_gnb_million_rows_permutation():
    """1M + 1 rows (the fit's largest block split): theta within the sum bound of the math.fsum mean, and a permutation
    of the rows moves theta and var by no more than twice the bound"""
    import math
    X, y = _gnb_rows(1_000_001, 4, 3, seed=5)
    est = tc.GaussianNB().fit(X, y, backend="gpu")
    th_tol, Q, cnt = _gnb_tolerances(X, y, 3, est.theta_)
    for c in range(3):
        Xc = X[y == c]
        ref = np.array([math.fsum(Xc[:, j].tolist()) / len(Xc) for j in range(4)])
        assert np.all(np.abs(est.theta_[c] - ref) <= th_tol[c] + 2 * U * np.abs(ref))
        assert est.class_count_[c] == len(Xc)
    p = np.random.default_rng(0).permutation(len(X))
    sh = tc.GaussianNB().fit(X[p], y[p], backend="gpu")
    assert np.all(np.abs(sh.theta_ - est.theta_) <= 2 * th_tol)
    v_tol = fo.gamma(len(X) + 4) * Q / cnt[:, None] + th_tol ** 2 + 2 * U * est.var_
    assert np.all(np.abs(sh.var_ - est.var_) <= 2 * v_tol)


# ---- KMeans -------------------------------------------------------------------------------------------------------

def _assert_margins(X, centers, labels):
    """every row's exact gap to its second-nearest centre exceeds the E-step's rounding bound (module docstring)"""
    X = np.asarray(X, np.float64)
    n, d = X.shape
    if len(centers) == 1:
        return
    D = fo._sq_dist(X, centers)
    ax, ac = np.abs(X), np.abs(centers)
    E = fo.gamma(2 * d + 1) * ((centers ** 2).sum(axis=1)[None, :] + 2 * ax @ ac.T)
    best = D[np.arange(n), labels]
    gap = D - best[:, None]
    need = E + E[np.arange(n), labels][:, None] + fo.gamma(d + 3) * (D + best[:, None])
    gap[np.arange(n), labels] = np.inf
    assert np.all(gap > need), f"{int(np.sum(np.any(gap <= need, axis=1)))} rows too close to call"


def _check_kmeans(est, X, init, margins=True, **kw):
    X = np.asarray(X, np.float64)
    ref = fo.kmeans_fit(X, init, **kw)
    n, d = X.shape
    k = len(init)
    assert np.array_equal(est.labels_, ref["labels"])
    assert est.n_iter_ == ref["n_iter"]
    assert np.array_equal(est.predict(X), ref["labels"])
    if margins:
        _assert_margins(X, ref["centers"], ref["labels"])
    # centres: the sum bound over the last M-step's counts, with sum|x| over all rows (which also covers a relocated
    # row leaving its donor's sum, and the copy rule's sum(x) - (count - 1) * mean for clusters left at count 0)
    A = (np.abs(X).sum(axis=0) + n * np.abs(X.mean(axis=0))) * (1 + 1e-6)
    cnt = np.asarray(ref["counts"], np.float64)
    tol = fo.gamma(n + 4) * A[None, :] / np.maximum(cnt, 0.5)[:, None]
    err = np.abs(est.cluster_centers_ - _exact(ref["centers_exact"]))
    assert np.all(err <= tol), f"centres off by {np.max(err / np.maximum(tol, 1e-300)):.3g} x their bound"
    I = fo.inertia(X, est.cluster_centers_, est.labels_)
    assert abs(est.inertia_ - I) <= fo.gamma(n + k * d + 4) * I
    return ref


def _blobs(n, d, k, seed, spread=100.0):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-spread, spread, (k, d)) * np.sqrt(k)
    if d == 1:
        centres[:, 0] = np.arange(k) * spread
    lab = rng.integers(0, k, n)
    X = centres[lab] + rng.standard_normal((n, d))
    init = centres + rng.standard_normal((k, d)) * 2.0
    return X, init


@pytest.mark.parametrize("k", [1, 2, 33])
@pytest.mark.parametrize("d", [1, 12, 255])
def test_kmeans_shapes(k, d):
    X, init = _blobs(6_000 if d < 255 else 2_000, d, k, seed=k * 1000 + d)
    est = tc.KMeans(n_clusters=k, init=init, n_init=1).fit(X, backend="gpu")
    _check_kmeans(est, X, init)


def _flows_with_unreachable(m):
    X = synth.make_flows(20_000, seed=9, return_labels=False)
    init = X[np.random.default_rng(3).choice(len(X), 5, replace=False)].copy()
    init[2] = X.max(axis=0) * 3
    if m == 2:
        init[4] = X.max(axis=0) * 5
    return X, init


@pytest.mark.parametrize("m", [1, 2])
def test_kmeans_relocates_empty_clusters(m):
    """init centres nearest to no row: each empty cluster takes the row farthest from its centre (sklearn's
    _relocate_empty_clusters_dense)"""
    X, init = _flows_with_unreachable(m)
    est = tc.KMeans(n_clusters=5, init=init, n_init=1).fit(X, backend="gpu")
    ref = _check_kmeans(est, X, init, margins=False)
    assert ref["n_relocated"] == m and np.all(np.bincount(est.labels_, minlength=5) > 0)
    Xb, ib = _blobs(8_000, 6, 5, seed=m)
    ib[1] = 1e4                                          # and on blobs, where the margins are checked
    est = tc.KMeans(n_clusters=5, init=ib, n_init=1).fit(Xb, backend="gpu")
    assert _check_kmeans(est, Xb, ib)["n_relocated"] >= 1


@pytest.mark.parametrize("order", ["largest_first", "largest_last"])
def test_kmeans_more_clusters_than_distinct_rows(order):
    """every row a duplicate of one of 3 points, k = 5: nothing to relocate; the empty clusters take the largest
    cluster's entry as sklearn's averaging loop leaves it"""
    P = np.array([[1.0, 2.0, 0.5], [5.0, 7.0, -1.0], [-3.0, 4.0, 2.0]])
    X = P[np.arange(3_000) % 3 if order == "largest_first" else np.minimum(np.arange(3_000) // 900, 2)]
    far = np.array([[0.0, 0.0, 0.0], [100.0, 100.0, 100.0]])
    init = np.vstack([P, far]) if order == "largest_first" else np.vstack([far, P])
    est = tc.KMeans(n_clusters=5, init=init, n_init=1).fit(X, backend="gpu")
    ref = _check_kmeans(est, X, init, margins=False)
    assert ref["n_relocated"] == 0
    if order == "largest_first":                         # copies of dyadic means: exact.  Otherwise the copied value
        assert np.array_equal(est.cluster_centers_, ref["centers"])   # holds (count - 1) * mean(X), 0.6 here: rounded


def test_kmeans_donor_loses_its_only_row():
    L = np.zeros((400, 2))
    L[:, 1] = np.arange(400) % 4
    L[-1] = [100.0, 1.0]
    init = np.array([[0.0, 1.5], [60.0, 1.0], [1000.0, 1000.0]])
    est = tc.KMeans(n_clusters=3, init=init, n_init=1).fit(L, backend="gpu")
    ref = _check_kmeans(est, L, init, margins=False)
    assert ref["n_relocated"] >= 1 and np.array_equal(est.cluster_centers_, ref["centers"])   # small integers: exact


def test_kmeans_lattice_ties_go_to_the_lower_index():
    """rows at x0 = 6 are exactly equidistant from centres 3 and 9 in every iteration (dyadic means, exact arithmetic)"""
    T = np.array([[a, b] for a in (0.0, 2.0, 4.0, 6.0, 8.0, 10.0) for b in (0.0, 1.0)] * 500)
    init = np.array([[3.0, 0.5], [9.0, 0.5]])
    est = tc.KMeans(n_clusters=2, init=init, n_init=1).fit(T, backend="gpu")
    _check_kmeans(est, T, init, margins=False)
    assert np.all(est.labels_[T[:, 0] == 6.0] == 0)
    assert np.array_equal(est.cluster_centers_, [[3.0, 0.5], [9.0, 0.5]])


@pytest.mark.parametrize("kw", [{"max_iter": 1}, {"tol": 0.0}])
def test_kmeans_stopping_rules(kw):
    X, init = _blobs(10_000, 4, 6, seed=31)
    init = init + 30.0                                   # several iterations to go
    est = tc.KMeans(n_clusters=6, init=init, n_init=1, **kw).fit(X, backend="gpu")
    ref = _check_kmeans(est, X, init, **kw)
    if "max_iter" in kw:
        assert ref["n_iter"] == 1


def test_kmeans_float32_rows_are_fitted_widened():
    from sklearn.cluster import KMeans as SK
    X, init = _blobs(12_000, 12, 7, seed=4)
    X32 = X.astype(np.float32)
    est = tc.KMeans(n_clusters=7, init=init, n_init=1).fit(X32, backend="gpu")
    _check_kmeans(est, X32.astype(np.float64), init)
    sk = SK(n_clusters=7, init=init, n_init=1).fit(X32.astype(np.float64))
    assert np.array_equal(est.labels_, sk.labels_) and est.n_iter_ == sk.n_iter_


@pytest.mark.parametrize("m", [0, 1])
def test_kmeans_device_rows_and_determinism(m):
    """CUDA-tensor rows: labels_ present, and every result bit-identical to the host-rows fit and to a second run"""
    import torch
    X, init = _flows_with_unreachable(1) if m else _blobs(30_000, 12, 9, seed=8)
    k = len(init)
    host = tc.KMeans(n_clusters=k, init=init, n_init=1).fit(X, backend="gpu")
    again = tc.KMeans(n_clusters=k, init=init, n_init=1).fit(X, backend="gpu")
    dev = tc.KMeans(n_clusters=k, init=init, n_init=1).fit(torch.from_numpy(X).cuda(), backend="gpu")
    for other in (again, dev):
        assert isinstance(other.labels_, np.ndarray) and other.labels_.dtype == np.int32
        assert np.array_equal(other.labels_, host.labels_)
        assert np.array_equal(other.cluster_centers_, host.cluster_centers_)
        assert other.inertia_ == host.inertia_ and other.n_iter_ == host.n_iter_


def test_kmeans_256_features_is_sklearns_fit():
    from sklearn.cluster import KMeans as SK
    X, init = _blobs(1_000, 256, 3, seed=2)
    sk = SK(n_clusters=3, init=init, n_init=1).fit(X)
    est = tc.KMeans(n_clusters=3, init=init, n_init=1).fit(X)
    assert np.array_equal(est.labels_, sk.labels_)
    np.testing.assert_allclose(est.cluster_centers_, sk.cluster_centers_, rtol=1e-12)   # sklearn's threads add in any order
    with pytest.raises(ValueError, match="at most 255 features"):
        tc.KMeans(n_clusters=3, init=init, n_init=1).fit(X, backend="gpu")
