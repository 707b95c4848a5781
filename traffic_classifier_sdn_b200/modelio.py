"""Model import: fitted estimators -> flat parameter specs the CUDA library packs to HBM.

This is boundary row a7 of SURVEY.md section 8: the reference obtains its model with
``model = pickle.load(infile)`` (reference ``traffic_classifier.py:243``) from one of the
six files under ``models/`` (``traffic_classifier.py:229-240``).  Those files are
scikit-learn 1.0.1 pickles; two of them (``KNeighbors`` and ``RandomForestClassifier``)
no longer unpickle under the scikit-learn shipped in this image because private Cython
classes moved or changed their node dtype.  Nothing here needs scikit-learn: the
unpickler below resolves every ``sklearn.*`` global to an inert attribute bag, so a
reference pickle is read as *data* (numpy arrays and scalars), never as code.

A "spec" is a plain dict of numpy arrays/scalars with a ``kind`` key:

=========  ==========================================================================
kind       keys
=========  ==========================================================================
linear     coef [R,d] f64, intercept [R] f64, classes  (R == 1 means binary), ovr (bool:
           one-vs-rest probabilities)
gnb        theta [C,d], var [C,d], class_prior [C], classes
kmeans     centers [k,d]
knn        fit_X [n_t,d] f64, y [n_t] int32 (class index), k, classes, weights ("uniform" or
           "distance"; a spec without the key is uniform), metric ("euclidean", "manhattan" or
           "chebyshev"; a spec without the key is euclidean)
svc        sv [nSV,d], dual_coef [C-1,nSV], intercept [P], n_support [C] int32,
           gamma, classes, decision_function_shape, break_ties, kernel ("linear", "poly", "rbf" or
           "sigmoid"; a spec without the key is rbf), coef0, degree, prob_a / prob_b [P] f64 (probA_ /
           probB_: the Platt parameters of a probability=True model; absent for other models)
forest     tree_offsets [T+1] int64, left/right/feature int32 [N], threshold f64 [N],
           value [N,C] f64 (per-node class fractions), classes
=========  ==========================================================================
"""
from __future__ import annotations

import io
import pickle
from typing import Any, Dict

import numpy as np

__all__ = ["load_reference_pickle", "spec_from_estimator", "spec_from_pickle_bytes",
           "knn_weights", "knn_metric", "svc_kernel", "svc_platt", "MODEL_FILES", "SpecError"]

# argv word -> pickle file, as dispatched at reference traffic_classifier.py:229-240
MODEL_FILES = {
    "logistic": "LogisticRegression",
    "kmeans": "KMeans_Clustering",
    "svm": "SVC",
    "kneighbors": "KNeighbors",
    "Randomforest": "RandomForestClassifier",
    "gaussiannb": "GaussianNB",
}


class SpecError(ValueError):
    """The estimator uses an option the CUDA path does not implement."""


class _Bag:
    """Inert stand-in for any sklearn class found in a pickle stream."""

    def __init__(self, *args, **kwargs):
        self._ctor_args = args

    def __setstate__(self, state):
        # sklearn estimators pickle their __dict__; Cython classes pickle dicts or tuples
        if isinstance(state, dict):
            self.__dict__.update(state)
        else:
            self._state = state


def _new_obj(cls, *args):  # replaces sklearn.neighbors.*.newObj (Cython __reduce__ helper)
    return cls.__new__(cls)


class _DataOnlyUnpickler(pickle.Unpickler):
    _NUMPY_OK = {
        ("numpy.core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "_reconstruct"),
        ("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar"),
        ("numpy", "ndarray"), ("numpy", "dtype"),
        ("numpy.core.numeric", "_frombuffer"), ("numpy._core.numeric", "_frombuffer"),
    }

    def find_class(self, module, name):
        if module.split(".")[0] == "sklearn":
            if name == "newObj":
                return _new_obj
            return type(name, (_Bag,), {"_sk_module": module})
        if (module, name) in self._NUMPY_OK:
            return super().find_class(module.replace("numpy.core", "numpy._core"), name)
        if module in ("builtins", "copyreg", "collections") and name in (
                "dict", "list", "tuple", "set", "frozenset", "slice", "range", "complex",
                "_reconstructor", "object", "OrderedDict", "bytearray"):
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"refusing to load global {module}.{name}")


def spec_from_pickle_bytes(data: bytes) -> Dict[str, Any]:
    obj = _DataOnlyUnpickler(io.BytesIO(data)).load()
    return _spec_from_attrs(type(obj).__name__, obj)


def load_reference_pickle(path: str) -> Dict[str, Any]:
    """Read one of the reference's ``models/*`` files into a spec (no sklearn needed)."""
    with open(path, "rb") as fh:
        return spec_from_pickle_bytes(fh.read())


def spec_from_estimator(est) -> Dict[str, Any]:
    """Spec from a live, fitted scikit-learn estimator (the ``.fit`` route)."""
    return _spec_from_attrs(type(est).__name__, est)


# --------------------------------------------------------------------------------------
def _f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def _classes(obj):
    c = getattr(obj, "classes_", None)
    return None if c is None else np.asarray(c)


def _tree_arrays(tree):
    """(left, right, feature, threshold, value[N,C]) from a live Tree or an unpickled bag."""
    if hasattr(tree, "children_left"):  # live sklearn.tree._tree.Tree
        nodes_left = np.asarray(tree.children_left)
        nodes_right = np.asarray(tree.children_right)
        feature = np.asarray(tree.feature)
        threshold = np.asarray(tree.threshold)
        value = np.asarray(tree.value)
    else:  # _Bag: state dict {max_depth,node_count,nodes,values} (sk:tree/_tree.pyx __getstate__)
        nodes = tree.nodes
        nodes_left, nodes_right = nodes["left_child"], nodes["right_child"]
        feature, threshold = nodes["feature"], nodes["threshold"]
        value = tree.values
    value = np.asarray(value, dtype=np.float64)
    if value.ndim != 3 or value.shape[1] != 1:
        raise SpecError("multi-output forests are not supported")
    value = value[:, 0, :]
    # sklearn <= 1.3 stored weighted class counts and normalised at predict time
    # (proba /= proba.sum(axis=1)); >= 1.4 stores fractions (sk:tree/_classes.py:1052-1055).
    # count / sum is a single fp64 division in both, so per-node normalisation is identical.
    s = value.sum(axis=1, keepdims=True)
    needs = np.abs(s - 1.0) > 1e-9
    value = np.where(needs & (s != 0.0), value / np.where(s == 0.0, 1.0, s), value)
    return (np.asarray(nodes_left, np.int32), np.asarray(nodes_right, np.int32),
            np.asarray(feature, np.int32), _f64(threshold), np.ascontiguousarray(value))


def knn_weights(w) -> str:
    """KNeighborsClassifier's ``weights`` as a spec value: "uniform" (also for None, sklearn's older spelling) or
    "distance".  A callable cannot become a kernel and is refused."""
    if w is None or (isinstance(w, str) and w == "uniform"):
        return "uniform"
    if isinstance(w, str) and w == "distance":
        return "distance"
    if callable(w):
        raise SpecError("callable weights are not implemented (weights must be 'uniform' or 'distance')")
    raise SpecError(f"weights must be 'uniform' or 'distance', got {w!r}")


_KNN_METRIC_NAMES = {"euclidean": "euclidean", "l2": "euclidean", "manhattan": "manhattan", "cityblock": "manhattan",
                     "l1": "manhattan", "chebyshev": "chebyshev", "infinity": "chebyshev"}
_KNN_MINKOWSKI_P = {1: "manhattan", 2: "euclidean", np.inf: "chebyshev"}


def knn_metric(metric, p=2, metric_params=None) -> str:
    """KNeighborsClassifier's metric as a spec value: "euclidean", "manhattan" or "chebyshev".  Takes scikit-learn's
    spellings of the three (manhattan = cityblock = l1 = minkowski with p=1, chebyshev = infinity = minkowski with p=inf,
    euclidean = l2 = minkowski with p=2; ``metric_params`` may hold ``p``, which overrides ``p`` as in scikit-learn).
    Everything else is refused: minkowski with another p (libm's pow and CUDA's are not bit-identical), weights ``w``,
    other metrics and callables."""
    params = {key: v for key, v in dict(metric_params or {}).items() if not (key == "w" and v is None)}
    supported = "the supported metrics are 'euclidean', 'manhattan' and 'chebyshev'"
    extra = sorted(set(params) - {"p"})
    if extra:
        raise SpecError(f"metric_params {extra} are not implemented; {supported}")
    if callable(metric) or not isinstance(metric, str):
        raise SpecError(f"metric {metric!r} is not implemented; {supported}")
    if metric == "minkowski":
        p = params.get("p", p)
        try:
            name = _KNN_MINKOWSKI_P.get(float(p))
        except (TypeError, ValueError):
            name = None
        if name is None:
            raise SpecError(f"minkowski with p={p!r} is not implemented; {supported} (minkowski with p=1, 2 or inf)")
        return name
    if metric not in _KNN_METRIC_NAMES:
        raise SpecError(f"metric {metric!r} is not implemented; {supported}")
    return _KNN_METRIC_NAMES[metric]


def svc_kernel(k) -> str:
    """SVC's ``kernel`` as a spec value: one of libsvm's four built-in kernels.  'precomputed' and callables need the
    training rows at predict time and are refused."""
    if callable(k):
        raise SpecError("callable kernels are not implemented (kernel must be 'linear', 'poly', 'rbf' or 'sigmoid')")
    if isinstance(k, str) and k in ("linear", "poly", "rbf", "sigmoid"):
        return k
    raise SpecError(f"kernel must be 'linear', 'poly', 'rbf' or 'sigmoid', got {k!r}")


def svc_platt(prob_a, prob_b, n_classes):
    """SVC's Platt parameters (probA_, probB_) as spec values: None when both are missing or empty (a model fitted with
    probability=False), else two contiguous float64 arrays of n_classes * (n_classes - 1) / 2 finite values."""
    a = np.zeros(0) if prob_a is None else np.asarray(prob_a, dtype=np.float64).ravel()
    b = np.zeros(0) if prob_b is None else np.asarray(prob_b, dtype=np.float64).ravel()
    if a.size == 0 and b.size == 0:
        return None
    P = n_classes * (n_classes - 1) // 2
    if a.size != P or b.size != P:
        raise SpecError(f"probA_ / probB_ must hold {P} values each (one per class pair), got {a.size} and {b.size}")
    if not (np.isfinite(a).all() and np.isfinite(b).all()):
        raise SpecError("probA_ / probB_ must be finite")
    return np.ascontiguousarray(a), np.ascontiguousarray(b)


def _spec_from_attrs(name: str, o) -> Dict[str, Any]:
    if name == "LogisticRegression":
        coef = _f64(o.coef_)
        # one-vs-rest models (multi_class='ovr', or 'auto' with the liblinear solver, in the scikit-learn releases that
        # still had the option) turn scores into probabilities with normalised sigmoids, not a softmax
        # (sk:linear_model/_base.py:429-451 against sk:linear_model/_logistic.py:1620-1625); labels are the same
        mc, solver = str(getattr(o, "multi_class", "auto")), str(getattr(o, "solver", "lbfgs"))
        ovr = mc in ("ovr", "warn") or (mc == "auto" and solver == "liblinear")
        return dict(kind="linear", coef=coef, intercept=_f64(np.broadcast_to(o.intercept_, (coef.shape[0],))),
                    classes=_classes(o), n_features=coef.shape[1], ovr=bool(ovr))
    if name == "GaussianNB":
        var = getattr(o, "var_", None)
        if var is None:
            var = o.sigma_  # attribute name before sklearn 1.0
        return dict(kind="gnb", theta=_f64(o.theta_), var=_f64(var), class_prior=_f64(o.class_prior_),
                    classes=_classes(o), n_features=int(np.asarray(o.theta_).shape[1]))
    if name == "KMeans":
        c = _f64(o.cluster_centers_)
        return dict(kind="kmeans", centers=c, classes=np.arange(c.shape[0], dtype=np.int32),
                    n_features=c.shape[1])
    if name == "KNeighborsClassifier":
        weights = knn_weights(getattr(o, "weights", "uniform"))
        # scikit-learn fixes the metric at fit: effective_metric_ / effective_metric_params_ (sk:neighbors/_base.py:527-552)
        if hasattr(o, "effective_metric_"):
            metric = knn_metric(o.effective_metric_, getattr(o, "p", 2), getattr(o, "effective_metric_params_", None))
        else:
            metric = knn_metric(getattr(o, "metric", "minkowski"), getattr(o, "p", 2), getattr(o, "metric_params", None))
        fx = _f64(o._fit_X)
        y = np.asarray(o._y)
        if y.ndim != 1:
            raise SpecError("multi-output KNN is not supported")
        return dict(kind="knn", fit_X=fx, y=np.ascontiguousarray(y, dtype=np.int32),
                    k=int(o.n_neighbors), classes=_classes(o), n_features=fx.shape[1], weights=weights, metric=metric)
    if name == "SVC":
        kernel = svc_kernel(getattr(o, "kernel", "rbf"))   # pickles without the attribute are rbf models
        if getattr(o, "_sparse", False):
            raise SpecError("sparse SVC is not supported")
        sv = _f64(o.support_vectors_)
        cls = _classes(o)
        C = len(cls)
        # libsvm's own sign convention lives in the private attributes (sk:svm/_base.py:259-266):
        # for two classes the public intercept_/dual_coef_ are negated copies.
        dual = _f64(getattr(o, "_dual_coef_", o.dual_coef_))
        icpt = _f64(getattr(o, "_intercept_", o.intercept_))
        nsup = np.asarray(getattr(o, "_n_support", getattr(o, "n_support_", None)), dtype=np.int32)
        spec = dict(kind="svc", sv=sv, dual_coef=dual, intercept=icpt, n_support=np.ascontiguousarray(nsup),
                    gamma=float(o._gamma), classes=cls, n_features=sv.shape[1],
                    decision_function_shape=str(o.decision_function_shape),
                    break_ties=bool(getattr(o, "break_ties", False)), n_classes=C, kernel=kernel,
                    coef0=float(getattr(o, "coef0", 0.0)), degree=int(getattr(o, "degree", 3)))
        # Platt parameters of a probability=True fit (sk:svm/_base.py: _probA / _probB, public as probA_ / probB_)
        # (the private names first: scikit-learn 1.9 warns on every read of the deprecated public ones)
        pa, pb = getattr(o, "_probA", None), getattr(o, "_probB", None)
        if pa is None and pb is None:
            pa, pb = getattr(o, "probA_", None), getattr(o, "probB_", None)
        platt = svc_platt(pa, pb, C)
        if platt is not None:
            spec["prob_a"], spec["prob_b"] = platt
        return spec
    if name == "RandomForestClassifier":
        cls = _classes(o)
        if cls is None or (len(cls) and isinstance(cls[0], np.ndarray)):
            raise SpecError("multi-output forests are not supported")
        lefts, rights, feats, thrs, vals, offs = [], [], [], [], [], [0]
        nfeat = None
        for est in o.estimators_:
            t = est.tree_
            l, r, f, th, v = _tree_arrays(t)
            if v.shape[1] != len(cls):
                raise SpecError("tree class count differs from forest class count")
            lefts.append(l); rights.append(r); feats.append(f); thrs.append(th); vals.append(v)
            offs.append(offs[-1] + len(l))
            nf = getattr(t, "n_features", None)
            if nf is None and getattr(t, "_ctor_args", None):
                nf = t._ctor_args[0]
            nfeat = nf if nfeat is None else nfeat
        nfeat = int(getattr(o, "n_features_in_", nfeat))
        return dict(kind="forest", tree_offsets=np.asarray(offs, np.int64),
                    left=np.concatenate(lefts), right=np.concatenate(rights),
                    feature=np.concatenate(feats), threshold=np.concatenate(thrs),
                    value=np.ascontiguousarray(np.concatenate(vals, axis=0)), classes=cls,
                    n_features=nfeat)
    raise SpecError(f"unsupported estimator type {name}")
