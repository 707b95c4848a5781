"""sklearn-like estimators whose ``predict`` runs on the H100 through libtcsdn.so.

These classes are the drop-in for the objects the reference gets from ``pickle.load`` at
``traffic_classifier.py:243`` and calls at ``traffic_classifier.py:106``
(``label = model.predict(features.tolist())``).  The duck type kept is scikit-learn's:

* ``fit(X, y=None) -> self``; ``predict(X) -> ndarray[n]`` of ``classes_`` dtype (int32 cluster ids for
  KMeans); ``classes_``, ``n_features_in_``; ``decision_function`` (LogisticRegression, SVC),
  ``predict_proba`` (GaussianNB, KNeighborsClassifier, RandomForestClassifier, SVC(probability=True)), ``predict_log_proba`` /
  ``transform`` where sklearn has them and they are a closed form of the kernel's score matrix;
  ``kneighbors`` (KNeighborsClassifier);
* ``ValueError`` on a wrong feature count or NaN/inf input, ``NotFittedError`` before ``fit``;
  inputs are never modified, outputs are freshly allocated.

``fit`` trains on the host with scikit-learn (training is outside the hot path, SURVEY.md 8b) and
imports the fitted attributes; ``from_sklearn`` / ``from_spec`` / ``load_model`` import an existing
model.  Inference never touches scikit-learn or the CPU: without libtcsdn.so or without a GPU,
``predict`` raises.

Beyond sklearn: ``predict_indices(X)`` returns int32 class indices and accepts a CUDA ``torch.Tensor``
(rows already in HBM, result stays on the device, asynchronous on the current stream).
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, Optional

import numpy as np

from . import _lib, modelio

try:  # sklearn's exception type, so that reference-side `except NotFittedError` keeps working
    from sklearn.exceptions import NotFittedError
except Exception:  # pragma: no cover - sklearn absent
    class NotFittedError(ValueError, AttributeError):
        pass

__all__ = ["LogisticRegression", "GaussianNB", "KMeans", "KNeighborsClassifier", "SVC",
           "RandomForestClassifier", "from_spec", "from_sklearn", "load_model", "NotFittedError"]


def _is_torch_cuda(x) -> bool:
    return type(x).__module__.startswith("torch") and hasattr(x, "is_cuda") and bool(x.is_cuda)


class _Base:
    _kind = ""
    _sk_name = ""

    def __init__(self, **params):
        self._params = dict(params)
        self._handle = None
        self._spec: Optional[Dict[str, Any]] = None
        self._device = None

    # ---- sklearn-ish plumbing -------------------------------------------------------------------
    def get_params(self, deep=True):
        return dict(self._params)

    def set_params(self, **params):
        self._params.update(params)
        return self

    def __repr__(self):
        args = ", ".join(f"{k}={v!r}" for k, v in self._params.items())
        return f"{type(self).__name__}({args})"

    def __del__(self):
        self._release()

    def _release(self):
        h, self._handle = self._handle, None
        if h is not None:
            try:
                _lib.load().tcsdn_destroy(h)
            except Exception:
                pass

    def __getstate__(self):  # picklable like the sklearn objects it replaces: parameters only
        return {"params": self._params, "spec": self._spec}

    def __setstate__(self, state):
        self._params = state["params"]
        self._handle = None
        self._spec = None
        self._device = None
        if state["spec"] is not None:
            self._adopt(state["spec"])

    def _check_fitted(self):
        if self._handle is None:
            raise NotFittedError(f"This {type(self).__name__} instance is not fitted yet. Call 'fit' with "
                                 "appropriate arguments before using this estimator.")

    # ---- model import ---------------------------------------------------------------------------
    def _sk_estimator(self):
        raise NotImplementedError

    def fit(self, X, y=None, backend="auto"):
        """Train, then move the fitted parameters to HBM.  GaussianNB and KMeans fit on the GPU (SURVEY row N3,
        csrc/fit.cu) unless ``backend="sklearn"``; the other four train with scikit-learn on the host."""
        if backend not in ("auto", "gpu", "sklearn"):
            raise ValueError("backend must be 'auto', 'gpu' or 'sklearn'")
        if backend != "sklearn" and self._fit_gpu(X, y, strict=backend == "gpu"):
            return self
        est = self._sk_estimator()
        est.fit(X) if y is None and self._kind == "kmeans" else est.fit(X, y)
        self._adopt(modelio.spec_from_estimator(est))
        for attr in ("n_iter_", "inertia_", "labels_", "feature_names_in_"):
            if hasattr(est, attr):
                setattr(self, attr, getattr(est, attr))
        return self

    def _fit_gpu(self, X, y, strict):
        """-> True when the GPU fitted the model.  Estimators without a GPU fit return False (or raise if strict)."""
        if strict:
            raise ValueError(f"{type(self).__name__} has no GPU fit: it trains with scikit-learn on the host")
        return False

    @staticmethod
    def _fit_rows(X):
        """-> (pointer, n, d, dtype code, loc code, keepalive) for a fit call: numpy rows or a CUDA torch tensor."""
        if _is_torch_cuda(X):
            t = X.contiguous()
            if t.dim() != 2 or str(t.dtype) not in ("torch.float32", "torch.float64"):
                raise ValueError("expected a 2-D float32/float64 CUDA tensor")
            return C.c_void_p(t.data_ptr()), t.shape[0], t.shape[1], _lib.F32 if str(t.dtype) == "torch.float32" else _lib.F64, \
                _lib.DEVICE, t
        a = np.asarray(X)
        if a.ndim != 2:
            raise ValueError(f"Expected 2D array, got {a.ndim}D array instead")
        a = np.ascontiguousarray(a, dtype=np.float32 if a.dtype == np.float32 else np.float64)
        return _p(a, C.c_void_p), a.shape[0], a.shape[1], _lib.F32 if a.dtype == np.float32 else _lib.F64, _lib.HOST, a

    def _adopt(self, spec):
        if spec["kind"] != self._kind:
            raise ValueError(f"{type(self).__name__} cannot adopt a '{spec['kind']}' model")
        self._release()
        self._spec = spec
        self.n_features_in_ = int(spec["n_features"])
        self.classes_ = np.asarray(spec["classes"])
        lib = _lib.load()
        h = C.c_void_p()
        self._create(lib, spec, h)
        self._handle = h
        self._score_cols = int(lib.tcsdn_model_score_cols(h))
        return self

    def _create(self, lib, spec, h):
        raise NotImplementedError

    def set_option(self, key: int, value: int):
        self._check_fitted()
        _lib.check(_lib.load().tcsdn_set_option(self._handle, key, int(value)))
        return self

    def stats(self):
        self._check_fitted()
        out = np.zeros(8, np.int64)
        _lib.check(_lib.load().tcsdn_model_stats(self._handle, _lib.ptr(out, _lib._i64p)))
        return out

    # ---- the hot call -----------------------------------------------------------------------------
    def _run(self, X, want_scores: bool, out=None):
        """-> (indices, scores or None); numpy in -> numpy out, CUDA tensor in -> CUDA tensors out.
        `out`: optional preallocated int32 index buffer (same kind/location as X), e.g. for CUDA graphs."""
        self._check_fitted()
        X, n, d, dt, loc = _rows(X)
        if out is not None:
            if loc == _lib.DEVICE:
                import torch
                if not (_is_torch_cuda(out) and out.dtype == torch.int32 and out.numel() == n and out.is_contiguous()):
                    raise ValueError("out must be a contiguous CUDA int32 tensor with one element per row")
            elif not (isinstance(out, np.ndarray) and out.dtype == np.int32 and out.shape == (n,) and out.flags.c_contiguous):
                raise ValueError("out must be a contiguous int32 array with one element per row")
        lib = _lib.load()
        return _call(X, loc, [((n,), np.int32) if out is None else out, ((n, self._score_cols), np.float64) if want_scores else None],
                     lambda x, o, st: lib.tcsdn_predict(self._handle, x, n, d, dt, loc, o[0], o[1], st))

    def sync_check(self):
        """After CUDA-tensor predicts: wait for the current stream and raise ValueError on NaN/inf input."""
        self._check_fitted()
        import torch
        _lib.check(_lib.load().tcsdn_sync_check(self._handle, torch.cuda.current_stream().cuda_stream))

    def predict_indices(self, X, out=None):
        """int32 index into ``classes_`` per row (cluster id for KMeans)."""
        return self._run(X, False, out)[0]

    def predict(self, X):
        idx, _ = self._run(X, False)
        if _is_torch_cuda(X):
            idx = idx.cpu().numpy()
            self.sync_check()
        return self._labels_from_indices(idx)

    def _labels_from_indices(self, idx):
        """classes_.take(idx) (sk:linear_model/_base.py:423): string class names make this a 4-byte read and a 24-byte write
        per row -- on a million-row batch more host time than the H2D copy and the kernel together -- so large batches of
        fixed-width labels are gathered by the library on a few host threads (tcsdn_take_labels)."""
        n = len(idx)
        cls = self.classes_
        if n < (1 << 16) or cls.dtype.hasobject or cls.dtype.itemsize == 0:
            return cls.take(idx)
        import os
        table = np.ascontiguousarray(cls)
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        out = np.empty(n, dtype=table.dtype)
        _lib.check(_lib.load().tcsdn_take_labels(_lib.ptr(idx), n, _lib.ptr(table), len(table), table.dtype.itemsize, _lib.ptr(out),
                                                 max(1, min(16, (os.cpu_count() or 2) // 2))))
        return out

    def _scores(self, X):
        s = self._run(X, True)[1]
        if _is_torch_cuda(X):
            s = s.cpu().numpy()
            self.sync_check()
        return s

    def score(self, X, y):
        return float(np.mean(self.predict(X) == np.asarray(y)))


def _p(a, t):
    return a.ctypes.data_as(t)


def _rows(X):
    """-> (rows, n, d, dtype code, loc code) for a query: a contiguous float32/float64 CUDA tensor or numpy array (other
    dtypes are widened to float64, what validate_data does with ints / Python floats)."""
    if _is_torch_cuda(X):
        import torch
        if X.dim() != 2:
            raise ValueError(f"Expected 2D array, got {X.dim()}D tensor instead")
        if X.dtype not in (torch.float32, torch.float64):
            X = X.to(torch.float64)
        X = X.contiguous()
        return X, X.shape[0], X.shape[1], _lib.F32 if X.dtype == torch.float32 else _lib.F64, _lib.DEVICE
    A = X if isinstance(X, np.ndarray) else np.asarray(X)
    if A.ndim != 2:
        raise ValueError(f"Expected 2D array, got {A.ndim}D array instead:\narray={A!r}.\nReshape your data "
                         "either using array.reshape(-1, 1) if your data has a single feature or "
                         "array.reshape(1, -1) if it contains a single sample.")
    if A.dtype not in (np.float32, np.float64):
        A = A.astype(np.float64)
    A = np.ascontiguousarray(A)
    return A, A.shape[0], A.shape[1], _lib.F32 if A.dtype == np.float32 else _lib.F64, _lib.HOST


def _call(X, loc, outs, fn):
    """-> the outputs of ``fn(x, out_pointers, stream)`` on the rows X (from _rows).  Each entry of ``outs`` is a
    ``(shape, numpy dtype)`` allocated where X lives, a preallocated buffer, or None (no output, a null pointer).  CUDA rows
    run on the current stream of X's device; host rows pass no stream."""
    if loc == _lib.DEVICE:
        import torch
        outs = [torch.empty(o[0], dtype=getattr(torch, np.dtype(o[1]).name), device=X.device) if isinstance(o, tuple) else o
                for o in outs]
        with torch.cuda.device(X.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(fn(X.data_ptr(), [None if o is None else o.data_ptr() for o in outs], st))
        return tuple(outs)
    outs = [np.empty(*o) if isinstance(o, tuple) else o for o in outs]
    _lib.check(fn(_lib.ptr(X), [None if o is None else _lib.ptr(o) for o in outs], None))
    return tuple(outs)


class LogisticRegression(_Base):
    """sk:linear_model/_base.py:366-427 -- decision_function = X @ coef_.T + intercept_; argmax."""
    _kind = "linear"

    def _sk_estimator(self):
        from sklearn.linear_model import LogisticRegression as SK
        return SK(**self._params)

    def _create(self, lib, spec, h):
        coef = np.ascontiguousarray(spec["coef"], np.float64)
        icpt = np.ascontiguousarray(spec["intercept"], np.float64)
        self.coef_, self.intercept_ = coef, icpt
        _lib.check(lib.tcsdn_linear_create(_p(coef, _lib._f64p), _p(icpt, _lib._f64p), coef.shape[0], coef.shape[1],
                                           C.byref(h)))

    def decision_function(self, X):
        s = self._scores(X)
        return s[:, 0] if s.shape[1] == 1 else s

    def predict_proba(self, X):
        return lr_proba(self._scores(X), bool(self._spec.get("ovr", False)))


def lr_proba(s, ovr):
    """LogisticRegression.predict_proba from the decision values s [n, R] (sk:linear_model/_logistic.py:1595-1625):
    binary -> sigmoid; multinomial -> softmax; one-vs-rest models -> sigmoids normalised over the classes
    (sk:linear_model/_base.py:429-451, rows of all-zero sigmoids become uniform)."""
    with np.errstate(over="ignore"):
        if s.shape[1] == 1:
            p1 = 1.0 / (1.0 + np.exp(-s[:, 0]))
            return np.column_stack([1.0 - p1, p1])
        if ovr:
            p = 1.0 / (1.0 + np.exp(-s))
            tot = p.sum(axis=1)
            zero = tot == 0
            p[zero] = 1.0
            tot[zero] = p.shape[1]
            return p / tot[:, None]
    s = s - s.max(axis=1, keepdims=True)
    e = np.exp(s)
    return e / e.sum(axis=1, keepdims=True)


class GaussianNB(_Base):
    """sk:naive_bayes.py:96-117,533-545 -- joint log likelihood per class; argmax."""
    _kind = "gnb"

    def _sk_estimator(self):
        from sklearn.naive_bayes import GaussianNB as SK
        return SK(**self._params)

    def _create(self, lib, spec, h):
        th = np.ascontiguousarray(spec["theta"], np.float64)
        var = np.ascontiguousarray(spec["var"], np.float64)
        pr = np.ascontiguousarray(spec["class_prior"], np.float64)
        self.theta_, self.var_, self.class_prior_ = th, var, pr
        _lib.check(lib.tcsdn_gnb_create(_p(th, _lib._f64p), _p(var, _lib._f64p), _p(pr, _lib._f64p), th.shape[0],
                                        th.shape[1], C.byref(h)))

    def _fit_gpu(self, X, y, strict):
        """GaussianNB.fit on the GPU (tcsdn_gnb_fit): per-class mean/variance, epsilon_, priors."""
        p = self._params
        if p.get("priors") is not None or y is None:
            if strict:
                raise ValueError("the GPU fit supports priors=None and needs y")
            return False
        if _is_torch_cuda(y):
            y = y.cpu().numpy()
        classes, yi = np.unique(np.asarray(y), return_inverse=True)
        ptr, n, d, dt, loc, keep = self._fit_rows(X)
        if len(yi) != n:
            raise ValueError(f"Found input variables with inconsistent numbers of samples: [{n}, {len(yi)}]")
        if len(classes) > 32 or d > 255:   # the fit kernel's per-block accumulators: classes + 1 <= 33, d + 1 <= 256
            if strict:
                raise ValueError(f"the GPU fit supports at most 32 classes and 255 features (got {len(classes)} and {d})")
            return False
        yi = np.ascontiguousarray(yi, np.int32)
        ydev = None
        if loc == _lib.DEVICE:
            import torch
            ydev = torch.from_numpy(yi).to(keep.device)
            yptr = C.c_void_p(ydev.data_ptr())
        else:
            yptr = _p(yi, C.c_void_p)
        Cn = len(classes)
        th, var = np.empty((Cn, d)), np.empty((Cn, d))
        pr, cnt, eps = np.empty(Cn), np.empty(Cn), C.c_double(0.0)
        f = _lib._f64p
        _lib.check(_lib.load().tcsdn_gnb_fit(ptr, yptr, n, d, Cn, dt, loc, float(p.get("var_smoothing", 1e-9)), _p(th, f),
                                             _p(var, f), _p(pr, f), _p(cnt, f), C.byref(eps), None))
        self._adopt(dict(kind="gnb", theta=th, var=var, class_prior=pr, classes=classes, n_features=d))
        self.class_count_, self.epsilon_ = cnt, float(eps.value)
        return True

    def _joint_log_likelihood(self, X):
        return self._scores(X)

    def predict_log_proba(self, X):  # sk:naive_bayes.py:119-140: jll - logsumexp(jll)
        jll = self._scores(X)
        m = jll.max(axis=1, keepdims=True)
        return jll - (m + np.log(np.exp(jll - m).sum(axis=1, keepdims=True)))

    def predict_proba(self, X):
        return np.exp(self.predict_log_proba(X))


class KMeans(_Base):
    """sk:cluster/_k_means_lloyd.pyx:168-213 -- argmin_j ||c_j||^2 - 2 x.c_j (strict <)."""
    _kind = "kmeans"

    def __init__(self, n_clusters=8, **params):
        super().__init__(n_clusters=n_clusters, **params)

    def _sk_estimator(self):
        from sklearn.cluster import KMeans as SK
        return SK(**self._params)

    def _create(self, lib, spec, h):
        ctr = np.ascontiguousarray(spec["centers"], np.float64)
        self.cluster_centers_ = ctr
        _lib.check(lib.tcsdn_kmeans_create(_p(ctr, _lib._f64p), ctr.shape[0], ctr.shape[1], C.byref(h)))

    def _labels_from_indices(self, idx):
        return idx.astype(np.int32, copy=False)

    def _fit_gpu(self, X, y, strict):
        """Lloyd iterations on the GPU (tcsdn_kmeans_fit) from ONE set of initial centres: an ``init`` array, or
        scikit-learn's k-means++ seeding run on the host with this estimator's ``random_state`` (the same centres
        ``sklearn.cluster.KMeans(n_init=1)`` starts from).  Several restarts (n_init > 1) stay with scikit-learn."""
        p = self._params
        k = int(p.get("n_clusters", 8))
        init = p.get("init", "k-means++")
        n_init = p.get("n_init", "auto")
        ok = (isinstance(init, np.ndarray) or init == "k-means++") and n_init in ("auto", 1) and \
            p.get("algorithm", "lloyd") == "lloyd" and k <= 33
        if not ok:
            if strict:
                raise ValueError("the GPU fit supports init=array or 'k-means++', n_init in ('auto', 1), algorithm='lloyd', "
                                 "n_clusters <= 33")
            return False
        ptr, n, d, dt, loc, keep = self._fit_rows(X)
        if d > 255:
            if strict:
                raise ValueError(f"the GPU fit supports at most 255 features (got {d})")
            return False
        if isinstance(init, np.ndarray):
            c0 = np.ascontiguousarray(init, np.float64)
            if c0.shape != (k, d):
                raise ValueError(f"The shape of the initial centers {c0.shape} does not match the number of clusters {k} "
                                 f"and features {d}.")
        else:
            from sklearn.cluster import kmeans_plusplus
            from sklearn.utils import check_random_state
            host = keep.cpu().numpy() if loc == _lib.DEVICE else keep
            host = np.asarray(host, np.float64)
            mean = host.mean(axis=0)                      # sklearn seeds on the mean-centred rows
            c0, _ = kmeans_plusplus(host - mean, k, random_state=check_random_state(p.get("random_state")))
            c0 = np.ascontiguousarray(c0 + mean, np.float64)
        ctr = np.empty((k, d))
        inertia, n_iter = C.c_double(0.0), C.c_int32(0)
        if loc == _lib.HOST:
            labels = np.empty(n, np.int32)
            lptr = _p(labels, C.c_void_p)
        else:
            import torch
            labels = torch.empty(n, dtype=torch.int32, device=keep.device)
            lptr = C.c_void_p(labels.data_ptr())
        _lib.check(_lib.load().tcsdn_kmeans_fit(ptr, n, d, k, dt, loc, _p(c0, _lib._f64p), int(p.get("max_iter", 300)),
                                                float(p.get("tol", 1e-4)), _p(ctr, _lib._f64p), lptr, C.byref(inertia),
                                                C.byref(n_iter), None))
        self._adopt(dict(kind="kmeans", centers=ctr, classes=np.arange(k, dtype=np.int32), n_features=d))
        self.inertia_, self.n_iter_ = float(inertia.value), int(n_iter.value)
        self.labels_ = labels if loc == _lib.HOST else labels.cpu().numpy()
        return True

    def fit_predict(self, X, y=None):
        return self.fit(X).predict(X)


class KNeighborsClassifier(_Base):
    """sk:neighbors/_classification.py:245-312 -- k nearest (euclidean, manhattan or chebyshev; heap order), uniform or
    distance-weighted vote (``weights='uniform'`` / ``'distance'``; sk:neighbors/_base.py:74-114)."""
    _kind = "knn"

    def __init__(self, n_neighbors=5, **params):
        super().__init__(n_neighbors=n_neighbors, **params)

    def _sk_estimator(self):
        from sklearn.neighbors import KNeighborsClassifier as SK
        return SK(**self._params)

    def _create(self, lib, spec, h):
        fx = np.ascontiguousarray(spec["fit_X"], np.float64)
        y = np.ascontiguousarray(spec["y"], np.int32)
        weights = modelio.knn_weights(spec.get("weights", "uniform"))
        metric = modelio.knn_metric(spec.get("metric", "euclidean"))
        self.n_samples_fit_ = fx.shape[0]
        self.weights = weights
        self.effective_metric_ = metric
        args = (_p(fx, _lib._f64p), _p(y, _lib._i32p), fx.shape[0], fx.shape[1], len(spec["classes"]), int(spec["k"]),
                _lib.KNN_DISTANCE if weights == "distance" else _lib.KNN_UNIFORM)
        # tcsdn_knn_create_weighted is the euclidean tcsdn_knn_create_metric
        _lib.check(lib.tcsdn_knn_create_weighted(*args, C.byref(h)) if metric == "euclidean"
                   else lib.tcsdn_knn_create_metric(*args, _lib.KNN_METRICS[metric], C.byref(h)))

    def set_params(self, **params):
        """sklearn applies ``weights`` at predict time, so on a fitted model a new weighting re-creates the handle from the
        fitted spec (the handle's options, set_option, start from their defaults again).  ``metric``, ``p`` and
        ``metric_params`` are different: sklearn fixes the metric at fit (``effective_metric_``), so on a fitted model they
        only change the parameters, and the fitted metric stays until the next ``fit``."""
        if "weights" in params and self._spec is not None:
            w = modelio.knn_weights(params["weights"])
            if w != modelio.knn_weights(self._spec.get("weights", "uniform")):
                self._adopt(dict(self._spec, weights=w))
        return super().set_params(**params)

    def predict_proba(self, X):
        return self._scores(X)

    def kneighbors(self, X=None, n_neighbors=None, return_distance=True):
        """sk:neighbors/_base.py:750-960 -- the n_neighbors nearest training rows of every row of X: ``(dist, ind)`` (float64,
        int64, [n, n_neighbors]; distances in ``effective_metric_``), or ``ind`` alone.  The neighbours are the ones ``predict`` votes on (sklearn's index-order
        heap); each row is sorted by (distance, training index), where sklearn leaves equal distances in no defined order.
        ``X=None`` queries the training rows and leaves each row's own index out (sklearn's rule).  A CUDA ``torch.Tensor``
        gives CUDA tensors, enqueued on the current stream (``sync_check()`` reports NaN/inf rows).  At most 64 neighbours
        (63 with ``X=None``)."""
        import numbers
        self._check_fitted()
        if n_neighbors is None:
            n_neighbors = int(self._spec["k"])
        elif n_neighbors <= 0:
            raise ValueError("Expected n_neighbors > 0. Got %d" % n_neighbors)
        elif not isinstance(n_neighbors, numbers.Integral):
            raise TypeError("n_neighbors does not take %s value, enter integer value" % type(n_neighbors))
        n_neighbors = int(n_neighbors)
        query_is_train = X is None
        if query_is_train:
            X = np.ascontiguousarray(self._spec["fit_X"], np.float64)
            n_neighbors += 1                         # the row itself comes back too and is removed below
        X, n, d, dt, loc = _rows(X)
        if d != self.n_features_in_:
            raise ValueError(f"X has {d} features, but {type(self).__name__} is expecting {self.n_features_in_} features as input")
        if n_neighbors > self.n_samples_fit_:
            if query_is_train:
                n_neighbors -= 1
                inequality = "n_neighbors < n_samples_fit"
            else:
                inequality = "n_neighbors <= n_samples_fit"
            raise ValueError(f"Expected {inequality}, but n_neighbors = {n_neighbors}, n_samples_fit = {self.n_samples_fit_}, "
                             f"n_samples = {n}")
        if n_neighbors > 64:
            raise ValueError(f"kneighbors keeps at most 64 neighbours per row (with X=None: 63), got n_neighbors = "
                             f"{n_neighbors - 1 if query_is_train else n_neighbors}")
        lib = _lib.load()
        ind, dist = _call(X, loc, [((n, n_neighbors), np.int64), ((n, n_neighbors), np.float64) if return_distance else None],
                          lambda x, o, st: lib.tcsdn_knn_kneighbors(self._handle, x, n, d, dt, loc, n_neighbors, o[0], o[1], st))
        if loc == _lib.DEVICE:
            return (dist, ind) if return_distance else ind
        if query_is_train:
            # sk:neighbors/_base.py:930-956: drop each row's own index; where more duplicates than neighbours push it out
            # of the n_neighbors + 1 kept rows, drop the first column instead
            keep = ind != np.arange(n)[:, None]
            keep[np.all(keep, axis=1), 0] = False
            ind = ind[keep].reshape(n, n_neighbors - 1)
            if return_distance:
                dist = dist[keep].reshape(n, n_neighbors - 1)
        return (dist, ind) if return_distance else ind


class SVC(_Base):
    """sk:svm/src/libsvm/svm.cpp:452-515,2846-2904 -- kernel values (linear, poly, rbf, sigmoid), one-vs-one sums, vote."""
    _kind = "svc"

    def _sk_estimator(self):
        from sklearn.svm import SVC as SK
        return SK(**self._params)

    def _create(self, lib, spec, h):
        sv = np.ascontiguousarray(spec["sv"], np.float64)
        dual = np.ascontiguousarray(spec["dual_coef"], np.float64)
        icpt = np.ascontiguousarray(spec["intercept"], np.float64)
        nsup = np.ascontiguousarray(spec["n_support"], np.int32)
        self.support_vectors_, self.n_support_, self._gamma = sv, nsup, float(spec["gamma"])
        self.decision_function_shape = spec.get("decision_function_shape", "ovr")
        self.break_ties = bool(spec.get("break_ties", False))
        self.kernel = modelio.svc_kernel(spec.get("kernel", "rbf"))
        self.coef0, self.degree = float(spec.get("coef0", 0.0)), int(spec.get("degree", 3))
        self._platt = modelio.svc_platt(spec.get("prob_a"), spec.get("prob_b"), len(nsup))
        if self._platt is not None:   # probability=True: the same handle plus probA_ / probB_ in HBM
            f = _lib._f64p
            _lib.check(lib.tcsdn_svc_create_proba(_p(sv, f), _p(dual, f), _p(icpt, f), _p(nsup, _lib._i32p), sv.shape[0],
                                                  sv.shape[1], len(nsup), _lib.SVC_KERNELS[self.kernel], float(spec["gamma"]),
                                                  self.coef0, self.degree, _p(self._platt[0], f), _p(self._platt[1], f),
                                                  C.byref(h)))
        elif self.kernel == "rbf":
            _lib.check(lib.tcsdn_svc_create(_p(sv, _lib._f64p), _p(dual, _lib._f64p), _p(icpt, _lib._f64p),
                                            _p(nsup, _lib._i32p), sv.shape[0], sv.shape[1], len(nsup),
                                            float(spec["gamma"]), C.byref(h)))
        else:
            _lib.check(lib.tcsdn_svc_create_kernel(_p(sv, _lib._f64p), _p(dual, _lib._f64p), _p(icpt, _lib._f64p),
                                                   _p(nsup, _lib._i32p), sv.shape[0], sv.shape[1], len(nsup),
                                                   _lib.SVC_KERNELS[self.kernel], float(spec["gamma"]), self.coef0,
                                                   self.degree, C.byref(h)))

    @property
    def coef_(self):
        """Primal weights of a linear model, one row per class pair (sk:svm/_base.py:_get_coef, _one_vs_one_coef): from the
        public dual coefficients, which are libsvm's negated for two classes.  Read-only, as in sklearn."""
        self._check_fitted()
        if self.kernel != "linear":
            raise AttributeError("coef_ is only available when using a linear kernel")
        sv, dual = self.support_vectors_, np.asarray(self._spec["dual_coef"], np.float64)
        if dual.shape[0] == 1:
            coef = (-dual) @ sv
        else:
            loc = np.cumsum(np.hstack([[0], self.n_support_]))
            rows = []
            for c1 in range(dual.shape[0] + 1):
                for c2 in range(c1 + 1, dual.shape[0] + 1):
                    rows.append(dual[c2 - 1, loc[c1]:loc[c1 + 1]] @ sv[loc[c1]:loc[c1 + 1]] +
                                dual[c1, loc[c2]:loc[c2 + 1]] @ sv[loc[c2]:loc[c2 + 1]])
            coef = np.vstack(rows)
        coef.flags.writeable = False
        return coef

    def _platt_array(self, i):
        self._check_fitted()
        a = np.zeros(0) if self._platt is None else self._platt[i].copy()
        a.flags.writeable = False
        return a

    @property
    def probA_(self):
        """Platt scaling parameter A per class pair (empty unless fitted with probability=True).  Read-only, as in sklearn."""
        return self._platt_array(0)

    @property
    def probB_(self):
        """Platt scaling parameter B per class pair (empty unless fitted with probability=True).  Read-only, as in sklearn."""
        return self._platt_array(1)

    def _check_proba(self):
        """sk:svm/_base.py _check_proba: predict_proba / predict_log_proba exist only for probability=True (or an imported
        model that carries Platt parameters); hasattr() is False otherwise."""
        if not (self._params.get("probability", False) or getattr(self, "_platt", None) is not None):
            raise AttributeError("predict_proba is not available when probability=False")
        return True

    @property
    def predict_proba(self):
        """sk:svm/_base.py:867-911 -- libsvm's Platt sigmoid per class pair and pairwise coupling, on the GPU
        (tcsdn_svc_predict_proba): [n, n_classes] float64 in ``classes_`` order.  ``predict`` stays libsvm's vote, which can
        differ from the argmax of these probabilities, as in sklearn.  A CUDA ``torch.Tensor`` gives a CUDA tensor,
        enqueued on the current stream (``sync_check()`` reports NaN/inf rows)."""
        self._check_proba()
        return self._predict_proba

    @property
    def predict_log_proba(self):
        """log(predict_proba(X)): ``np.log`` for numpy rows, ``torch.log`` for CUDA tensors."""
        self._check_proba()
        return self._predict_log_proba

    def _predict_proba(self, X):
        self._check_fitted()
        if self._platt is None:
            raise NotFittedError("predict_proba is not available when fitted with probability=False")
        X, n, d, dt, loc = _rows(X)
        lib = _lib.load()
        return _call(X, loc, [((n, len(self.classes_)), np.float64)],
                     lambda x, o, st: lib.tcsdn_svc_predict_proba(self._handle, x, n, d, dt, loc, o[0], st))[0]

    def _predict_log_proba(self, X):
        p = self._predict_proba(X)
        if isinstance(p, np.ndarray):
            return np.log(p)
        import torch
        return torch.log(p)

    def _ovo(self, X):
        return self._scores(X)

    def decision_function(self, X):
        """sk:svm/_base.py:798-828: OvO values (negated for two classes), 'ovr' transform for C > 2."""
        dec = self._ovo(X)
        n_classes = len(self.classes_)
        if n_classes == 2:
            return -dec[:, 0]
        if self.decision_function_shape == "ovr":
            out = np.empty((dec.shape[0], n_classes), np.float64)
            dec = np.ascontiguousarray(dec)
            _lib.check(_lib.load().tcsdn_svc_ovr_from_ovo(_lib.ptr(dec), dec.shape[0], n_classes, _lib.HOST,
                                                          _lib.ptr(out), None))
            return out
        return dec

    def predict(self, X):
        if self.break_ties and self.decision_function_shape == "ovr" and len(self.classes_) > 2:
            return self.classes_.take(np.argmax(self.decision_function(X), axis=1))  # sk:svm/_base.py:851-858
        return super().predict(X)


class RandomForestClassifier(_Base):
    """sk:ensemble/_forest.py:882-967 + sk:tree/_tree.pyx:954-996 -- bit-exact soft vote over the trees."""
    _kind = "forest"

    def _sk_estimator(self):
        from sklearn.ensemble import RandomForestClassifier as SK
        return SK(**self._params)

    def _create(self, lib, spec, h):
        offs = np.ascontiguousarray(spec["tree_offsets"], np.int64)
        left = np.ascontiguousarray(spec["left"], np.int32)
        right = np.ascontiguousarray(spec["right"], np.int32)
        feat = np.ascontiguousarray(spec["feature"], np.int32)
        thr = np.ascontiguousarray(spec["threshold"], np.float64)
        val = np.ascontiguousarray(spec["value"], np.float64)
        self.n_estimators_ = len(offs) - 1
        _lib.check(lib.tcsdn_forest_create(_p(offs, _lib._i64p), _p(left, _lib._i32p), _p(right, _lib._i32p),
                                           _p(feat, _lib._i32p), _p(thr, _lib._f64p), _p(val, _lib._f64p),
                                           len(offs) - 1, int(spec["n_features"]), val.shape[1], C.byref(h)))

    def predict_proba(self, X):
        return self._scores(X)


_BY_KIND = {c._kind: c for c in (LogisticRegression, GaussianNB, KMeans, KNeighborsClassifier, SVC,
                                 RandomForestClassifier)}


def from_spec(spec):
    """Estimator from a parameter spec (traffic_classifier_sdn_b200.modelio)."""
    cls = _BY_KIND[spec["kind"]]
    est = cls.__new__(cls)
    _Base.__init__(est)
    if spec["kind"] == "kmeans":
        est._params["n_clusters"] = int(np.asarray(spec["centers"]).shape[0])
    if spec["kind"] == "knn":
        est._params["n_neighbors"] = int(spec["k"])
        est._params["weights"] = modelio.knn_weights(spec.get("weights", "uniform"))
        est._params["metric"] = modelio.knn_metric(spec.get("metric", "euclidean"))
    if spec["kind"] == "svc" and spec.get("prob_a") is not None and np.asarray(spec["prob_a"]).size:
        est._params["probability"] = True
    return est._adopt(spec)


def from_sklearn(estimator):
    """Import an already fitted scikit-learn estimator."""
    return from_spec(modelio.spec_from_estimator(estimator))


def load_model(path):
    """The reference's ``pickle.load(open('models/<Name>','rb'))`` (traffic_classifier.py:229-244), read as
    data only (works for all six bundled pickles, including the two sklearn >= 1.3 can no longer load)."""
    return from_spec(modelio.load_reference_pickle(path))
