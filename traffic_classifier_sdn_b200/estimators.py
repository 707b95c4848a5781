"""sklearn-like estimators whose ``predict`` runs on the H100 through libtcsdn.so.

These classes are the drop-in for the objects the reference gets from ``pickle.load`` at
``traffic_classifier.py:243`` and calls at ``traffic_classifier.py:106``
(``label = model.predict(features.tolist())``).  The duck type kept is scikit-learn's:

* ``fit(X, y=None) -> self``; ``predict(X) -> ndarray[n]`` of ``classes_`` dtype (int32 cluster ids for
  KMeans); ``classes_``, ``n_features_in_``; ``decision_function`` (LogisticRegression, SVC),
  ``predict_proba`` (GaussianNB, KNeighborsClassifier, RandomForestClassifier, SVC(probability=True)), ``predict_log_proba`` /
  ``transform`` where sklearn has them and they are a closed form of the kernel's score matrix;
  ``kneighbors`` (KNeighborsClassifier); ``transform``, ``fit_transform`` and ``score`` (KMeans, their own kernels);
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
           "RandomForestClassifier", "from_spec", "from_sklearn", "load_model", "kmeans_plusplus", "NotFittedError"]


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
        csrc/fit.cu) unless ``backend="sklearn"``; RandomForestClassifier and SVC fit on the GPU with ``backend="gpu"``
        (csrc/forest_fit.cu, csrc/svc_fit.cu) and with scikit-learn on the host otherwise; LogisticRegression and
        KNeighborsClassifier train with scikit-learn."""
        if backend not in ("auto", "gpu", "sklearn"):
            raise ValueError("backend must be 'auto', 'gpu' or 'sklearn'")
        if backend != "sklearn" and self._fit_gpu(X, y, strict=backend == "gpu"):
            return self
        est = self._sk_estimator()
        est.fit(X) if y is None and self._kind == "kmeans" else est.fit(X, y)
        self._adopt(modelio.spec_from_estimator(est))
        for attr in ("n_iter_", "inertia_", "labels_", "feature_names_in_", "feature_importances_"):
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
        """Lloyd iterations on the GPU (tcsdn_kmeans_fit) from ONE set of initial centres: an ``init`` array, or k-means++
        seeding on the GPU (kmeans_plusplus) with scikit-learn's draws from this estimator's ``random_state``.  scikit-learn
        seeds on the mean-centred rows, this seeding on the rows as given: the centres are the same unless a draw falls
        within rounding of a prefix-sum boundary.  Several restarts (n_init > 1) stay with scikit-learn."""
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
        else:   # the rows stay where they are: host rows are uploaded once more by the fit below
            c0 = _seed_plusplus(ptr, n, d, dt, loc, k, p.get("random_state"), None)[0]
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

    def fit_transform(self, X, y=None):
        """``fit(X)`` followed by ``transform(X)``."""
        return self.fit(X).transform(X)

    def transform(self, X):
        """sk:cluster/_kmeans.py ``transform``: the distance of every row to every centre, [n, n_clusters] float64
        (tcsdn_kmeans_transform: scikit-learn's _euclidean_dense_dense in fp64, correctly rounded sqrt).  A CUDA
        ``torch.Tensor`` gives a CUDA tensor, enqueued on the current stream (``sync_check()`` reports NaN/inf rows)."""
        self._check_fitted()
        X, n, d, dt, loc = _rows(X)
        if d != self.n_features_in_:
            raise ValueError(f"X has {d} features, but {type(self).__name__} is expecting {self.n_features_in_} features as input")
        lib = _lib.load()
        return _call(X, loc, [((n, len(self.cluster_centers_)), np.float64)],
                     lambda x, o, st: lib.tcsdn_kmeans_transform(self._handle, x, n, d, dt, loc, o[0], st))[0]

    def score(self, X, y=None, sample_weight=None):
        """sk:cluster/_kmeans.py ``score``: minus the inertia of X against the fitted centres, each row with the centre
        ``predict`` gives it (tcsdn_kmeans_score).  Unit weights only."""
        if sample_weight is not None:
            raise ValueError("KMeans.score supports sample_weight=None only")
        self._check_fitted()
        X, n, d, dt, loc = _rows(X)
        if d != self.n_features_in_:
            raise ValueError(f"X has {d} features, but {type(self).__name__} is expecting {self.n_features_in_} features as input")
        lib = _lib.load()
        inertia = C.c_double(0.0)
        if loc == _lib.DEVICE:
            import torch
            with torch.cuda.device(X.device):
                _lib.check(lib.tcsdn_kmeans_score(self._handle, X.data_ptr(), n, d, dt, loc, C.byref(inertia),
                                                  torch.cuda.current_stream().cuda_stream))
            self.sync_check()
        else:
            _lib.check(lib.tcsdn_kmeans_score(self._handle, _lib.ptr(X), n, d, dt, loc, C.byref(inertia), None))
        return -float(inertia.value)


def _seed_plusplus(ptr, n, d, dt, loc, k, random_state, n_local_trials):
    """tcsdn_kmeans_plusplus on rows from _Base._fit_rows, with scikit-learn's draws: -> (centers [k, d] float64, indices)."""
    from sklearn.utils import check_random_state
    if k > n:
        raise ValueError(f"n_samples={n} should be >= n_clusters={k}.")
    if n_local_trials is None:
        n_local_trials = 2 + int(np.log(k))
    elif int(n_local_trials) < 1:
        raise ValueError(f"n_local_trials must be >= 1, got {n_local_trials}")
    L = int(n_local_trials)
    # sk:cluster/_kmeans.py:_kmeans_plusplus with sample_weight = ones: the draws do not depend on the data, so all of them
    # are made here, in scikit-learn's order
    rs = check_random_state(random_state)
    w = np.ones(n)
    first = int(rs.choice(n, p=w / w.sum()))
    u = np.ascontiguousarray(np.concatenate([rs.uniform(size=L) for _ in range(k - 1)]) if k > 1 else np.zeros(1))
    centers = np.empty((k, d))
    indices = np.empty(k, np.int64)
    st = None
    if loc == _lib.DEVICE:
        import torch
        st = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.load().tcsdn_kmeans_plusplus(ptr, n, d, k, dt, loc, first, L, _p(u, _lib._f64p), _p(indices, _lib._i64p),
                                                 _p(centers, _lib._f64p), st))
    return centers, indices


def kmeans_plusplus(X, n_clusters, *, random_state=None, n_local_trials=None):
    """sklearn.cluster.kmeans_plusplus on the GPU (tcsdn_kmeans_plusplus), unit sample weights: ``(centers, indices)``,
    centers [n_clusters, n_features] in X's dtype, indices int64.  The random numbers are scikit-learn's, drawn in its order
    from ``check_random_state(random_state)``; the distances and sums are fp64 on the GPU.  X may be a CUDA
    ``torch.Tensor`` (its rows are not copied to the host); the results are numpy arrays either way."""
    n_clusters = int(n_clusters)
    if n_clusters < 1:
        raise ValueError(f"n_clusters must be >= 1, got {n_clusters}")
    ptr, n, d, dt, loc, keep = _Base._fit_rows(X)
    if loc == _lib.DEVICE:
        import torch
        with torch.cuda.device(keep.device):
            centers, indices = _seed_plusplus(ptr, n, d, dt, loc, n_clusters, random_state, n_local_trials)
    else:
        centers, indices = _seed_plusplus(ptr, n, d, dt, loc, n_clusters, random_state, n_local_trials)
    return centers.astype(np.float32 if dt == _lib.F32 else np.float64, copy=False), indices


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

    def _fit_gpu(self, X, y, strict):
        """SVC.fit on the GPU (svc_fit), only with ``backend="gpu"``: scikit-learn 1.9.0's fitted model, bit for bit.
        ``backend="auto"`` keeps scikit-learn on the host."""
        if not strict:
            return False
        m = svc_fit(X, y, self._params)
        self._adopt(dict(kind="svc", sv=m["support_vectors_"], dual_coef=m["_dual_coef_"], intercept=m["_intercept_"],
                         n_support=m["n_support_"], gamma=m["_gamma"], classes=m["classes_"], n_features=m["shape_fit_"][1],
                         decision_function_shape=str(self._params.get("decision_function_shape", "ovr")),
                         break_ties=bool(self._params.get("break_ties", False)), n_classes=len(m["classes_"]),
                         kernel=m["kernel"], coef0=m["coef0"], degree=m["degree"]))
        for k in ("support_", "dual_coef_", "intercept_", "_dual_coef_", "_intercept_", "n_iter_", "fit_status_",
                  "class_weight_", "shape_fit_"):
            setattr(self, k, m[k])
        return True


_SVC_GPU_PARAMS = ("C", "kernel", "degree", "gamma", "coef0", "shrinking", "probability", "tol", "cache_size",
                   "class_weight", "verbose", "max_iter", "decision_function_shape", "break_ties", "random_state")
SVC_FIT_MAX_FEATURES = 15


def _real(v):
    import numbers
    return isinstance(v, numbers.Real) and not isinstance(v, bool)


def svc_fit_plan(params, X, y):
    """Host half of SVC.fit (sk:svm/_base.py BaseLibSVM.fit and BaseSVC._validate_targets) for the GPU fit: -> dict with
    ``classes_``, ``y_index`` (int32 class index per row), ``class_weight_``, ``class_C`` (C * class_weight_),
    ``_gamma``, ``kernel``, ``degree``, ``coef0``, ``tol``, ``shrinking`` and ``max_iter``.  X: numpy rows or a CUDA
    tensor (gamma='scale' then takes numpy's X.var() on the device, tcsdn_row_var); y: labels on the host or the device.
    Raises ValueError naming what the GPU fit does not support: probability=True, kernel 'sigmoid' / 'precomputed' /
    callable, 16 or more features, NaN / inf host rows, lengths that differ, a single class."""
    import numbers
    from sklearn.utils.class_weight import compute_class_weight
    p = dict(params)
    for k in p:
        if k not in _SVC_GPU_PARAMS:
            raise ValueError(f"SVC GPU fit: unknown parameter {k}")
    prob = p.get("probability", "deprecated")
    if prob is True:
        raise ValueError("SVC GPU fit: probability=True is not supported (Platt scaling needs libsvm's internal "
                         "cross-validation); fit with backend='sklearn'")
    kernel = p.get("kernel", "rbf")
    if callable(kernel) or not isinstance(kernel, str) or kernel not in ("linear", "poly", "rbf"):
        raise ValueError(f"SVC GPU fit: kernel={kernel!r} is not supported (kernel must be 'linear', 'poly' or 'rbf')")
    Cv = p.get("C", 1.0)
    if not _real(Cv) or not 0.0 < Cv < np.inf:
        raise ValueError(f"C must be a float > 0, got {Cv!r}")
    degree = p.get("degree", 3)
    if not isinstance(degree, numbers.Integral) or isinstance(degree, bool) or not 0 <= degree < 2 ** 31:
        raise ValueError(f"degree must be an integer >= 0, got {degree!r}")
    coef0 = p.get("coef0", 0.0)
    if not _real(coef0) or not np.isfinite(coef0):
        raise ValueError(f"coef0 must be a finite float, got {coef0!r}")
    tol = p.get("tol", 1e-3)
    if not _real(tol) or not 0.0 < tol < np.inf:
        raise ValueError(f"tol must be a float > 0, got {tol!r}")
    max_iter = p.get("max_iter", -1)
    if not isinstance(max_iter, numbers.Integral) or isinstance(max_iter, bool) or max_iter < -1:
        raise ValueError(f"max_iter must be an integer >= -1, got {max_iter!r}")
    shrinking = p.get("shrinking", True)
    if not isinstance(shrinking, (bool, np.bool_)):
        raise ValueError(f"shrinking must be a bool, got {shrinking!r}")
    gamma = p.get("gamma", "scale")
    if not (gamma in ("scale", "auto") if isinstance(gamma, str) else _real(gamma) and 0.0 <= gamma < np.inf):
        raise ValueError(f"gamma must be 'scale', 'auto' or a float >= 0, got {gamma!r}")
    ptr, n, d, dt, loc, keep = _Base._fit_rows(X)
    if d > SVC_FIT_MAX_FEATURES:
        raise ValueError(f"SVC GPU fit: X has {d} features; the GPU fit supports at most {SVC_FIT_MAX_FEATURES} "
                         "(n_features_in_ <= 15, where libsvm's BLAS dot is an FMA chain in feature order)")
    if loc == _lib.HOST and not np.isfinite(keep).all():
        raise ValueError("Input X contains NaN or infinity.")
    if y is None:
        raise ValueError("SVC.fit needs y")
    if _is_torch_cuda(y):
        y = y.cpu().numpy()
    y = np.asarray(y)
    if y.ndim != 1:
        y = y.ravel() if y.ndim == 2 and y.shape[1] == 1 else y
    if y.ndim != 1:
        raise ValueError(f"y should be a 1d array, got an array of shape {y.shape} instead.")
    if len(y) != n:
        raise ValueError(f"Found input variables with inconsistent numbers of samples: [{n}, {len(y)}]")
    if n >= 2 ** 31:
        raise ValueError(f"the GPU fit supports fewer than 2^31 rows (got {n})")
    classes, yi = np.unique(y, return_inverse=True)
    class_weight = compute_class_weight(p.get("class_weight"), classes=classes, y=y)
    if len(classes) < 2:
        raise ValueError("The number of classes has to be greater than one; got %d class" % len(classes))
    if isinstance(gamma, str) and gamma == "scale":
        if loc == _lib.HOST:
            var = np.asarray(keep, dtype=np.float64).var()
        else:
            v = C.c_double()
            import torch
            _lib.check(_lib.load().tcsdn_row_var(ptr, n, d, dt, loc, C.byref(v), torch.cuda.current_stream(keep.device).cuda_stream))
            var = np.float64(v.value)
        g = 1.0 / (d * var) if var != 0 else 1.0
    elif isinstance(gamma, str):
        g = 1.0 / d
    else:
        g = gamma
    class_C = np.ascontiguousarray(np.asarray(class_weight, np.float64) * float(Cv))   # libsvm: weighted_C = C * weight
    if not (np.isfinite(class_C).all() and (class_C > 0).all()):
        raise ValueError(f"class_weight: every class needs a weight > 0 for the GPU fit, got {class_weight!r}")
    return dict(classes_=classes, y_index=np.ascontiguousarray(yi.ravel(), np.int32), class_weight_=class_weight,
                class_C=class_C, _gamma=g, kernel=kernel, degree=int(degree), coef0=float(coef0), tol=float(tol),
                shrinking=bool(shrinking), max_iter=int(max_iter), rows=(ptr, n, d, dt, loc, keep))


def svc_fit(X, y, params):
    """SVC(**params).fit(X, y) on the GPU (tcsdn_svc_fit): -> dict of scikit-learn's fitted attributes (``support_``,
    ``support_vectors_``, ``n_support_``, ``dual_coef_``, ``intercept_``, ``_dual_coef_``, ``_intercept_``, ``n_iter_``,
    ``fit_status_``, ``class_weight_``, ``_gamma``, ``classes_``, ``shape_fit_``) plus ``kernel``, ``coef0`` and
    ``degree``.  Raises scikit-learn's ConvergenceWarning when max_iter stopped a class pair."""
    import warnings
    plan = svc_fit_plan(params, X, y)
    ptr, n, d, dt, loc, keep = plan.pop("rows")
    classes = plan["classes_"]
    Cn, lib = len(classes), _lib.load()
    P = Cn * (Cn - 1) // 2
    st = None
    if loc == _lib.DEVICE:
        import torch
        st = torch.cuda.current_stream(keep.device).cuda_stream
    h = C.c_void_p()
    _lib.check(lib.tcsdn_svc_fit(ptr, _p(plan["y_index"], _lib._i32p), n, d, Cn, dt, loc, _lib.SVC_KERNELS[plan["kernel"]],
                                 float(plan["_gamma"]), plan["coef0"], plan["degree"], _p(plan["class_C"], _lib._f64p),
                                 plan["tol"], int(plan["shrinking"]), plan["max_iter"], C.byref(h), st))
    try:
        n_sv, status = C.c_int64(), C.c_int32()
        nsup, n_iter = np.empty(Cn, np.int32), np.empty(P, np.intc)
        _lib.check(lib.tcsdn_svc_fit_sizes(h, C.byref(n_sv), _p(nsup, _lib._i32p), _p(n_iter, _lib._i32p), C.byref(status)))
        m = int(n_sv.value)
        support, sv = np.empty(m, np.int32), np.empty((m, d), np.float64)
        dual, icpt = np.empty((Cn - 1, m), np.float64), np.empty(P, np.float64)
        _lib.check(lib.tcsdn_svc_fit_read(h, _p(support, _lib._i32p), _p(sv, _lib._f64p), _p(dual, _lib._f64p),
                                          _p(icpt, _lib._f64p)))
    finally:
        lib.tcsdn_svc_fit_free(h)
    out = dict(support_=support, support_vectors_=sv, n_support_=nsup, _dual_coef_=dual, _intercept_=icpt,
               dual_coef_=-dual if Cn == 2 else dual, intercept_=-icpt if Cn == 2 else icpt.copy(), n_iter_=n_iter,
               fit_status_=int(status.value), class_weight_=plan["class_weight_"], _gamma=plan["_gamma"], classes_=classes,
               shape_fit_=(n, d), kernel=plan["kernel"], coef0=plan["coef0"], degree=plan["degree"])
    if out["fit_status_"] == 1:   # sk:svm/_base.py _warn_from_fit_status
        from sklearn.exceptions import ConvergenceWarning
        warnings.warn("Solver terminated early (max_iter=%i).  Consider pre-processing your data with StandardScaler "
                      "or MinMaxScaler." % plan["max_iter"], ConvergenceWarning)
    return out


_FOREST_GPU_PARAMS = ("n_estimators", "criterion", "max_depth", "min_samples_split", "min_samples_leaf", "max_features",
                      "bootstrap", "max_samples", "min_impurity_decrease", "random_state", "n_jobs", "verbose",
                      "min_weight_fraction_leaf", "max_leaf_nodes", "class_weight", "monotonic_cst", "oob_score",
                      "warm_start", "ccp_alpha")
# parameters the GPU fit refuses unless they hold scikit-learn's default
_FOREST_GPU_DEFAULTS = {"criterion": "gini", "min_weight_fraction_leaf": 0.0, "max_leaf_nodes": None, "class_weight": None,
                        "monotonic_cst": None, "oob_score": False, "warm_start": False, "ccp_alpha": 0.0}


def forest_fit_plan(params, n, d):
    """Host half of RandomForestClassifier.fit (sk:ensemble/_forest.py fit, sk:tree/_classes.py BaseDecisionTree._fit) for
    the GPU fit: the resolved tree parameters and every random number, drawn in scikit-learn's order.  -> dict with
    ``n_trees``, ``max_depth``, ``min_samples_split``, ``min_samples_leaf``, ``max_features``, ``min_impurity_decrease``,
    ``n_boot`` (0 without bootstrap), ``bootstrap_idx`` ([n_trees][n_boot] int32 or None) and ``rand_r_seeds``
    ([n_trees] uint32, each tree splitter's ``rand_r_state``).  Raises ValueError naming a parameter it does not support."""
    import numbers
    from math import ceil
    from sklearn.utils import check_random_state
    p = dict(params)
    for k in p:
        if k not in _FOREST_GPU_PARAMS:
            raise ValueError(f"RandomForestClassifier GPU fit: unknown parameter {k}")
    for k, default in _FOREST_GPU_DEFAULTS.items():
        v = p.get(k, default)
        same = v is None if default is None else (type(v) is type(default) or isinstance(v, numbers.Real) and
                                                  not isinstance(v, bool) and isinstance(default, float)) and v == default
        if not same:
            raise ValueError(f"RandomForestClassifier GPU fit: {k}={v!r} is not supported (only {k}={default!r})")
    T = p.get("n_estimators", 100)
    if not isinstance(T, numbers.Integral) or T < 1:
        raise ValueError(f"n_estimators must be an integer >= 1, got {T!r}")
    md = p.get("max_depth")
    if md is not None and (not isinstance(md, numbers.Integral) or md < 1):
        raise ValueError(f"max_depth must be None or an integer >= 1, got {md!r}")
    max_depth = np.iinfo(np.int32).max if md is None else int(md)
    msl, mss = p.get("min_samples_leaf", 1), p.get("min_samples_split", 2)
    if isinstance(msl, numbers.Integral) and not isinstance(msl, bool) and msl >= 1:
        msl = int(msl)
    elif isinstance(msl, numbers.Real) and not isinstance(msl, numbers.Integral) and 0.0 < msl < 1.0:
        msl = ceil(msl * n)
    else:
        raise ValueError(f"min_samples_leaf must be an integer >= 1 or a float in (0, 1), got {msl!r}")
    if isinstance(mss, numbers.Integral) and not isinstance(mss, bool) and mss >= 2:
        mss = int(mss)
    elif isinstance(mss, numbers.Real) and not isinstance(mss, numbers.Integral) and 0.0 < mss <= 1.0:
        mss = max(2, ceil(mss * n))
    else:
        raise ValueError(f"min_samples_split must be an integer >= 2 or a float in (0, 1], got {mss!r}")
    mss = max(mss, 2 * msl)
    mf = p.get("max_features", "sqrt")
    if isinstance(mf, str) and mf in ("sqrt", "log2"):
        mf = max(1, int(np.sqrt(d) if mf == "sqrt" else np.log2(d)))
    elif mf is None:
        mf = d
    elif isinstance(mf, numbers.Integral) and not isinstance(mf, bool) and 1 <= mf <= d:
        mf = int(mf)
    elif isinstance(mf, numbers.Real) and not isinstance(mf, numbers.Integral) and 0.0 < mf <= 1.0:
        mf = max(1, int(mf * d))
    else:
        raise ValueError(f"max_features must be 'sqrt', 'log2', None, an integer in [1, {d}] or a float in (0, 1], "
                         f"got {mf!r}")
    mid = p.get("min_impurity_decrease", 0.0)
    if not isinstance(mid, numbers.Real) or isinstance(mid, bool) or not mid >= 0.0:
        raise ValueError(f"min_impurity_decrease must be a float >= 0, got {mid!r}")
    bootstrap, ms = p.get("bootstrap", True), p.get("max_samples")
    if not bootstrap and ms is not None:
        raise ValueError("max_samples cannot be set if bootstrap=False")
    n_boot = 0
    if bootstrap:   # sk:ensemble/_bootstrap.py _get_n_samples_bootstrap
        if ms is None:
            n_boot = n
        elif isinstance(ms, numbers.Integral) and not isinstance(ms, bool) and ms >= 1:
            n_boot = int(ms)
        elif isinstance(ms, numbers.Real) and not isinstance(ms, numbers.Integral) and 0.0 < ms <= 1.0:
            n_boot = max(int(ms * n), 1)
        else:
            raise ValueError(f"max_samples must be None, an integer >= 1 or a float in (0, 1], got {ms!r}")
    # sk:ensemble/_base.py _set_random_states: one seed per tree, in estimator order; then per tree a FRESH
    # RandomState(seed) draws the bootstrap indices (_generate_sample_indices) and another the splitter's rand_r_state
    # (sk:tree/_splitter.pyx Splitter.init)
    rs = check_random_state(p.get("random_state"))
    seeds = [rs.randint(np.iinfo(np.int32).max) for _ in range(T)]
    idx = np.empty((T, n_boot), np.int32) if bootstrap else None
    rr = np.empty(T, np.uint32)
    for t, s in enumerate(seeds):
        if bootstrap:
            idx[t] = np.random.RandomState(s).randint(0, n, n_boot)
        rr[t] = np.random.RandomState(s).randint(0, 2147483647)
    return dict(n_trees=int(T), max_depth=int(max_depth), min_samples_split=int(mss), min_samples_leaf=int(msl),
                max_features=int(mf), min_impurity_decrease=float(mid), n_boot=int(n_boot), bootstrap_idx=idx,
                rand_r_seeds=rr)


def forest_fit(X, y, params, node_capacity=0):
    """RandomForestClassifier(**params).fit(X, y) on the GPU (tcsdn_forest_fit, criterion='gini', no sample or class
    weights): -> (classes_, dict of the concatenated per-tree node arrays with ``tree_offsets`` and ``n_features``).  X:
    numpy rows or a CUDA tensor (its rows are not copied to the host); y on the host or the device.  ``node_capacity``:
    nodes per tree of the first attempt (0: the library's default)."""
    if y is None:
        raise ValueError("RandomForestClassifier.fit needs y")
    ptr, n, d, dt, loc, keep = _Base._fit_rows(X)
    if _is_torch_cuda(y):
        y = y.cpu().numpy()
    y = np.asarray(y)
    if y.ndim != 1:
        raise ValueError("the GPU fit supports a 1-D y (one output)")
    if len(y) != n:
        raise ValueError(f"Found input variables with inconsistent numbers of samples: [{n}, {len(y)}]")
    classes, yi = np.unique(y, return_inverse=True)
    if len(classes) > 32 or d > 255 or n >= 2 ** 31:
        raise ValueError(f"the GPU fit supports at most 32 classes, 255 features and 2^31 - 1 rows "
                         f"(got {len(classes)}, {d} and {n})")
    plan = forest_fit_plan(params, n, d)
    yi = np.ascontiguousarray(yi, np.int32)
    ydev = None
    if loc == _lib.DEVICE:
        import torch
        ydev = torch.from_numpy(yi).to(keep.device)
        yptr = C.c_void_p(ydev.data_ptr())
    else:
        yptr = _p(yi, C.c_void_p)
    boot = plan["bootstrap_idx"]
    if boot is not None and plan["n_boot"] >= 2 ** 31:
        raise ValueError(f"max_samples: the GPU fit draws fewer than 2^31 rows per tree (got {plan['n_boot']})")
    T, Cn, lib = plan["n_trees"], len(classes), _lib.load()
    h = C.c_void_p()
    st = None
    if loc == _lib.DEVICE:
        import torch
        st = torch.cuda.current_stream(keep.device).cuda_stream
    _lib.check(lib.tcsdn_forest_fit(ptr, yptr, n, d, Cn, dt, loc, T, None if boot is None else _p(boot, C.c_void_p),
                                    plan["n_boot"], _p(plan["rand_r_seeds"], C.c_void_p), plan["max_features"],
                                    plan["max_depth"], plan["min_samples_split"], plan["min_samples_leaf"],
                                    plan["min_impurity_decrease"], int(node_capacity), C.byref(h), st))
    try:
        offs = np.empty(T + 1, np.int64)
        _lib.check(lib.tcsdn_forest_fit_nodes(h, _p(offs, _lib._i64p)))
        N = int(offs[-1])
        a = dict(left=np.empty(N, np.int32), right=np.empty(N, np.int32), feature=np.empty(N, np.int32),
                 threshold=np.empty(N), value=np.empty((N, Cn)), impurity=np.empty(N),
                 n_node_samples=np.empty(N, np.int64), weighted_n_node_samples=np.empty(N))
        _lib.check(lib.tcsdn_forest_fit_read(h, _p(a["left"], _lib._i32p), _p(a["right"], _lib._i32p),
                                             _p(a["feature"], _lib._i32p), _p(a["threshold"], _lib._f64p),
                                             _p(a["value"], _lib._f64p), _p(a["impurity"], _lib._f64p),
                                             _p(a["n_node_samples"], _lib._i64p),
                                             _p(a["weighted_n_node_samples"], _lib._f64p)))
    finally:
        lib.tcsdn_forest_fit_free(h)
    return classes, dict(a, tree_offsets=offs, n_features=d)


def forest_feature_importances(offsets, left, right, feature, impurity, weighted_n_node_samples, d):
    """RandomForestClassifier.feature_importances_ from the concatenated tree arrays, in scikit-learn's operation order:
    per tree sk:tree/_tree.pyx Tree.compute_feature_importances (a node-order sum of each split's weighted impurity
    decrease, then / root weight, then / sum), then the mean over the trees with more than one node
    (sk:ensemble/_forest.py feature_importances_), divided by its sum."""
    per_tree = []
    for t in range(len(offsets) - 1):
        a, b = int(offsets[t]), int(offsets[t + 1])
        if b - a <= 1:
            continue
        lf, rt, ft = (np.asarray(v[a:b]) for v in (left, right, feature))
        wn = np.asarray(weighted_n_node_samples[a:b], np.float64)
        im = np.asarray(impurity[a:b], np.float64)
        inner = np.flatnonzero(lf != -1)
        l, r = lf[inner], rt[inner]
        imp = np.zeros(d, np.float64)
        np.add.at(imp, ft[inner], wn[inner] * im[inner] - wn[l] * im[l] - wn[r] * im[r])   # unbuffered: node order
        imp /= wn[0]
        s = np.sum(imp)
        if s > 0.0:
            imp /= s
        per_tree.append(imp)
    if not per_tree:
        return np.zeros(d, np.float64)
    m = np.mean(per_tree, axis=0, dtype=np.float64)
    return m / np.sum(m)


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

    def _fit_gpu(self, X, y, strict, node_capacity=0):
        """RandomForestClassifier.fit on the GPU (forest_fit), only with ``backend="gpu"``: the trees scikit-learn 1.9 grows
        with the same ``random_state``, node for node and bit for bit.  ``backend="auto"`` keeps scikit-learn on the host."""
        if not strict:
            return False
        classes, a = forest_fit(X, y, self._params, node_capacity)
        offs, d = a["tree_offsets"], a["n_features"]
        self._adopt(dict(kind="forest", tree_offsets=offs, left=a["left"], right=a["right"], feature=a["feature"],
                         threshold=a["threshold"], value=a["value"], classes=classes, n_features=d))
        self.tree_arrays_ = {k: v for k, v in a.items() if k != "n_features"}
        self.n_classes_ = len(classes)
        self.feature_importances_ = forest_feature_importances(offs, a["left"], a["right"], a["feature"], a["impurity"],
                                                               a["weighted_n_node_samples"], d)
        return True

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
