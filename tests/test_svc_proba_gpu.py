"""GPU: SVC.predict_proba / predict_log_proba (tcsdn_svc_predict_proba) on both fp64 kernels -- the register kernel (d <= 12,
C <= 8) and the generic one (d = 14, and C = 9 and 16) -- for all four kernel functions, float32 / float64, host / device
rows.  Held to the CPU definition (tests/svc_proba_oracle.py) applied to the same handle's own decision values, to
scikit-learn's predict_proba and to the golden rows (tests/golden/svc_proba.npz)."""
import ctypes as C
import functools

import numpy as np
import pytest

import svc_kernel_oracle as so
import svc_proba_oracle as po
from traffic_classifier_sdn_b200 import _lib, from_sklearn, from_spec

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::FutureWarning")]

NS = (0, 1, 127, 128, 129, 100_000)
DEF_TOL = 1e-13     # against the definition on the handle's own decision values: CUDA's exp against numpy's, nothing else
SK_TOL = 1e-10      # against scikit-learn: largest seen on an H100 1.1e-11 (golden rows, whose decision values differ by 5.7e-12)
MARGIN = 1e-9       # rows whose stopping test came closer than this to eps may stop one round apart
# (kernel, d, C): d = 12 with C <= 8 is the register kernel, the rest the generic one
MODELS = [(k, d, 6) for k in po.KERNEL_KW for d in (12, 14)] + [("rbf", 12, 2), ("rbf", 12, 8), ("rbf", 14, 9),
                                                                 ("rbf", 12, 16), ("poly", 14, 16)]


@functools.lru_cache(maxsize=None)
def _model(kernel, d, n_classes):
    return po.fit(kernel, n_classes, d=d, n=max(600, 80 * n_classes))


@functools.lru_cache(maxsize=None)
def _sk_proba(kernel, d, n_classes, dtype):
    return _model(kernel, d, n_classes).predict_proba(_rows(d, dtype).astype(np.float64))


@functools.lru_cache(maxsize=None)
def _rows(d, dtype):
    X, _ = so.flows(max(NS), seed=31, d=d)
    return np.ascontiguousarray(X.astype(dtype))


def _to(x, loc):
    if loc == "host":
        return x
    import torch
    return torch.from_numpy(x).cuda()


def _np(t):
    return t if isinstance(t, np.ndarray) else t.cpu().numpy()


def _check_definition(est, X, p, what):
    """p against the definition on the handle's own decision values (tcsdn_predict's scores of the same rows)"""
    dec = _np(est._run(X, True)[1])
    ref, rounds, margin = po.proba(dec, est.probA_, est.probB_)
    sure = margin >= MARGIN
    if sure.any():
        err = float(np.abs(p[sure] - ref[sure]).max())
        assert err <= DEF_TOL, f"{what}: |p - definition| = {err:.2e}"
    close = int((~sure).sum())
    if close:
        err = float(np.abs(p[~sure] - ref[~sure]).max())
        assert err <= 0.005 / p.shape[1], f"{what}: {close} rows near a stopping test differ by {err:.2e}"
    print(f"{what}: {len(p)} rows, rounds {rounds.min() if len(p) else 0}-{rounds.max() if len(p) else 0}, "
          f"{close} rows with a stopping margin below {MARGIN:g}")
    return rounds


@pytest.mark.parametrize("loc", ["host", "device"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("kernel,d,n_classes", MODELS, ids=[f"{k}-d{d}-C{c}" for k, d, c in MODELS])
def test_proba_against_definition_and_sklearn(kernel, d, n_classes, dtype, loc):
    sk = _model(kernel, d, n_classes)
    X = _rows(d, dtype)
    est = from_sklearn(sk)
    plain = from_sklearn(sk)
    plain._release()
    lib = _lib.load()
    spec = est._spec
    h = C.c_void_p()
    f = _lib._f64p
    sv, dual, icpt = (np.ascontiguousarray(spec[k], np.float64) for k in ("sv", "dual_coef", "intercept"))
    nsup = np.ascontiguousarray(spec["n_support"], np.int32)
    _lib.check(lib.tcsdn_svc_create_kernel(_lib.ptr(sv, f), _lib.ptr(dual, f), _lib.ptr(icpt, f), _lib.ptr(nsup, _lib._i32p),
                                           sv.shape[0], d, n_classes, _lib.SVC_KERNELS[kernel], float(spec["gamma"]),
                                           float(spec["coef0"]), int(spec["degree"]), C.byref(h)))
    plain._handle = h                                       # the same model without Platt parameters
    ref_sk = _sk_proba(kernel, d, n_classes, dtype)
    for n in NS:
        xs = _to(X[:n], loc)
        p = est.predict_proba(xs)
        st = est.stats()
        lp = est.predict_log_proba(xs)
        if loc == "device":
            import torch
            assert p.is_cuda and lp.is_cuda and p.dtype == torch.float64
            assert torch.equal(lp, torch.log(p))              # torch.log on the device, np.log for host rows
            est.sync_check()
        else:
            assert np.array_equal(lp, np.log(p))
        p = _np(p)
        assert p.shape == (n, n_classes)
        if n:
            assert st[0] >= 1 and st[2] == n, st
        what = f"{kernel} d={d} C={n_classes} {np.dtype(dtype).name} {loc} n={n}"
        _check_definition(est, X[:n], p, what)
        assert np.all(np.abs(p.sum(axis=1) - 1) <= 1e-12)
        err = float(np.abs(p - ref_sk[:n]).max()) if n else 0.0
        assert err <= SK_TOL, f"{what}: |p - sklearn| = {err:.2e}"
        assert np.array_equal(_np(est.predict_indices(xs)), _np(plain.predict_indices(xs)))
    print(f"{kernel} d={d} C={n_classes}: max |p - sklearn| over {max(NS)} rows {err:.2e}")


def test_golden_rows(golden):
    spec, dec, ref, _ = po.load_fixture()
    g = from_spec(spec)
    assert g.get_params()["probability"] is True
    X = golden["X"]
    p = g.predict_proba(X)
    err = float(np.abs(p - ref).max())
    print(f"golden: {len(X)} rows, max |p - sklearn 1.9.0| {err:.2e}, "
          f"max |dec - sklearn| {float(np.abs(g._ovo(X) - dec).max()):.2e}")
    assert err <= SK_TOL
    _check_definition(g, X, p, "golden")
    f32 = np.ascontiguousarray(X.astype(np.float32))
    _check_definition(g, f32, g.predict_proba(f32), "golden float32")


def test_ragged_host_chunks_and_engine_option():
    sk = _model("rbf", 12, 6)
    X = _rows(12, np.float64)[:99_999]
    want = from_sklearn(sk).predict_proba(X)
    est = from_sklearn(sk).set_option(_lib.OPT_CHUNK_ROWS, 1000)
    assert np.array_equal(est.predict_proba(X), want)
    for v in (1, 2):                                        # the fp64 kernels on every option
        assert np.array_equal(from_sklearn(sk).set_option(_lib.OPT_ENGINE, v).predict_proba(X), want)


def test_nonfinite_rows():
    import torch
    sk = _model("rbf", 12, 6)
    X = _rows(12, np.float32)[:1000].copy()
    X[517, 3] = np.nan
    est = from_sklearn(sk)
    with pytest.raises(ValueError, match="NaN"):
        est.predict_proba(X)
    est.predict_proba(torch.from_numpy(X).cuda())
    with pytest.raises(ValueError, match="NaN"):
        est.sync_check()
    est.sync_check()                                        # the flag is cleared by the check


def test_graph_replay_equals_eager():
    import torch
    from traffic_classifier_sdn_b200 import _lib as L
    sk = _model("rbf", 12, 6)
    est = from_sklearn(sk)
    n = 50_003
    X = torch.from_numpy(_rows(12, np.float32)[:n]).cuda()
    ref = est.predict_proba(X).cpu().numpy()
    out = torch.empty((n, 6), dtype=torch.float64, device="cuda")
    lib = L.load()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        L.check(lib.tcsdn_svc_predict_proba(est._handle, X.data_ptr(), n, 12, L.F32, L.DEVICE, out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), ref)
    est.sync_check()


def test_abi_refusals_and_reference_model(specs, golden):
    lib = _lib.load()
    X = np.ascontiguousarray(golden["X"][:10])
    out = np.empty((10, 16))
    ref_svc = from_spec(specs["svc"])                       # the reference's SVC pickle: probability=False
    assert not hasattr(ref_svc, "predict_proba") and ref_svc.probA_.size == 0
    gnb = from_spec(specs["gnb"])
    for est, d, msg in ((gnb, 12, "SVC handle"), (ref_svc, 12, "Platt"), (from_sklearn(_model("rbf", 12, 6)), 11, "features")):
        rc = lib.tcsdn_svc_predict_proba(est._handle, _lib.ptr(X), 10, d, _lib.F64, _lib.HOST, _lib.ptr(out), None)
        assert rc == _lib.EINVAL and msg in _lib.last_error()
    est = from_sklearn(_model("rbf", 12, 6))
    assert lib.tcsdn_svc_predict_proba(est._handle, _lib.ptr(X), 10, 12, 7, _lib.HOST, _lib.ptr(out), None) == _lib.EINVAL
    assert lib.tcsdn_svc_predict_proba(est._handle, _lib.ptr(X), 10, 12, _lib.F64, _lib.HOST, None, None) == _lib.EINVAL
    with pytest.raises(ValueError, match="features"):
        est.predict_proba(X[:, :11])
