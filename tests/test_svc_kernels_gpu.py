"""GPU: SVC(kernel='linear' | 'poly' | 'sigmoid') on both fp64 kernels (the register kernel: d <= 12, C <= 8; the generic one:
d > 12) against the CPU definition (tests/svc_kernel_oracle.py) and scikit-learn, and the linear collapsed label path
against the fp64 kernel: bit-identical labels, its certificate's bound holding on every pair (engine options 3 / 4), inside
CUDA graphs and the gathered predict."""
import ctypes as C
import functools

import numpy as np
import pytest

import svc_kernel_oracle as so
from traffic_classifier_sdn_b200 import _lib, from_sklearn, from_spec, modelio

pytestmark = pytest.mark.gpu

DEC_REL = 1e-12   # |dec - definition| <= DEC_REL * (sum_s |c_ps K_s| + |rho_p|): fma chains against sequential sums, fp64
NS = (0, 1, 127, 128, 129, 100_000)
MODELS = {"linear": ("linear", {}), "poly": ("poly", dict(degree=3, coef0=-0.5)), "sigmoid": ("sigmoid", dict(coef0=-0.5))}


@functools.lru_cache(maxsize=None)
def _model(kernel, d):
    k, kw = MODELS[kernel]
    sk = so.fit(k, kw, d=d)
    return sk, modelio.spec_from_estimator(sk)


@functools.lru_cache(maxsize=None)
def _rows(d, dtype):
    X, _ = so.flows(max(NS), seed=31, d=d)
    return np.ascontiguousarray(X.astype(dtype))


@functools.lru_cache(maxsize=None)
def _reference(kernel, d, dtype):
    return so.predict(_model(kernel, d)[1], _rows(d, dtype).astype(np.float64))


def _to(x, loc):
    if loc == "host":
        return x
    import torch
    return torch.from_numpy(x).cuda()


def _np(t):
    return t if isinstance(t, np.ndarray) else t.cpu().numpy()


@pytest.mark.parametrize("loc", ["host", "device"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("d", [12, 14], ids=["register", "generic"])
@pytest.mark.parametrize("kernel", list(MODELS))
def test_kernels_against_definition_and_sklearn(kernel, d, dtype, loc):
    sk, spec = _model(kernel, d)
    X = _rows(d, dtype)
    ref_lab, ref_dec, scale = _reference(kernel, d, dtype)
    est = from_sklearn(sk)
    assert est.kernel == kernel
    for n in NS:
        xs = _to(X[:n], loc)
        idx, dec = est._run(xs, True)                      # decision values: the fp64 kernel
        lab = est.predict_indices(xs)                      # labels only: the collapsed path for linear models
        idx, dec, lab = _np(idx), _np(dec), _np(lab)
        assert np.array_equal(idx, ref_lab[:n]), f"n={n}: {int((idx != ref_lab[:n]).sum())} labels differ"
        assert np.array_equal(lab, ref_lab[:n]), f"n={n}: {int((lab != ref_lab[:n]).sum())} label-only labels differ"
        if n:
            err = float(np.max(np.abs(dec - ref_dec[:n]) / scale[:n]))
            assert err <= DEC_REL, f"n={n}: relative decision value error {err:.2e}"
        if loc == "device":
            est.sync_check()
    assert np.array_equal(est.predict(X), sk.predict(X))
    if kernel == "linear":
        assert np.array_equal(est.coef_, sk.coef_)
    else:
        with pytest.raises(AttributeError):
            est.coef_


def _boundary_rows(sk, X, seed):
    """rows moved onto a pair's decision boundary: x - (dec / ||W||^2) W (W = the pair's primal weights)"""
    W = np.asarray(sk.coef_)
    rho = -np.asarray(sk._intercept_)
    if W.shape[0] == 1:
        W = -W                                             # coef_ carries sklearn's binary sign flip
    p = np.random.default_rng(seed).integers(0, W.shape[0], len(X))
    dec = np.einsum("ij,ij->i", X, W[p]) - rho[p]
    return np.ascontiguousarray(X - (dec / np.einsum("ij,ij->i", W[p], W[p]))[:, None] * W[p])


@pytest.mark.parametrize("d", [12, 14])
def test_linear_collapsed_equals_fp64_and_bound_holds(d):
    sk, spec = _model("linear", d)
    X = _rows(d, np.float64)[:50_000]
    B = _boundary_rows(sk, X[:20_000], seed=d)
    ref = from_sklearn(sk).set_option(_lib.OPT_ENGINE, 1)
    for name, rows in (("random", X), ("boundary", B)):
        est = from_sklearn(sk)
        lab = est.predict_indices(rows)
        st = est.stats()
        want = ref.predict_indices(rows)
        assert np.array_equal(lab, want), f"{name}: {int((lab != want).sum())} labels differ from the fp64 kernel"
        assert st[2] == len(rows) and st[1] == 0
        print(f"linear d={d} {name}: {len(rows)} rows, {int(st[6])} re-run by the fp64 kernel")
        if name == "boundary":
            assert st[6] > 0
        else:
            assert st[6] < 0.01 * len(rows)
        _, ddef = ref._run(rows, True)
        _, raw = from_sklearn(sk).set_option(_lib.OPT_ENGINE, 3)._run(rows, True)
        _, bound = from_sklearn(sk).set_option(_lib.OPT_ENGINE, 4)._run(rows, True)
        viol = np.abs(raw - ddef) > bound
        assert not viol.any(), f"{name}: bound violated on {int(viol.sum())} pairs"
        f32 = np.ascontiguousarray(rows.astype(np.float32))
        assert np.array_equal(from_sklearn(sk).predict_indices(f32), ref.predict_indices(f32))


def test_linear_option2_on_unsupported_shape_is_einval():
    sk, _ = _model("linear", 17)                           # d = 17: no collapsed path
    X = _rows(17, np.float64)[:1000]
    est = from_sklearn(sk)
    assert np.array_equal(est.predict_indices(X), from_sklearn(sk).set_option(_lib.OPT_ENGINE, 1).predict_indices(X))
    with pytest.raises(ValueError, match="forced"):
        est.set_option(_lib.OPT_ENGINE, 2).predict_indices(X)
    sk12, _ = _model("linear", 12)
    est12 = from_sklearn(sk12).set_option(_lib.OPT_ENGINE, 2)
    assert np.array_equal(est12.predict_indices(_rows(12, np.float64)[:1000]), _reference("linear", 12, np.float64)[0][:1000])


@pytest.mark.parametrize("kernel", ["poly", "sigmoid"])
def test_poly_sigmoid_reject_fast_path_options(kernel):
    est = from_sklearn(_model(kernel, 12)[0])
    for v in (2, 3, 4):
        with pytest.raises(ValueError):
            est.set_option(_lib.OPT_ENGINE, v)
    est.set_option(_lib.OPT_ENGINE, 1)


def test_linear_10m_rows_strided_sample():
    import torch
    sk, spec = _model("linear", 12)
    n = 10_000_000
    g = torch.Generator(device="cuda").manual_seed(7)
    X = torch.randn((n, 12), generator=g, device="cuda", dtype=torch.float32)
    est = from_sklearn(sk)
    full = est.predict_indices(X)
    est.sync_check()
    st = est.stats()
    s = slice(0, n, 20_011)
    xs = X[s].cpu().numpy()
    assert np.array_equal(full[s].cpu().numpy(), from_sklearn(sk).set_option(_lib.OPT_ENGINE, 1).predict_indices(xs))
    assert np.array_equal(full[s].cpu().numpy(), so.predict(spec, xs.astype(np.float64))[0])
    print(f"linear 10M rows: {int(st[6])} re-run by the fp64 kernel")


def test_linear_graph_replay_and_gathered_world1():
    import torch
    import torch.distributed as dist
    from traffic_classifier_sdn_b200.parallel import Communicator
    sk, _ = _model("linear", 12)
    est = from_sklearn(sk)
    n = 50_003
    X = torch.from_numpy(_rows(12, np.float32)[:n]).cuda()
    ref = est.predict_indices(X).cpu().numpy()
    out = torch.empty(n, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        est.predict_indices(X, out=out)
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), ref)
    torch.cuda.set_device(0)
    if not dist.is_initialized():
        dist.init_process_group("gloo", init_method="tcp://127.0.0.1:29643", rank=0, world_size=1)
    comm = Communicator()
    try:
        for _ in range(2):
            got = comm.predict_gathered(est, X)
            torch.cuda.synchronize()
            assert np.array_equal(got.cpu().numpy()[0, :n], ref.astype(np.uint8))
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            got = comm.predict_gathered(est, X)
        got.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(got.cpu().numpy()[0, :n], ref.astype(np.uint8))
    finally:
        comm.close()


def test_svc_create_and_create_kernel_rbf_identical(golden, specs):
    spec = specs["svc"]
    X = golden["X"]
    a = from_spec(spec)
    b = from_spec(spec)
    sv = np.ascontiguousarray(spec["sv"], np.float64)
    dual = np.ascontiguousarray(spec["dual_coef"], np.float64)
    icpt = np.ascontiguousarray(spec["intercept"], np.float64)
    nsup = np.ascontiguousarray(spec["n_support"], np.int32)
    h = C.c_void_p()
    lib = _lib.load()
    _lib.check(lib.tcsdn_svc_create_kernel(_lib.ptr(sv, _lib._f64p), _lib.ptr(dual, _lib._f64p), _lib.ptr(icpt, _lib._f64p),
                                           _lib.ptr(nsup, _lib._i32p), sv.shape[0], sv.shape[1], len(nsup), _lib.SVC_RBF,
                                           float(spec["gamma"]), 0.0, 3, C.byref(h)))
    b._release()
    b._handle = h
    for est in (a, b):
        est._out = (est._run(X, True), est.predict_indices(X), est.stats())
    (ia, da), la, sa = a._out
    (ib, db), lb, sb = b._out
    assert np.array_equal(ia, ib) and np.array_equal(da, db) and np.array_equal(la, lb) and np.array_equal(sa, sb)
    assert np.array_equal(la, golden["svc.expected_label"])
