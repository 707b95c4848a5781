"""GPU: the host-pointer pipeline that tcsdn_predict and tcsdn_knn_kneighbors share (csrc/abi.cu).

Host rows go through the device in chunks on two streams.  Results land directly in the caller's arrays when those are
page-locked; predict fills pageable arrays through pinned staging buffers, kneighbors copies to them directly.  Every host
call here, at several chunk sizes with a ragged last chunk, must equal one device-pointer call bit for bit.
"""
import numpy as np
import pytest

from conftest import KINDS
from traffic_classifier_sdn_b200 import _lib, from_spec, synth

pytestmark = pytest.mark.gpu

N = 12_345            # rows per call: every chunk size below leaves a ragged last chunk
CHUNKS = (1000, 4096)


@pytest.fixture(scope="module")
def rows():
    X = synth.make_flows(N, seed=91, return_labels=False)
    X[:200] = X[5000:5200]   # exact duplicates: distance ties for KNN
    return X


def _model(spec, chunk):
    est = from_spec(spec)
    if spec["kind"] in ("knn", "svc"):
        est.set_option(_lib.OPT_ENGINE, 2)   # the engine on every chunk, as on the single device call
    est.set_option(_lib.OPT_CHUNK_ROWS, chunk)
    return est


def _buffer(shape, dtype, memory):
    """a C-contiguous numpy array: pageable, or a view of a page-locked torch buffer (kept alive by the view's base)"""
    if memory == "pageable":
        return np.full(shape, -7, dtype)
    import torch
    return torch.full(shape, -7, dtype=getattr(torch, np.dtype(dtype).name)).pin_memory().numpy()


def _ptr(a):
    return None if a is None else _lib.ptr(a)


def _host_predict(est, X, labels, scores):
    _lib.check(_lib.load().tcsdn_predict(est._handle, _lib.ptr(X), len(X), X.shape[1], _lib.F64, _lib.HOST, _lib.ptr(labels),
                                         _ptr(scores), None))


def _host_kneighbors(est, X, m, ind, dist):
    _lib.check(_lib.load().tcsdn_knn_kneighbors(est._handle, _lib.ptr(X), len(X), X.shape[1], _lib.F64, _lib.HOST, m,
                                                _lib.ptr(ind), _ptr(dist), None))


@pytest.mark.parametrize("memory", ["pageable", "pinned", "mixed"])
@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("kind", KINDS)
def test_host_predict_equals_one_device_call(specs, rows, kind, chunk, memory):
    """labels only and labels with scores; "mixed" has page-locked labels and pageable scores, so it stages both"""
    import torch
    one = _model(specs[kind], 0)
    ref_labels, ref_scores = (t.cpu().numpy() for t in one._run(torch.from_numpy(rows).cuda(), True))
    one.sync_check()
    est = _model(specs[kind], chunk)
    labels = _buffer((N,), np.int32, "pageable" if memory == "pageable" else "pinned")
    assert est.predict_indices(rows, out=labels) is labels
    assert np.array_equal(labels, ref_labels)
    labels = _buffer((N,), np.int32, "pageable" if memory == "pageable" else "pinned")
    scores = _buffer((N, ref_scores.shape[1]), np.float64, "pinned" if memory == "pinned" else "pageable")
    _host_predict(est, rows, labels, scores)
    assert np.array_equal(labels, ref_labels) and np.array_equal(scores, ref_scores)


@pytest.mark.parametrize("memory", ["pageable", "pinned"])
@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("m", [5, 40])
def test_host_kneighbors_equals_one_device_call(specs, rows, m, chunk, memory):
    """with and without distances; m = 40 is beyond the engine's 32 neighbours and takes the fp64 kernel"""
    import torch
    spec = specs["knn"]
    one = from_spec(spec)
    ref_dist, ref_ind = (t.cpu().numpy() for t in one.kneighbors(torch.from_numpy(rows).cuda(), m))
    one.sync_check()
    est = from_spec(spec)
    est.set_option(_lib.OPT_CHUNK_ROWS, chunk)
    if memory == "pageable":
        dist, ind = est.kneighbors(rows, m)
        assert np.array_equal(est.kneighbors(rows, m, return_distance=False), ref_ind)
    else:
        ind, dist = _buffer((N, m), np.int64, memory), _buffer((N, m), np.float64, memory)
        _host_kneighbors(est, rows, m, ind, dist)
        ind_only = _buffer((N, m), np.int64, memory)
        _host_kneighbors(est, rows, m, ind_only, None)
        assert np.array_equal(ind_only, ref_ind)
    assert np.array_equal(ind, ref_ind) and np.array_equal(dist, ref_dist)


def test_host_kneighbors_nan_in_second_chunk(specs, rows):
    """a NaN row in the second chunk is reported as ValueError once every chunk has run, and the handle keeps working"""
    est = from_spec(specs["knn"])
    est.set_option(_lib.OPT_CHUNK_ROWS, 1000)
    ref_dist, ref_ind = est.kneighbors(rows, 5)
    bad = rows.copy()
    bad[1500, 3] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        est.kneighbors(bad, 5)
    dist, ind = est.kneighbors(rows, 5)
    assert np.array_equal(ind, ref_ind) and np.array_equal(dist, ref_dist)
