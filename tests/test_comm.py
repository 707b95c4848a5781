"""The multi-GPU C ABI (include/tcsdn.h: tcsdn_comm_*): argument checking on CPU, a world-size-1 all-gather and --
when the box has two GPUs -- the two-rank torchrun check on the GPU."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from traffic_classifier_sdn_b200 import _lib
from conftest import spec_from_golden  # noqa: F401  (fixtures `specs` / `golden` come from conftest)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_comm_argument_errors_need_no_gpu():
    lib = _lib.load()
    h = C.c_void_p()
    ident = C.create_string_buffer(_lib.COMM_ID_BYTES)
    assert lib.tcsdn_comm_init(2, 2, ident, C.byref(h)) == _lib.EINVAL      # rank out of range
    assert lib.tcsdn_comm_init(0, 0, ident, C.byref(h)) == _lib.EINVAL      # empty world
    assert lib.tcsdn_comm_init(0, 1, None, C.byref(h)) == _lib.EINVAL       # no id
    assert lib.tcsdn_comm_unique_id(None) == _lib.EINVAL
    assert lib.tcsdn_allgather_labels(None, None, 0, 0, None, None) == _lib.EINVAL
    assert b"allgather_labels" in lib.tcsdn_last_error()
    lib.tcsdn_comm_destroy(None)   # no-op


@pytest.mark.gpu
def test_comm_world1_allgather_pads_short_shard():
    import torch
    lib = _lib.load()
    ident = C.create_string_buffer(_lib.COMM_ID_BYTES)
    _lib.check(lib.tcsdn_comm_unique_id(ident))
    h = C.c_void_p()
    torch.cuda.set_device(0)
    _lib.check(lib.tcsdn_comm_init(0, 1, ident, C.byref(h)))
    try:
        local = torch.arange(1000, dtype=torch.int32, device="cuda")
        out = torch.full((1024,), 7, dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.tcsdn_allgather_labels(h, C.c_void_p(local.data_ptr()), 1000, 1024, C.c_void_p(out.data_ptr()),
                                              C.c_void_p(st)))
        _lib.check(lib.tcsdn_allgather_labels(h, C.c_void_p(local.data_ptr()), 1000, 1000, C.c_void_p(out.data_ptr()),
                                              C.c_void_p(st)))   # full shard: no staging copy
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got[:1000], np.arange(1000)) and np.all(got[1000:] == -1)
    finally:
        lib.tcsdn_comm_destroy(h)


@pytest.mark.gpu
@pytest.mark.parametrize("n_local,n_block,n_classes", [(1000, 1024, 6), (1001, 1001, 6), (997, 1003, 255), (1000, 1024, 300), (0, 8, 3)])
def test_comm_world1_allgather_u8_wire(n_local, n_block, n_classes):
    """tcsdn_allgather_labels_u8: labels cross the wire as bytes (n_classes <= 255; wider models fall back to int32), short
    shards are padded with -1, block lengths that are not multiples of four take the per-rank unpack path; the call is
    capturable into a CUDA graph once its staging buffer exists"""
    import torch
    lib = _lib.load()
    ident = C.create_string_buffer(_lib.COMM_ID_BYTES)
    _lib.check(lib.tcsdn_comm_unique_id(ident))
    h = C.c_void_p()
    torch.cuda.set_device(0)
    _lib.check(lib.tcsdn_comm_init(0, 1, ident, C.byref(h)))
    try:
        g = torch.Generator().manual_seed(n_local + n_block)
        local = torch.randint(0, n_classes, (max(n_local, 1),), generator=g, dtype=torch.int32).cuda()[:n_local]
        out = torch.full((n_block,), 7, dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        args = (h, C.c_void_p(local.data_ptr() if n_local else 0), n_local, n_block, C.c_void_p(out.data_ptr()), n_classes)
        _lib.check(lib.tcsdn_allgather_labels_u8(*args, C.c_void_p(st)))
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got[:n_local], local.cpu().numpy()) and np.all(got[n_local:] == -1)
        # the same call inside a CUDA graph (no allocation, no host synchronisation on the second call)
        out.fill_(9)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            _lib.check(lib.tcsdn_allgather_labels_u8(*args, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        graph.replay()
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got[:n_local], local.cpu().numpy()) and np.all(got[n_local:] == -1)
    finally:
        lib.tcsdn_comm_destroy(h)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["gnb", "linear", "forest", "knn"])
def test_predict_gathered_world1(kind, specs):
    """tcsdn_predict_gathered on one rank: the fused store path of the scorers and the scatter path of the other estimators
    fill slot 0 of the peer-memory buffer with the labels as bytes (255 padding), also inside a CUDA graph replayed twice"""
    import torch
    import torch.distributed as dist
    from traffic_classifier_sdn_b200 import from_spec, synth
    from traffic_classifier_sdn_b200.parallel import Communicator
    torch.cuda.set_device(0)
    if not dist.is_initialized():
        dist.init_process_group("gloo", init_method="tcp://127.0.0.1:29631", rank=0, world_size=1)
    est = from_spec(specs[kind])
    comm = Communicator()
    try:
        for n in (5003, 1000):
            X = torch.from_numpy(synth.make_flows(n, seed=n, return_labels=False).astype(np.float32)).cuda()
            ref = est.predict_indices(X).cpu().numpy()
            for rep in range(3):                           # several generations of both barriers
                got = comm.predict_gathered(est, X)
                torch.cuda.synchronize()
                g = got.cpu().numpy()
                assert g.shape[0] == 1 and g.shape[1] % 16 == 0 and g.shape[1] >= n
                assert np.array_equal(g[0, :n], ref.astype(np.uint8)) and np.all(g[0, n:] == 255)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            got = comm.predict_gathered(est, X)
        for _ in range(2):
            got.zero_()
            graph.replay()
            torch.cuda.synchronize()
            assert np.array_equal(got.cpu().numpy()[0, :n], ref.astype(np.uint8))
    finally:
        comm.close()


@pytest.mark.gpu
def test_two_rank_sharded_predict_and_gather():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29617", os.path.join(ROOT, "tools", "two_gpu_gather.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "gather ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
