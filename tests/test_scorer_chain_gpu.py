"""GPU: streaming-scorer launches chained on one stream, eagerly and replayed from a CUDA graph.

Back-to-back predicts on one stream are what a serving loop (and bench.py) runs, and the place where any overlap of one scorer
launch with the kernel before it -- programmatic dependent launch, early prefetch of the rows -- would go wrong first.  These
tests put the preceding kernel in every role it can play:
  1. the producer of the rows (a torch kernel writes X, then the scorer reads it: read after write);
  2. the previous predict into the same label buffer (write after write);
  3. a scorer of another model (GaussianNB -> LR -> KMeans -> GaussianNB: different kernels, each the primary of the next);
  4. the previous predict's sticky non-finite flag and GaussianNB's refined-row counter;
  5. the host-pointer pipeline, whose chunks alternate between two internal streams.
Every chained result must equal the same predict run alone and synchronised.  Models: the bench GaussianNB (d = 8; float32
rows take the certified fp32 pre-pass, float64 rows the fp64 path) and the bench LR and KMeans (d = 12); every CTA shape.
"""
import ctypes as C

import numpy as np
import pytest

from traffic_classifier_sdn_b200 import _lib, from_spec

pytestmark = pytest.mark.gpu

SHAPES = (1, 2, 3)                             # OPT_SCORER_SHAPE: 128 x 4, 256 x 2, 128 x 2 (csrc/scorers.cu)
MODES = ("eager", "graph")
MODELS = ("gnb_f32", "gnb_f64", "logistic", "kmeans")
STEPS = 6


def _sm_count():
    n = C.c_int32(0)
    _lib.check(_lib.load().tcsdn_device_sm_count(C.byref(n)))
    return int(n.value)


def _rows_per_batch():
    """every CTA of every shape runs more than one 256- or 512-row tile (at most four CTAs per SM), and the last tile is
    ragged"""
    return 2 * _sm_count() * 4 * 512 + 333


@pytest.fixture(scope="module")
def workloads():
    import bench
    return {name: bench.build_workload(name) for name in ("gnb", "logistic", "kmeans")}


def _model(workloads, model, shape):
    """-> (estimator with the CTA shape forced, n_features, torch dtype of its rows)"""
    import torch
    w = workloads["gnb" if model.startswith("gnb") else model]
    est = from_spec(w["spec"])
    est.set_option(_lib.OPT_SCORER_SHAPE, shape)
    return est, w["d"], torch.float64 if model == "gnb_f64" else torch.float32


def _batches(d, dtype, k, seed):
    """k row permutations of one batch of flow rows: a kernel that read the previous step's rows would get other labels"""
    import torch
    import bench
    base = bench.synth_rows(_rows_per_batch(), d, seed=seed, device=torch.device("cuda", 0)).to(dtype)
    g = torch.Generator().manual_seed(seed)
    return [base if i == 0 else base[torch.randperm(len(base), generator=g).cuda()].contiguous() for i in range(k)]


def _alone(est, batches):
    """each batch predicted by itself, synchronised before the next"""
    import torch
    out = []
    for b in batches:
        out.append(est.predict_indices(b))
        torch.cuda.synchronize()
    est.sync_check()
    return out


def _chained(enqueue, mode):
    """enqueue() puts a chain of steps on the current stream: run it eagerly on the default stream, or capture it into a CUDA
    graph on a side stream and replay the graph once"""
    import torch
    if mode == "eager":
        enqueue()
    else:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            enqueue()
        graph.replay()
    torch.cuda.synchronize()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("model", MODELS)
def test_scorer_reads_the_rows_the_previous_kernel_wrote(workloads, model, shape, mode):
    """each step: a torch kernel writes X from batch i, then a predict reads X into its own label buffer"""
    import torch
    est, d, dtype = _model(workloads, model, shape)
    batches = _batches(d, dtype, STEPS, seed=100 + shape)
    ref = _alone(est, batches)
    assert not torch.equal(ref[0], ref[1]), "the permuted batches must have different labels"
    X = torch.zeros_like(batches[0])
    labels = [torch.full_like(r, -1) for r in ref]

    def enqueue():
        for b, lab in zip(batches, labels):
            torch.mul(b, 1.0, out=X)
            est.predict_indices(X, out=lab)

    _chained(enqueue, mode)
    est.sync_check()
    for i, (lab, r) in enumerate(zip(labels, ref)):
        assert torch.equal(lab, r), f"step {i}: {int((lab != r).sum())} labels differ"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("model", MODELS)
def test_back_to_back_predicts_into_one_buffer(workloads, model, shape, mode):
    """STEPS predicts of different batches into one label buffer: it ends holding the last batch's labels"""
    import torch
    est, d, dtype = _model(workloads, model, shape)
    batches = _batches(d, dtype, STEPS, seed=200 + shape)
    ref = _alone(est, batches)
    out = torch.full_like(ref[0], -1)

    def enqueue():
        for b in batches:
            est.predict_indices(b, out=out)

    _chained(enqueue, mode)
    est.sync_check()
    assert torch.equal(out, ref[-1]), f"{int((out != ref[-1]).sum())} labels differ from the last batch's"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", SHAPES)
def test_chain_of_different_models(workloads, shape, mode):
    """GaussianNB (float32 rows) -> LR -> KMeans -> GaussianNB (float64 rows), back to back on one stream"""
    import torch
    chain = [_model(workloads, m, shape) for m in ("gnb_f32", "logistic", "kmeans", "gnb_f64")]
    rows = [_batches(d, dtype, 1, seed=300 + i)[0] for i, (_, d, dtype) in enumerate(chain)]
    ref = [_alone(est, [x])[0] for (est, _, _), x in zip(chain, rows)]
    labels = [torch.full_like(r, -1) for r in ref]

    def enqueue():
        for (est, _, _), x, lab in zip(chain, rows, labels):
            est.predict_indices(x, out=lab)

    _chained(enqueue, mode)
    for (est, _, _), lab, r, name in zip(chain, labels, ref, ("gnb_f32", "logistic", "kmeans", "gnb_f64")):
        est.sync_check()
        assert torch.equal(lab, r), f"{name}: {int((lab != r).sum())} labels differ"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", SHAPES)
def test_sticky_flag_and_refined_count_across_a_chain(workloads, shape, mode):
    """float32 GaussianNB (the pre-pass counts the rows it re-runs in fp64), one step with a NaN row in the middle of the
    chain: sync_check raises after the whole chain, and the refined rows add up to those of the batches run one at a time"""
    import torch
    batches = _batches(8, torch.float32, STEPS, seed=400 + shape)
    batches[2][12345, 3] = float("nan")
    one, _, _ = _model(workloads, "gnb_f32", shape)
    for i, b in enumerate(batches):
        one.predict_indices(b)
        torch.cuda.synchronize()
        if i == 2:
            with pytest.raises(ValueError, match="NaN|infinity"):
                one.sync_check()
        else:
            one.sync_check()
    refined = int(one.stats()[6])
    assert refined > 0
    est, _, _ = _model(workloads, "gnb_f32", shape)
    est.predict_indices(batches[0])                    # first launch (attributes) outside the capture
    est.sync_check()
    before = int(est.stats()[6])
    out = torch.empty(len(batches[0]), dtype=torch.int32, device="cuda")

    def enqueue():
        for b in batches:
            est.predict_indices(b, out=out)

    _chained(enqueue, mode)
    with pytest.raises(ValueError, match="NaN|infinity"):
        est.sync_check()
    est.sync_check()                                   # the flag was read and cleared
    assert int(est.stats()[6]) - before == refined


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("model", MODELS)
def test_host_pointer_chunks_equal_the_device_call(workloads, model, shape):
    """host rows in five chunks alternating between the pipeline's two streams: the labels of one device-pointer call"""
    est, d, dtype = _model(workloads, model, shape)
    Xd = _batches(d, dtype, 1, seed=500 + shape)[0]
    ref = _alone(est, [Xd])[0].cpu().numpy()
    X = Xd.cpu().numpy()
    est.set_option(_lib.OPT_CHUNK_ROWS, -(-len(X) // 5))
    got = est.predict_indices(X)
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} labels differ"
