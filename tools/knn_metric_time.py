#!/usr/bin/env python
"""Device time of KNeighborsClassifier(metric='manhattan' | 'chebyshev') on the bench KNN workload (10M float32 device rows x
the 50k-row synthetic model, k = 5): the pruned CUDA-core kernel (engine option 0) against the fp64 kernel (engine option 1),
alternated, REPS runs each, with the euclidean tensor-core engine timed in the same call as the yardstick.  Prints the card,
its power limit and SM clock, per run the time, stats[4] (tiles per pass x 1000) and stats[7] (tie rows re-run in index
order), checks that the two paths give identical labels on every row, then sweeps small batches (1k .. 64k rows) to place
the dispatch crossover between the two kernels."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import bench
from traffic_classifier_sdn_b200 import _lib, from_spec

REPS = 5
n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card (name, power limit, SM clock, max SM clock): {card}")
w = bench.build_workload("knn")
spec = w["spec"]
X = bench.synth_rows(n, w["d"], seed=3, device=torch.device("cuda", 0))


def timed(est, Xd):
    s0 = est.stats()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    out = est.predict_indices(Xd)
    ev[1].record()
    torch.cuda.synchronize()
    s1 = est.stats()
    return ev[0].elapsed_time(ev[1]), out, int(s1[4]), int(s1[7] - s0[7])


ok = True
euclid = from_spec(dict(spec, metric="euclidean"))
euclid.predict_indices(X)
for metric in ("manhattan", "chebyshev"):
    models = {"pruned": from_spec(dict(spec, metric=metric)), "fp64": from_spec(dict(spec, metric=metric))}
    models["fp64"].set_option(_lib.OPT_ENGINE, 1)
    for est in models.values():   # warm-up: module loads, pool allocations
        est.predict_indices(X)
    torch.cuda.synchronize()
    times = {k: [] for k in list(models) + ["euclidean"]}
    labels = {}
    for r in range(REPS):
        for name, est in list(models.items()) + [("euclidean", euclid)]:
            ms, out, tiles, ties = timed(est, X)
            times[name].append(ms)
            labels[name] = out
            print(f"{metric:9s} run {r} {name:9s} {ms:9.2f} ms  stats[4] {tiles}  stats[7] (this call) {ties}")
    for est in models.values():
        est.sync_check()
    for name, ts in times.items():
        best = min(ts)
        print(f"{metric:9s} {name:9s} best {best:9.2f} ms  median {sorted(ts)[len(ts) // 2]:9.2f} ms  {n / best * 1e3:.3e} rows/s")
    same = bool(torch.equal(labels["pruned"], labels["fp64"]))
    ok &= same
    print(f"{metric}: labels identical between the pruned and the fp64 kernel on all {n} rows: {same}")

    # crossover: forced pruned kernel (option 2) against the fp64 kernel, median of 7 calls per size
    pr = from_spec(dict(spec, metric=metric))
    pr.set_option(_lib.OPT_ENGINE, 2)
    for m in (1024, 4096, 16384, 65536):
        Xs = X[:m].contiguous()
        res = {}
        for name, est in (("pruned", pr), ("fp64", models["fp64"])):
            est.predict_indices(Xs)
            res[name] = sorted(timed(est, Xs)[0] for _ in range(7))[3]
        print(f"{metric:9s} crossover n={m:6d}  pruned {res['pruned']:8.3f} ms  fp64 {res['fp64']:8.3f} ms")
sys.exit(0 if ok else 1)
