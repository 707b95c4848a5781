#!/usr/bin/env python
"""Device time of KMeans.transform and KMeans.score against predict_indices, and of the GPU k-means++ seeding against
scikit-learn's, on the bench KMeans workload.
Workload: bench.py's KMeans model (6 centres, 12 features) and N float32 device rows (default 10M: the bench's flow rows).
transform writes [N][6] float64 on the device; score returns the inertia on the host (so its time includes the one
synchronisation it needs).  CUDA events after warm-up, the three calls alternated, each REPS times.  Then
kmeans_plusplus(k=6, random_state=0) on the device rows against sklearn.cluster.kmeans_plusplus on the same rows on the
host (one run: it takes seconds), with the same random numbers (float64 rows on the host: scikit-learn rounds float32 rows' distances to float32).  Prints the card and its power limit, best and median ms."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
import traffic_classifier_sdn_b200 as tc

REPS = 5
n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
w = bench._build_workload("kmeans", False)
est = tc.from_spec(w["spec"])
X = bench.synth_rows(n, 12, seed=3, device=torch.device("cuda", 0)).contiguous()
out = torch.empty(n, dtype=torch.int32, device="cuda")


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


calls = {"predict_indices": lambda: est.predict_indices(X, out=out), "transform": lambda: est.transform(X),
         "score": lambda: est.score(X)}
for f in calls.values():
    f()
torch.cuda.synchronize()
times = {k: [] for k in calls}
for _ in range(REPS):
    for k, f in calls.items():
        times[k].append(timed(f))
est.sync_check()
for k, t in times.items():
    print(f"{k:16s} best {min(t):8.3f} ms  median {float(np.median(t)):8.3f} ms  ({n} rows)")
print(f"transform / predict_indices: {min(times['transform']) / min(times['predict_indices']):.2f}x; "
      f"score / predict_indices: {min(times['score']) / min(times['predict_indices']):.2f}x")

k = 6
gpu = []
for _ in range(REPS):
    t0 = time.perf_counter()
    c_gpu, i_gpu = tc.kmeans_plusplus(X, k, random_state=0)
    gpu.append((time.perf_counter() - t0) * 1e3)
t0 = time.perf_counter()
w = np.ones(n)
np.random.RandomState(0).choice(n, p=w / w.sum())
draw_ms = (time.perf_counter() - t0) * 1e3
print(f"  of which the host draw of the first index (scikit-learn's rs.choice(n, p=ones / n)): {draw_ms:.1f} ms")
host = X.cpu().numpy().astype(np.float64)   # scikit-learn keeps float32 rows' distances in float32: compare in float64
from sklearn.cluster import kmeans_plusplus
t0 = time.perf_counter()
c_sk, i_sk = kmeans_plusplus(host, k, random_state=0)
sk_ms = (time.perf_counter() - t0) * 1e3
print(f"kmeans_plusplus k={k}: GPU best {min(gpu):.1f} ms median {float(np.median(gpu)):.1f} ms (device rows, wall clock); "
      f"scikit-learn on the host {sk_ms:.0f} ms ({os.cpu_count()} CPUs); same rows chosen: "
      f"{bool(np.array_equal(host[i_gpu], host[i_sk]))}")
