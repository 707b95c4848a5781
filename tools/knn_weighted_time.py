#!/usr/bin/env python
"""Device time of the distance-weighted KNN vote against the uniform vote on the bench KNN workload (10M device rows x 50k
training rows, k = 5): predict_indices on two handles of the same model, weights='uniform' and weights='distance', CUDA
events after warm-up, the two alternated, each repeated REPS times.  Prints the card and its power limit, rows/s per variant,
the tie rows re-run in index order (stats[7]), and checks the weighted labels of a seeded sample of rows against the CPU
definition (tests/knn_weighted_oracle.py)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import bench
import knn_weighted_oracle as kwo
from traffic_classifier_sdn_b200 import from_spec

REPS = 5
SAMPLE = 2000
n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
w = bench.build_workload("knn")
spec = w["spec"]
X = bench.synth_rows(n, w["d"], seed=3, device=torch.device("cuda", 0))
models = {"uniform": from_spec(dict(spec, weights="uniform")), "distance": from_spec(dict(spec, weights="distance"))}
for est in models.values():   # warm-up: module loads, pool allocations
    est.predict_indices(X)
torch.cuda.synchronize()
times = {k: [] for k in models}
ties = {}
for _ in range(REPS):
    for name, est in models.items():
        t0 = est.stats()[7]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        out = est.predict_indices(X)
        ev[1].record()
        torch.cuda.synchronize()
        times[name].append(ev[0].elapsed_time(ev[1]))
        ties[name] = int(est.stats()[7] - t0)
        del out
for est in models.values():
    est.sync_check()
base = min(times["uniform"])
for name, ts in times.items():
    best = min(ts)
    print(f"weights={name:9s} best {best:8.2f} ms  median {sorted(ts)[len(ts) // 2]:8.2f} ms  {n / best * 1e3:.3e} rows/s  "
          f"x{best / base:.4f} of uniform  tie rows {ties[name]}")

lab = models["distance"].predict_indices(X)
rng = np.random.default_rng(17)
sel = np.sort(rng.choice(n, SAMPLE, replace=False))
sel_d = torch.from_numpy(sel).cuda()
ref, _ = kwo.predict(dict(spec, weights="distance"), X[sel_d].cpu().numpy())
same = bool(np.array_equal(lab[sel_d].cpu().numpy(), ref))
print(f"weighted labels equal the definition on a seeded sample of {SAMPLE} rows: {same}")
changed = int((lab != models["uniform"].predict_indices(X)).sum())
print(f"rows whose label differs between the uniform and the weighted vote: {changed} of {n}")
sys.exit(0 if same else 1)
