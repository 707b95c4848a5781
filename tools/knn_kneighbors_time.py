#!/usr/bin/env python
"""Device time of KNeighborsClassifier.kneighbors against predict_indices on the bench KNN workload (10M device rows x 50k
training rows, k = 5): CUDA events after warm-up, the variants alternated, each repeated REPS times.  Prints the card and its
power limit, rows/s per variant, the tie rows re-run in index order (stats[7]), and checks on the device that the vote of
y[ind] equals predict_indices on every row.  --profile: afterwards, one torch.profiler run per variant, kernel time by name
(profiling in its own phase, so that the timings above are taken without it)."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from traffic_classifier_sdn_b200 import from_spec

REPS = 3
n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
w = bench.build_workload("knn")
spec = w["spec"]
X = bench.synth_rows(n, w["d"], seed=3, device=torch.device("cuda", 0))
est = from_spec(spec)
variants = {
    "predict_indices": lambda: est.predict_indices(X),
    "kneighbors(m=5)": lambda: est.kneighbors(X, 5),
    "kneighbors(m=5, return_distance=False)": lambda: est.kneighbors(X, 5, return_distance=False),
    "kneighbors(m=32)": lambda: est.kneighbors(X, 32),
}
for f in variants.values():   # warm-up: module loads, pool allocations
    f()
torch.cuda.synchronize()
est.sync_check()
times = {k: [] for k in variants}
ties = {}
for _ in range(REPS):
    for name, f in variants.items():
        t0 = est.stats()[7]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        out = f()
        ev[1].record()
        torch.cuda.synchronize()
        times[name].append(ev[0].elapsed_time(ev[1]))
        ties[name] = int(est.stats()[7] - t0)
        del out
base = min(times["predict_indices"])
for name, ts in times.items():
    best = min(ts)
    print(f"{name:40s} best {best:8.2f} ms  median {sorted(ts)[len(ts) // 2]:8.2f} ms  {n / best * 1e3:.3e} rows/s  "
          f"x{best / base:.3f} of predict_indices  tie rows {ties[name]}")

lab = est.predict_indices(X)
dist, ind = est.kneighbors(X, 5)
est.sync_check()
y = torch.from_numpy(spec["y"]).to(device=X.device, dtype=torch.int64)
cnt = torch.zeros((n, len(spec["classes"])), dtype=torch.int32, device=X.device)
cnt.scatter_add_(1, y[ind], torch.ones_like(ind, dtype=torch.int32))
same = bool(torch.equal(cnt.argmax(1).to(torch.int32), lab))   # argmax: first maximum, as predict's vote
print(f"vote of y[ind] equals predict_indices on all {n} rows: {same}")
del cnt, dist, ind

if "--profile" in sys.argv:
    from torch.profiler import ProfilerActivity, profile
    for name in ("predict_indices", "kneighbors(m=5)", "kneighbors(m=32)"):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            variants[name]()
            torch.cuda.synchronize()
        tot = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                key = e.name.split("(")[0][:60]
                tot[key] = tot.get(key, 0.0) + e.device_time_total / 1e3
        print(f"profile {name}: " + "; ".join(f"{k} {v:.2f} ms" for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:6]))
sys.exit(0 if same else 1)
