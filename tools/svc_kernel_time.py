#!/usr/bin/env python
"""Device time of the linear SVC label path: the collapsed path (per pair W_p . x - rho_p with a certified error bound,
csrc/svc.cu) against the fp64 kernel's walk over the support vectors (TCSDN_OPT_ENGINE = 1) on the same handle's model.
Workload: SVC(kernel='linear') fitted on 6 000 standardised synthetic flows (6 classes, 15 pairs, 12 features) and N float32
device rows (default 10M: the bench's flow rows, log1p-transformed and standardised on the device).  CUDA events after
warm-up, the two paths alternated, each REPS times.  Prints the card and its power limit, ms and rows/s per path, the rows the
collapsed path handed to the fp64 kernel (stats[6]) and whether the two label vectors are identical."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import bench
import svc_kernel_oracle as so
from traffic_classifier_sdn_b200 import _lib, from_sklearn

REPS = 5
n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
sk = so.fit("linear", {}, n=6000, seed=77)
print(f"model: SVC(kernel='linear'), {len(sk.classes_)} classes, {sk.support_vectors_.shape[0]} support vectors, "
      f"{sk.support_vectors_.shape[1]} features")
raw = bench.synth_rows(n, 12, seed=3, device=torch.device("cuda", 0))
X = torch.log1p(raw.abs())
X = ((X - X.mean(0)) / (X.std(0) + 1e-12)).to(torch.float32).contiguous()
del raw
models = {"collapsed": from_sklearn(sk), "fp64": from_sklearn(sk).set_option(_lib.OPT_ENGINE, 1)}
labels = {}
for name, est in models.items():   # warm-up: module loads
    labels[name] = est.predict_indices(X)
torch.cuda.synchronize()
times = {k: [] for k in models}
refined = {}
for _ in range(REPS):
    for name, est in models.items():
        r0 = est.stats()[6]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        out = est.predict_indices(X)
        ev[1].record()
        torch.cuda.synchronize()
        times[name].append(ev[0].elapsed_time(ev[1]))
        refined[name] = int(est.stats()[6] - r0)
        del out
for est in models.values():
    est.sync_check()
base = min(times["fp64"])
for name, ts in times.items():
    best = min(ts)
    print(f"{name:9s} best {best:9.3f} ms  median {sorted(ts)[len(ts) // 2]:9.3f} ms  {n / best * 1e3:.3e} rows/s  "
          f"x{base / best:.1f} of the fp64 kernel  rows re-run in fp64 {refined[name]}")
same = bool(torch.equal(labels["collapsed"], labels["fp64"]))
print(f"collapsed labels equal the fp64 kernel's on all {n} rows: {same}")
hist = np.bincount(labels["fp64"].cpu().numpy(), minlength=len(sk.classes_))
print(f"label histogram: {hist.tolist()}")
sys.exit(0 if same else 1)
