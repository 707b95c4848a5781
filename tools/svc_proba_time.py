#!/usr/bin/env python
"""Device time of SVC.predict_proba against the decision values it starts from, on one handle.
Workload: SVC(kernel='rbf', probability=True) fitted on 6 000 standardised synthetic flows (6 classes, 15 pairs, 12
features) and N float32 device rows (default 10M: the bench's flow rows, log1p-transformed and standardised on the device).
Both calls run the fp64 register kernel: score-only tcsdn_predict (the decision values, labels discarded) and
tcsdn_svc_predict_proba (the same walk plus Platt scaling and pairwise coupling per row).  CUDA events after warm-up, the
two calls alternated, each REPS times.  Prints the card and its power limit, best and median ms per call, the overhead of
the probabilities over the decision values, and whether argmax(predict_proba) agrees with predict on a sample."""
import os
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import bench
import svc_proba_oracle as po
from traffic_classifier_sdn_b200 import _lib, from_sklearn

warnings.simplefilter("ignore", FutureWarning)
REPS = 5
n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
sk = po.fit("rbf", 6, n=6000, seed=77)
print(f"model: SVC(kernel='rbf', probability=True), {len(sk.classes_)} classes, {sk.support_vectors_.shape[0]} support vectors, "
      f"{sk.support_vectors_.shape[1]} features")
raw = bench.synth_rows(n, 12, seed=3, device=torch.device("cuda", 0))
X = torch.log1p(raw.abs())
X = ((X - X.mean(0)) / (X.std(0) + 1e-12)).to(torch.float32).contiguous()
del raw
est = from_sklearn(sk)
lib = _lib.load()
labels = torch.empty(n, dtype=torch.int32, device="cuda")
scores = torch.empty((n, 15), dtype=torch.float64, device="cuda")
proba = torch.empty((n, 6), dtype=torch.float64, device="cuda")


def decision_values():
    _lib.check(lib.tcsdn_predict(est._handle, X.data_ptr(), n, 12, _lib.F32, _lib.DEVICE, labels.data_ptr(), scores.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream))


def predict_proba():
    _lib.check(lib.tcsdn_svc_predict_proba(est._handle, X.data_ptr(), n, 12, _lib.F32, _lib.DEVICE, proba.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream))


calls = {"decision_values": decision_values, "predict_proba": predict_proba}
for fn in calls.values():   # warm-up: module loads
    fn()
torch.cuda.synchronize()
times = {k: [] for k in calls}
for _ in range(REPS):
    for name, fn in calls.items():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        times[name].append(ev[0].elapsed_time(ev[1]))
est.sync_check()
for name, ts in times.items():
    print(f"{name:15s} best {min(ts):9.3f} ms  median {sorted(ts)[len(ts) // 2]:9.3f} ms  {n / min(ts) * 1e3:.3e} rows/s")
over = min(times["predict_proba"]) / min(times["decision_values"]) - 1
print(f"overhead of the probabilities over the decision values: {100 * over:+.1f} % (best against best)")
s = slice(0, n, 10_007)
p = proba[s].cpu().numpy()
ok = bool(np.all(np.abs(p.sum(axis=1) - 1) <= 1e-12))
agree = float(np.mean(p.argmax(axis=1) == labels[s].cpu().numpy()))
print(f"sample of {p.shape[0]} rows: rows sum to 1 within 1e-12: {ok}; argmax(predict_proba) == predict on {100 * agree:.2f} %")
sys.exit(0 if ok else 1)
