#!/usr/bin/env python
"""Wall time of RandomForestClassifier.fit on the GPU (backend="gpu", csrc/forest_fit.cu) against scikit-learn's on the
host, n_jobs=1 and n_jobs=-1.  Workload: synthetic flows (synth.make_flows, 12 features, 6 classes) at 20k, 200k and 1M
rows (or the row counts given as arguments), n_estimators=100, random_state=0, every other parameter at its default.

The GPU fit is split into the host draws (forest_fit_plan: numpy's per-tree seeds, bootstrap indices and splitter states)
and the library call (upload of the rows, y and bootstrap indices, the trees, and the copy of the node arrays back).  The
library call is timed again with the rows already on the device (a CUDA float32 tensor).  scikit-learn with n_jobs=1 is
skipped above 200k rows unless --sk-serial is given (it takes minutes).  Prints the card and its power limit, best of
REPS for the GPU, one run for scikit-learn, and whether the trees are the same bits."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import traffic_classifier_sdn_b200 as tc
from traffic_classifier_sdn_b200 import synth
from traffic_classifier_sdn_b200.estimators import forest_fit_plan
from forest_fit_oracle import forest_diff, sklearn_forest

REPS = 3
T = 100
sizes = [int(a) for a in sys.argv[1:] if a.isdigit()] or [20_000, 200_000, 1_000_000]
sk_serial_all = "--sk-serial" in sys.argv
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}; host: {os.cpu_count()} CPUs")


def wall(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


from sklearn.ensemble import RandomForestClassifier as SK

for n in sizes:
    X, y = synth.make_flows(n, seed=0)
    p = dict(n_estimators=T, random_state=0)
    tc.RandomForestClassifier(n_estimators=2, random_state=0).fit(X[:1000], y[:1000], backend="gpu")   # warm-up
    draws = min(wall(lambda: forest_fit_plan(p, n, X.shape[1]))[0] for _ in range(REPS))
    host = [wall(lambda: tc.RandomForestClassifier(**p).fit(X, y, backend="gpu")) for _ in range(REPS)]
    est = host[-1][1]
    Xd = torch.from_numpy(X.astype(np.float32)).cuda()
    yd = torch.from_numpy(y).cuda()
    torch.cuda.synchronize()
    dev = [wall(lambda: tc.RandomForestClassifier(**p).fit(Xd, yd, backend="gpu"))[0] for _ in range(REPS)]
    best = min(t for t, _ in host)
    nodes = int(est.tree_arrays_["tree_offsets"][-1])
    print(f"n={n:>9,} trees={T} nodes={nodes:,}: GPU fit best {best:9.1f} ms (host draws {draws:8.1f} ms, library call "
          f"{best - draws:8.1f} ms); device float32 rows {min(dev):9.1f} ms")
    sk_par_ms, sk = wall(lambda: SK(n_jobs=-1, **p).fit(X, y))
    same = forest_diff(dict(est.tree_arrays_, feature_importances=est.feature_importances_), sklearn_forest(sk)) == []
    line = f"             scikit-learn n_jobs=-1 {sk_par_ms:9.1f} ms"
    if n <= 200_000 or sk_serial_all:
        sk_ms = wall(lambda: SK(n_jobs=1, **p).fit(X, y))[0]
        line += f", n_jobs=1 {sk_ms:9.1f} ms"
    print(f"{line}; same trees: {same}")
