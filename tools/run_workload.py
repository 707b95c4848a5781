#!/usr/bin/env python
"""Run one bench workload a few times on device-resident rows (for a profiler): tools/run_workload.py <name> <rows> [reps]"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from traffic_classifier_sdn_b200 import from_spec
name, rows = sys.argv[1], int(sys.argv[2]); reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
w = bench.build_workload(name)
est = from_spec(w["spec"])
for kv in os.environ.get("TCSDN_TOOL_OPTS", "").split(","):   # e.g. TCSDN_TOOL_OPTS=8=0,7=16 -> tcsdn_set_option(key, value)
    if kv:
        est.set_option(int(kv.split("=")[0]), int(kv.split("=")[1]))
X = bench.synth_rows(rows, w["d"], seed=1000, device=torch.device("cuda", 0))
out = torch.empty(rows, dtype=torch.int32, device="cuda")
for _ in range(reps):
    est.predict_indices(X, out=out)
torch.cuda.synchronize()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
ev0.record(); est.predict_indices(X, out=out); ev1.record(); torch.cuda.synchronize()
print(name, rows, "rows:", ev0.elapsed_time(ev1), "ms", rows / ev0.elapsed_time(ev1) * 1e3, "rows/s", est.stats().tolist())
