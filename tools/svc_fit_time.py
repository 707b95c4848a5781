"""SVC().fit(X, y, backend="gpu") (csrc/svc_fit.cu) against scikit-learn's SVC().fit on the host: the notebook split of
the bundled rows and synthetic flows (traffic_classifier_sdn_b200.synth, seed 3) at the sizes given, default parameters.

Per size: the GPU fit (best of 3, a host clock around the call, which returns when the model is on the host), scikit-learn
(once, or "not run" above --sk-max rows), the most iterations of any class pair and the GPU time per such iteration, and
an assertion that every fitted array is scikit-learn's, or, where scikit-learn does not run, the CPU definition's
(tests/svc_fit_oracle.py).  The card's name and power limit are read in the same run.

    python tools/svc_fit_time.py [rows ...] [--sk-max N]
"""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import traffic_classifier_sdn_b200 as tc  # noqa: E402
from traffic_classifier_sdn_b200 import synth  # noqa: E402
from svc_fit_oracle import CONTRACT, contract_diff, fit  # noqa: E402


def main():
    args = sys.argv[1:]
    sk_max = 50000
    if "--sk-max" in args:
        i = args.index("--sk-max")
        sk_max = int(args[i + 1])
        del args[i:i + 2]
    sizes = [int(a) for a in args] or [20000, 50000, 100000]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"device: {card}")
    from conftest import load_golden
    from sklearn.model_selection import train_test_split
    from sklearn.svm import SVC
    g = load_golden()
    Xtr, _, ytr, _ = train_test_split(g["X"], g["y"], test_size=0.5, random_state=101)
    data = [("notebook split", Xtr, ytr)] + [(f"{n} synthetic", *synth.make_flows(n, seed=3)) for n in sizes]
    tc.SVC().fit(Xtr[:200], ytr[:200], backend="gpu")   # load the module and create the context
    print("| training rows | classes | GPU fit (best of 3) | scikit-learn | most iterations of one pair | GPU time per "
          "iteration | support vectors |")
    print("|---|---|---|---|---|---|---|")
    for name, X, y in data:
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            est = tc.SVC().fit(X, y, backend="gpu")
            ts.append(time.perf_counter() - t0)
        it = int(max(est.n_iter_))
        sk_t = "not run"
        mine = {k: getattr(est, k) for k in CONTRACT}
        if len(X) <= sk_max:
            t0 = time.perf_counter()
            sk = SVC().fit(X, y)
            sk_t = f"{time.perf_counter() - t0:.2f} s"
            ref = {k: getattr(sk, k if k != "n_support_" else "_n_support") for k in CONTRACT}
            assert contract_diff(mine, ref) == [], f"{name}: the GPU fit differs from scikit-learn"
        else:
            assert contract_diff(mine, fit(X, y)) == [], f"{name}: the GPU fit differs from the CPU definition"
        print(f"| {name} ({len(X)}) | {len(est.classes_)} | {min(ts):.3f} s | {sk_t} | {it} | "
              f"{min(ts) / max(it, 1) * 1e6:.1f} us | {len(est.support_)} |", flush=True)


if __name__ == "__main__":
    main()
