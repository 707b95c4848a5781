import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

KINDS = ("linear", "gnb", "kmeans", "knn", "svc", "forest")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden():
    """tests/golden/bundled.*.npz, merged: the reference's bundled rows, its six models' parameters and
    scikit-learn's answers (made by tests/golden/make_golden.py, split into parts below 1 MB)."""
    g = {}
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "bundled.*.npz"))):
        z = np.load(path, allow_pickle=False)
        g.update({k: z[k] for k in z.files})
    assert "X" in g, "tests/golden/bundled.*.npz missing"
    return g


@pytest.fixture(scope="session")
def golden():
    return load_golden()


def spec_from_golden(g, kind):
    spec = {"kind": kind}
    for k, v in g.items():
        if k.startswith(kind + ".") and not k.startswith(kind + ".expected"):
            name = k.split(".", 1)[1]
            spec[name] = v.item() if v.ndim == 0 else v
    for key in ("n_features", "k", "n_classes"):
        if key in spec:
            spec[key] = int(spec[key])
    if "gamma" in spec:
        spec["gamma"] = float(spec["gamma"])
    for key in ("decision_function_shape",):
        if key in spec:
            spec[key] = str(spec[key])
    if "break_ties" in spec:
        spec["break_ties"] = bool(spec["break_ties"])
    return spec


@pytest.fixture(scope="session")
def specs(golden):
    return {k: spec_from_golden(golden, k) for k in KINDS}
