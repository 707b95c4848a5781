#!/usr/bin/env python
"""Generate tests/golden/bundled.*.npz and tests/golden/datasets/ from the reference tree.

    python tests/golden/make_golden.py REFERENCE_DIR

Inputs (read-only): the reference's five ``datasets/*_training_data.csv`` and its six
``models/*`` pickles.  The rows are assembled with the notebooks' recipe (SURVEY.md 8c:
ping, voice, dns, telnet tab-separated, game comma-separated, concat, dropna, drop the four
cumulative counters).  Expected outputs come from scikit-learn itself -- the library whose
``predict`` the reference calls at traffic_classifier.py:106 -- evaluated on estimators
revived from the pickles: the four that still unpickle are loaded with ``pickle.load`` and
must agree exactly with their rebuilt twins; KNeighbors / RandomForestClassifier are rebuilt
from the data-only spec (tests/sk_rebuild.py).  Nothing under /root/reference is copied as
source; the .npz files hold numeric rows, fitted parameters and sklearn's answers, split into parts of
less than 1 MB each (tests/conftest.py load_golden() merges them).  datasets/ holds the first and last
lines of each training file, so that the recipe test (tests/test_dataio.py) runs on the notebooks' own
text, together with the positions of those rows in the golden rows.
"""
import io
import os
import pickle
import sys
import warnings

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from traffic_classifier_sdn_b200 import modelio  # noqa: E402
from sk_rebuild import sklearn_from_spec  # noqa: E402

DROP = ["Forward Packets", "Forward Bytes", "Reverse Packets", "Reverse Bytes"]
PART_BYTES = 900_000          # compressed size of one golden part (every file stays below 1 MB)
SAMPLE_HEAD, SAMPLE_TAIL = 40, 8   # data lines kept from the start and the end of each training file


def save_parts(out):
    """Greedy split of `out` into tests/golden/bundled.<i>.npz, each at most PART_BYTES compressed."""
    def size(a):
        b = io.BytesIO()
        np.savez_compressed(b, a=a)
        return len(b.getvalue())
    parts, cur, cur_bytes = [], {}, 0
    for k in sorted(out, key=lambda k: -size(out[k])):
        n = size(out[k])
        assert n <= PART_BYTES, k
        if cur and cur_bytes + n > PART_BYTES:
            parts.append(cur)
            cur, cur_bytes = {}, 0
        cur[k] = out[k]
        cur_bytes += n
    parts.append(cur)
    for i, part in enumerate(parts):
        path = os.path.join(HERE, f"bundled.{i}.npz")
        np.savez_compressed(path, **part)
        print("wrote", path, os.path.getsize(path), "bytes")


def save_dataset_samples(ref):
    """Head and tail of every training file (as text), and where their rows sit in the golden rows."""
    os.makedirs(os.path.join(HERE, "datasets"), exist_ok=True)
    rows, offset = [], 0
    for name, sep in (("ping", "\t"), ("voice", "\t"), ("dns", "\t"), ("telnet", "\t"), ("game", ",")):
        src = os.path.join(ref, "datasets", f"{name}_training_data.csv")
        with open(src, "rb") as fh:
            lines = fh.read().split(b"\n")
        tail_nl = lines[-1] == b""          # a file that ends in a newline splits into a last empty piece
        data = lines[1:-1] if tail_nl else lines[1:]
        keep = list(range(SAMPLE_HEAD)) + list(range(len(data) - SAMPLE_TAIL, len(data)))
        with open(os.path.join(HERE, "datasets", f"{name}_training_data.csv"), "wb") as fh:
            fh.write(b"\n".join([lines[0]] + [data[i] for i in keep]) + (b"\n" if tail_nl else b""))
        n_rows = len(pd.read_csv(src, delimiter=sep).dropna())
        complete = len(pd.read_csv(src, delimiter=sep)) == n_rows   # only a truncated last line is dropped
        rows += [offset + i for i in keep if complete or i < len(data) - 1]
        offset += n_rows
    np.save(os.path.join(HERE, "datasets", "rows.npy"), np.asarray(rows, np.int32))


def load_bundled_rows(ref):
    frames = []
    for name, sep in (("ping", "\t"), ("voice", "\t"), ("dns", "\t"), ("telnet", "\t"), ("game", ",")):
        frames.append(pd.read_csv(os.path.join(ref, "datasets", f"{name}_training_data.csv"), delimiter=sep))
    df = pd.concat(frames, ignore_index=True).dropna()
    df = df.drop(columns=DROP)
    y = df["Traffic Type"].to_numpy().astype(str)
    X = df.drop(columns=["Traffic Type"]).to_numpy(dtype=np.float64)
    return np.ascontiguousarray(X), y


def main():
    ref = sys.argv[1]
    warnings.simplefilter("ignore")
    X, y = load_bundled_rows(ref)
    assert X.shape == (7653, 12), X.shape
    out = {"X": X, "y": y}
    for word, fname in modelio.MODEL_FILES.items():
        path = os.path.join(ref, "models", fname)
        spec = modelio.load_reference_pickle(path)
        kind = spec["kind"]
        for k, v in spec.items():
            if k == "kind":
                continue
            a = np.asarray(v)
            out[f"{kind}.{k}"] = a.astype(str) if a.dtype == object else a
        sk = sklearn_from_spec(spec)
        if kind == "knn":
            # one thread => sklearn's thread-count-independent `parallel_on_X` reduction (n > 4*256*1)
            from threadpoolctl import threadpool_limits
            threadpool_limits(limits=1)
        direct = None
        try:
            with open(path, "rb") as fh:
                direct = pickle.load(fh)
        except Exception as exc:  # KNeighbors, RandomForestClassifier under sklearn >= 1.3
            print(f"{fname}: pickle.load fails here ({type(exc).__name__}); using the rebuilt estimator")
        pred = sk.predict(X)
        if direct is not None:
            assert np.array_equal(np.asarray(direct.predict(X)), np.asarray(pred)), fname
        classes = np.asarray(spec["classes"])
        if kind == "kmeans":
            lab = np.asarray(pred, np.int32)
        else:
            lab = np.searchsorted(classes, pred).astype(np.int32)
            assert np.array_equal(classes[lab], pred)
        out[f"{kind}.expected_label"] = lab
        if kind == "linear":
            s = sk.decision_function(X)
            if direct is not None:
                assert np.array_equal(direct.decision_function(X), s)
            out["linear.expected_score"] = s
        elif kind == "gnb":
            s = sk._joint_log_likelihood(X)
            if direct is not None:
                assert np.array_equal(direct._joint_log_likelihood(X), s)
            out["gnb.expected_score"] = s
        elif kind == "kmeans":
            out["kmeans.expected_score"] = sk.transform(X)  # euclidean distances to centers
        elif kind == "knn":
            kd = sklearn_from_spec(spec, knn_algorithm="kd_tree")  # what 'auto' picks for 12 features
            assert np.array_equal(kd.predict(X), pred), "kd_tree and brute disagree"
            out["knn.expected_score"] = np.rint(sk.predict_proba(X) * spec["k"]).astype(np.uint8)
        elif kind == "svc":
            sk.decision_function_shape = "ovo"
            s = sk.decision_function(X)
            sk.decision_function_shape = spec["decision_function_shape"]
            if direct is not None:
                direct.decision_function_shape = "ovo"
                assert np.array_equal(direct.decision_function(X), s)
            out["svc.expected_score"] = s
            out["svc.expected_ovr"] = sk.decision_function(X)
        elif kind == "forest":
            out["forest.expected_score"] = sk.predict_proba(X)
        agree = float(np.mean(classes[lab] == y)) if kind != "kmeans" else float("nan")
        print(f"{fname}: kind={kind} labels ok, agreement with CSV labels {agree:.4f}")
    save_parts(out)
    save_dataset_samples(ref)


if __name__ == "__main__":
    main()
