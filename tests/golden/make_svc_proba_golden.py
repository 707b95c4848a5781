#!/usr/bin/env python
"""Generate tests/golden/svc_proba.npz: scikit-learn's SVC(probability=True) on the bundled rows.

    python tests/golden/make_svc_proba_golden.py

The model is ``SVC(probability=True, random_state=0)`` (rbf, scikit-learn's defaults otherwise) fitted on the 7 653 rows
of tests/golden/bundled.*.npz (the reference's five training files, make_golden.py's recipe), each labelled by the file
it came from.  Stored: the fitted spec arrays (``spec.<key>``, modelio's SVC spec, with ``prob_a`` / ``prob_b``), and
scikit-learn's one-vs-one ``decision_function`` and ``predict_proba`` of every row.  scikit-learn 1.9 deprecates
``probability`` and will remove it; this file keeps its behaviour on record for the models pickled before then.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from conftest import load_golden  # noqa: E402
from traffic_classifier_sdn_b200 import modelio  # noqa: E402


def main():
    import sklearn
    from sklearn.svm import SVC
    g = load_golden()
    X, y = g["X"], g["y"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        sk = SVC(probability=True, random_state=0).fit(X, y)
    spec = modelio.spec_from_estimator(sk)
    out = {f"spec.{k}": (np.asarray(v).astype(str) if np.asarray(v).dtype == object else np.asarray(v))
           for k, v in spec.items() if k != "kind"}
    sk.decision_function_shape = "ovo"
    out["dec_ovo"] = sk.decision_function(X)
    out["proba"] = sk.predict_proba(X)
    out["sklearn_version"] = np.asarray(sklearn.__version__)
    path = os.path.join(HERE, "svc_proba.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes;", spec["sv"].shape[0], "support vectors,", len(spec["classes"]), "classes")


if __name__ == "__main__":
    main()
