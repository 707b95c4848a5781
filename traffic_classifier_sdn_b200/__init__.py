"""traffic_classifier_sdn_b200 -- H100-native (sm_90a) per-flow classification for Traffic-classifier-SDN.

The package replaces one call of the reference, ``model.predict(rows)`` at ``traffic_classifier.py:106``, for its
six scikit-learn estimators, with hand-written CUDA kernels behind a C ABI (``include/tcsdn.h``,
``libtcsdn.so``) and an sklearn-like Python surface:

    from traffic_classifier_sdn_b200 import load_model
    model = load_model("models/RandomForestClassifier")   # the reference's own pickle, read as data
    labels = model.predict(rows)                           # runs on the GPU; no CPU fallback exists
"""
from .estimators import (GaussianNB, KMeans, KNeighborsClassifier, LogisticRegression, NotFittedError,  # noqa: F401
                         RandomForestClassifier, SVC, from_sklearn, from_spec, load_model)
from .modelio import MODEL_FILES, load_reference_pickle, spec_from_estimator  # noqa: F401

__version__ = "0.1.0"
