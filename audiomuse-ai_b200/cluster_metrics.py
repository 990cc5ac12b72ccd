"""Clustering scores on the GPU: the three ``sklearn.metrics`` functions tasks/clustering_helper.py:462-470 calls once
per evolutionary iteration on the matrix it just clustered.

    silhouette_score(X, labels, metric="euclidean")     -> float   (mean of silhouette_samples)
    silhouette_samples(X, labels, metric="euclidean")   -> float64 [N]
    davies_bouldin_score(X, labels)                     -> float
    calinski_harabasz_score(X, labels)                  -> float

Same meaning, return types and special cases as scikit-learn; all three run in am_cluster_scores.  Validation happens
on the host before any GPU work and raises scikit-learn's ValueError (label count outside 2 .. N - 1, length mismatch,
NaN / inf, a metric other than euclidean): the reference catches ValueError and scores the metric 0.  Labels are
re-encoded to 0 .. L - 1 like scikit-learn's LabelEncoder, so DBSCAN's -1 is an ordinary label.  float64 input is cast
to float32 for the device.  A GPU failure raises unless ``B200_ALLOW_SKLEARN_FALLBACK=1``, in which case scikit-learn
computes the value (the contract of clustering_gpu.GPUKMeans / GPUDBSCAN / GPUPCA).
"""
from __future__ import annotations

import logging
import os

import numpy as np

from . import _lib

logger = logging.getLogger("tasks.clustering_helper")

_SILHOUETTE, _DAVIES_BOULDIN, _CALINSKI_HARABASZ = 1, 2, 4


def _validate(X, labels, metric="euclidean"):
    """-> (X, labels re-encoded to int32 0..L-1, L), raising what scikit-learn raises for bad input"""
    from sklearn.preprocessing import LabelEncoder
    from sklearn.utils import check_X_y

    if metric != "euclidean":
        raise ValueError(f"metric={metric!r} is not supported on the GPU: only 'euclidean'")
    X, labels = check_X_y(X, labels)
    le = LabelEncoder()
    enc = le.fit_transform(labels)
    n_labels, n_samples = len(le.classes_), X.shape[0]
    if not 1 < n_labels < n_samples:
        raise ValueError("Number of labels is %d. Valid values are 2 to n_samples - 1 (inclusive)" % n_labels)
    return X, enc.astype(np.int32), n_labels


def _device_scores(X, enc, n_labels, which, want_samples=False):
    X32 = np.ascontiguousarray(X, dtype=np.float32)
    enc = np.ascontiguousarray(enc, dtype=np.int32)
    scores = np.zeros(3, dtype=np.float64)
    samples = np.empty(X32.shape[0], dtype=np.float32) if want_samples else None
    _lib.check(_lib.load().am_cluster_scores(_lib.ptr(X32), X32.shape[0], X32.shape[1], _lib.ptr(enc), int(n_labels),
                                             int(which), _lib.ptr(scores),
                                             None if samples is None else _lib.ptr(samples)))
    return scores, samples


def _run(name, gpu, cpu):
    try:
        return gpu()
    except Exception as e:
        if os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") != "1":
            raise
        logger.warning(f"GPU {name} failed, falling back to CPU: {e}")
    return cpu()


def silhouette_samples(X, labels, metric="euclidean"):
    X, enc, n_labels = _validate(X, labels, metric)

    def cpu():
        from sklearn.metrics import silhouette_samples as sk
        return sk(X, labels, metric=metric)

    return _run("silhouette_samples",
                lambda: _device_scores(X, enc, n_labels, _SILHOUETTE, want_samples=True)[1].astype(np.float64), cpu)


def silhouette_score(X, labels, metric="euclidean"):
    X, enc, n_labels = _validate(X, labels, metric)

    def cpu():
        from sklearn.metrics import silhouette_score as sk
        return float(sk(X, labels, metric=metric))

    return _run("silhouette_score", lambda: float(_device_scores(X, enc, n_labels, _SILHOUETTE)[0][0]), cpu)


def davies_bouldin_score(X, labels):
    X, enc, n_labels = _validate(X, labels)

    def cpu():
        from sklearn.metrics import davies_bouldin_score as sk
        return float(sk(X, labels))

    return _run("davies_bouldin_score", lambda: float(_device_scores(X, enc, n_labels, _DAVIES_BOULDIN)[0][1]), cpu)


def calinski_harabasz_score(X, labels):
    X, enc, n_labels = _validate(X, labels)

    def cpu():
        from sklearn.metrics import calinski_harabasz_score as sk
        return float(sk(X, labels))

    return _run("calinski_harabasz_score",
                lambda: float(_device_scores(X, enc, n_labels, _CALINSKI_HARABASZ)[0][2]), cpu)
