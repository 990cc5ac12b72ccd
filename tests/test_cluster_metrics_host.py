"""Host-side contracts of audiomuse_ai_b200.cluster_metrics (the clustering task's silhouette / Davies-Bouldin /
Calinski-Harabasz scores) and of its integration point, tasks/clustering_helper.py.  No GPU compute is issued here."""
import os
import types

import numpy as np
import pytest

METRICS = ("silhouette_score", "davies_bouldin_score", "calinski_harabasz_score")


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "cluster_metrics_golden.npz"))


def _blobs():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.standard_normal((60, 5)) + 4, rng.standard_normal((60, 5)) - 4, rng.standard_normal((60, 5))])
    return x, np.repeat([0, 1, 2], 60)


def test_validation_raises_value_error_before_the_library(monkeypatch):
    """The reference scores a metric 0 when it raises ValueError (clustering_helper.py:462-470): every bad input must
    raise exactly that, and before any device work."""
    from audiomuse_ai_b200 import _lib, cluster_metrics as cm

    def no_library():
        raise AssertionError("validation must not reach the library")

    monkeypatch.setattr(_lib, "load", no_library)
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    x, y = _blobs()
    fns = [cm.silhouette_score, cm.silhouette_samples, cm.davies_bouldin_score, cm.calinski_harabasz_score]
    for fn in fns:
        with pytest.raises(ValueError, match="Number of labels is 1. Valid values are 2 to n_samples - 1"):
            fn(x, np.zeros(len(x), int))
        with pytest.raises(ValueError, match="Number of labels is 180. Valid values are 2 to n_samples - 1"):
            fn(x, np.arange(len(x)))
        with pytest.raises(ValueError):
            fn(x, y[:-1])
        bad = x.copy()
        bad[7, 2] = np.nan
        with pytest.raises(ValueError):
            fn(bad, y)
        bad[7, 2] = np.inf
        with pytest.raises(ValueError):
            fn(bad, y)
    for fn in (cm.silhouette_score, cm.silhouette_samples):
        with pytest.raises(ValueError, match="euclidean"):
            fn(x, y, "cosine")
        with pytest.raises(ValueError, match="euclidean"):
            fn(x, y, metric="manhattan")


@pytest.mark.skipif(not _no_gpu(), reason="exercises the no-device failure path")
def test_fallback_contract_both_settings(monkeypatch):
    """Loud by default; scikit-learn's values with B200_ALLOW_SKLEARN_FALLBACK=1 (the GPUKMeans / GPUDBSCAN / GPUPCA
    contract)."""
    from sklearn import metrics
    from audiomuse_ai_b200 import _lib, cluster_metrics as cm
    x, y = _blobs()
    y = np.where(np.arange(len(y)) % 17 == 0, -1, y)            # DBSCAN-style noise label
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    for name in METRICS + ("silhouette_samples",):
        with pytest.raises(_lib.B200Error):
            getattr(cm, name)(x, y)
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    for name in METRICS:
        got = getattr(cm, name)(x, y)
        assert type(got) is float and got == getattr(metrics, name)(x, y)
    np.testing.assert_array_equal(cm.silhouette_samples(x, y), metrics.silhouette_samples(x, y))


def test_integration_replaces_exactly_the_three_scores(golden):
    """integration.apply(clustering_helper=...) on a stand-in with every name tasks/clustering_helper.py defines
    (recorded from the module by the golden generator)."""
    from audiomuse_ai_b200 import cluster_metrics as cm, integration
    names = [str(n) for n in golden["helper_names"]]
    assert set(METRICS) <= set(names) and "_format_and_score_iteration_result" in names

    def stand_in():
        m = types.ModuleType("tasks.clustering_helper")
        for n in names:
            setattr(m, n, object())
        return m

    ref, before = stand_in(), None
    before = dict(vars(ref))
    old = os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
    try:
        integration.apply(clustering_helper=ref)
        assert os.environ.get("B200_ALLOW_SKLEARN_FALLBACK") == "1"
        changed = {n for n in names if getattr(ref, n) is not before[n]}
        assert changed == set(METRICS)
        assert all(getattr(ref, n) is getattr(cm, n) for n in METRICS)
        os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
        untouched = stand_in()
        snapshot = dict(vars(untouched))
        integration.apply(clustering=None)                       # argument left out: the module is not touched
        assert dict(vars(untouched)) == snapshot and "B200_ALLOW_SKLEARN_FALLBACK" not in os.environ
    finally:
        os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
        if old is not None:
            os.environ["B200_ALLOW_SKLEARN_FALLBACK"] = old


def test_golden_values_equal_sklearn_on_the_recorded_inputs(golden):
    from sklearn import metrics
    for case in ("kmeans", "dbscan"):
        X, labels = golden[f"{case}_X"], golden[f"{case}_labels"]
        assert X.dtype == np.float64 and X.shape == (600, 13)
        for name in METRICS:   # equal up to the summation order of the BLAS build
            np.testing.assert_allclose(getattr(metrics, name)(X, labels), float(golden[f"{case}_{name}"]), rtol=1e-12)
    assert (golden["dbscan_labels"] == -1).any()
