"""Host-side contracts of GPUSpectralClustering / spectral_embedding (audiomuse_ai_b200.clustering_gpu) and of their
integration point, tasks/clustering_gpu.py.  No GPU compute is issued here."""
import ast
import os
import types

import numpy as np
import pytest


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "spectral_golden.npz"))


def _blobs(n=90, seed=3):
    rng = np.random.default_rng(seed)
    third = n // 3
    return np.concatenate([rng.standard_normal((third, 4)) + 6, rng.standard_normal((third, 4)) - 6,
                           rng.standard_normal((n - 2 * third, 4))])


def test_validation_raises_value_error_before_the_library(monkeypatch):
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg

    def no_library():
        raise AssertionError("validation must not reach the library")

    monkeypatch.setattr(_lib, "load", no_library)
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")      # validation errors are not GPU failures
    x = _blobs()
    N = len(x)
    bad_fits = [
        (dict(n_clusters=3), x[:, 0]),                            # 1-D
        (dict(n_clusters=3), x[None]),                            # 3-D
        (dict(n_clusters=1), x),
        (dict(n_clusters=N), x),
        (dict(n_clusters=3, n_neighbors=1), x),
        (dict(n_clusters=3, n_neighbors=N + 1), x),
        (dict(n_clusters=3, affinity="rbf"), x),
        (dict(n_clusters=3, affinity="precomputed"), x),
        (dict(n_clusters=3, assign_labels="discretize"), x),
        (dict(n_clusters=3, assign_labels="cluster_qr"), x),
    ]
    for kw, data in bad_fits:
        with pytest.raises(ValueError):
            cg.GPUSpectralClustering(**kw).fit_predict(data)
    for v in (np.nan, np.inf, -np.inf, 1e39):                    # 1e39 overflows float32
        bad = x.copy()
        bad[7, 2] = v
        with pytest.raises(ValueError, match="NaN or infinity"):
            cg.GPUSpectralClustering(n_clusters=3).fit_predict(bad)
    with pytest.raises(ValueError):
        cg.spectral_embedding(x, 0)
    with pytest.raises(ValueError):
        cg.spectral_embedding(x, N + 1)
    with pytest.raises(ValueError):
        cg.spectral_embedding(x, 3, n_neighbors=1)


@pytest.mark.skipif(not _no_gpu(), reason="exercises the no-device failure path")
def test_fallback_contract_both_settings(monkeypatch):
    """Loud by default; scikit-learn's SpectralClustering with the same arguments under B200_ALLOW_SKLEARN_FALLBACK=1
    (the GPUKMeans / GPUDBSCAN contract)."""
    from sklearn.cluster import SpectralClustering
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    x = _blobs()
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    m = cg.GPUSpectralClustering(n_clusters=3, n_neighbors=8, random_state=5)
    with pytest.raises(_lib.B200Error):
        m.fit_predict(x)
    assert m.labels_ is None and m.using_gpu is False
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    got = m.fit_predict(x)
    ref = SpectralClustering(n_clusters=3, affinity="nearest_neighbors", n_neighbors=8, random_state=5,
                             n_init=10).fit_predict(x)
    np.testing.assert_array_equal(got, ref)
    assert m.labels_ is got and m.using_gpu is False
    assert not hasattr(m, "cluster_centers_") and not hasattr(m, "means_")


def test_integration_installs_the_class_and_the_factory_matches_the_reference(golden):
    from sklearn.cluster import SpectralClustering
    from audiomuse_ai_b200 import clustering_gpu as cg, integration
    ref_cg = types.ModuleType("tasks.clustering_gpu")
    for n in ("GPUKMeans", "GPUDBSCAN", "GPUPCA", "GPUSpectralClustering", "GPUGaussianMixture", "check_gpu_available",
              "get_clustering_model", "get_pca_model"):
        setattr(ref_cg, n, object())
    before = dict(vars(ref_cg))
    old = os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
    try:
        integration.apply(clustering=ref_cg, allow_sklearn_fallback=False)
    finally:
        if old is not None:
            os.environ["B200_ALLOW_SKLEARN_FALLBACK"] = old
    assert ref_cg.GPUSpectralClustering is cg.GPUSpectralClustering
    assert ref_cg.GPUGaussianMixture is before["GPUGaussianMixture"]       # GMM stays with the reference
    # the reference's factory (recorded by the golden generator) and ours hand out the same class with the same arguments
    params = {"n_clusters": int(golden["n_clusters"]), "random_state": int(golden["random_state"])}
    want = {str(n): ast.literal_eval(str(v)) for n, v in zip(golden["ctor_names"], golden["ctor_values"])}
    gpu = cg.get_clustering_model("spectral", params, use_gpu=True)
    assert type(gpu).__name__ == str(golden["class_name"]) == "GPUSpectralClustering"
    assert {n: getattr(gpu, n) for n in want} == want
    cpu = cg.get_clustering_model("spectral", params, use_gpu=False)
    assert type(cpu) is SpectralClustering and {n: cpu.get_params()[n] for n in want} == want
    assert cg.get_clustering_model("spectral", {**params, "n_neighbors": 7}, use_gpu=True).n_neighbors == 7


def test_golden_labels_and_centres_are_sklearn_on_the_recorded_inputs(golden):
    from sklearn.cluster import SpectralClustering
    X, labels, centers = golden["X"], golden["labels"], golden["centers"]
    assert X.dtype == np.float64 and X.shape == (600, 13)
    want = {str(n): ast.literal_eval(str(v)) for n, v in zip(golden["ctor_names"], golden["ctor_values"])}
    ref = SpectralClustering(**want).fit_predict(X)
    np.testing.assert_array_equal(ref, labels)
    # the reference's centres of a model without cluster_centers_ / means_: per-label means of the data
    np.testing.assert_allclose(np.stack([X[labels == c].mean(0) for c in range(len(centers))]), centers, rtol=0,
                               atol=1e-12)
