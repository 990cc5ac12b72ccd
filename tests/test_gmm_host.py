"""Host-side contracts of GPUGaussianMixture / gmm_fit (audiomuse_ai_b200.clustering_gpu) and of their integration
point, tasks/clustering_gpu.py.  No GPU compute is issued here."""
import ast
import os
import types
import warnings

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
    return np.load(os.path.join(golden_dir, "gmm_golden.npz"))


def _rows(n=120, d=4, seed=2):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.standard_normal((n // 2, d)) + 5, rng.standard_normal((n - n // 2, d)) - 5])


def test_validation_raises_value_error_before_the_library(monkeypatch):
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg

    def no_library():
        raise AssertionError("validation must not reach the library")

    monkeypatch.setattr(_lib, "load", no_library)
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")      # validation errors are not GPU failures
    x = _rows()
    bad = [
        (dict(n_components=2), x[:, 0]),
        (dict(n_components=2), x[None]),
        (dict(n_components=2), x[:1]),
        (dict(n_components=len(x) + 1), x),
        (dict(n_components=0), x),
        (dict(n_components=2, n_init=0), x),
        (dict(n_components=2, reg_covar=-1e-3), x),
        (dict(n_components=2, covariance_type="diag"), x),
        (dict(n_components=2, covariance_type="tied"), x),
        (dict(n_components=2, covariance_type="spherical"), x),
        (dict(n_components=2, init_params="kmeans"), x),
        (dict(n_components=2, init_params="random"), x),
        (dict(n_components=513), np.zeros((600, 2))),
        (dict(n_components=2), np.zeros((10, 257))),
        (dict(n_components=512, n_init=128), np.zeros((600, 2))),
    ]
    for kw, data in bad:
        with pytest.raises(ValueError):
            cg.GPUGaussianMixture(**kw).fit_predict(data)
    with pytest.raises(ValueError, match="Expected n_samples >= n_components"):
        cg.GPUGaussianMixture(n_components=len(x) + 1).fit_predict(x)
    for v in (np.nan, np.inf, -np.inf):
        b = x.copy()
        b[3, 1] = v
        with pytest.raises(ValueError, match="NaN or infinity"):
            cg.GPUGaussianMixture(n_components=2).fit_predict(b)


@pytest.mark.parametrize("K", [1, 2, 40, 100])
@pytest.mark.parametrize("n_init", [1, 10])
def test_draws_leave_the_generator_where_sklearn_leaves_it(K, n_init):
    from sklearn.mixture import GaussianMixture
    from audiomuse_ai_b200.artist_gmm import kpp_draws
    X = np.random.default_rng(K).standard_normal((max(K, 2) * 3, 2))

    def sk_fit(rs):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            GaussianMixture(K, covariance_type="full", n_init=n_init, max_iter=1, reg_covar=1e-2,
                            init_params="k-means++", random_state=rs).fit(X)

    a, b = np.random.RandomState(5), np.random.RandomState(5)
    sk_fit(a)
    kpp_draws(b, K, n_init)
    assert all(np.array_equal(u, v) for u, v in zip(a.get_state(), b.get_state()))
    np.random.seed(9)
    sk_fit(None)
    want = np.random.get_state()
    np.random.seed(9)
    kpp_draws(None, K, n_init)
    assert all(np.array_equal(u, v) for u, v in zip(want, np.random.get_state()))


def test_factory_and_integration(golden):
    from sklearn.mixture import GaussianMixture
    from audiomuse_ai_b200 import clustering_gpu as cg, integration
    # the reference's factory (recorded by the golden generator) and ours hand out the same class with the same arguments
    want = {str(n): ast.literal_eval(str(v)) for n, v in zip(golden["ctor_names"], golden["ctor_values"])}
    params = {"n_components": int(golden["n_components"])}
    assert want["n_components"] == params["n_components"]
    gpu = cg.get_clustering_model("gmm", params, use_gpu=True)
    assert type(gpu).__name__ == str(golden["class_name"]) == "GPUGaussianMixture"
    assert type(gpu) is cg.GPUGaussianMixture and {n: getattr(gpu, n) for n in want} == want
    assert not hasattr(gpu, "predict")
    cpu = cg.get_clustering_model("gmm", params, use_gpu=False)
    assert type(cpu) is GaussianMixture and {n: cpu.get_params()[n] for n in want} == want
    ref_cg = types.ModuleType("tasks.clustering_gpu")
    for n in ("GPUKMeans", "GPUDBSCAN", "GPUPCA", "GPUSpectralClustering", "GPUGaussianMixture", "check_gpu_available"):
        setattr(ref_cg, n, object())
    before = ref_cg.GPUGaussianMixture
    old = os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
    try:
        integration.apply(clustering=ref_cg, allow_sklearn_fallback=False)
        assert ref_cg.GPUGaussianMixture is before
        assert "B200_ALLOW_SKLEARN_FALLBACK" not in os.environ
        integration.apply(gaussian_mixture=ref_cg, allow_sklearn_fallback=False)
        assert ref_cg.GPUGaussianMixture is cg.GPUGaussianMixture
        assert "B200_ALLOW_SKLEARN_FALLBACK" not in os.environ
        integration.apply(gaussian_mixture=ref_cg)
        assert os.environ.get("B200_ALLOW_SKLEARN_FALLBACK") == "1"
    finally:
        os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
        if old is not None:
            os.environ["B200_ALLOW_SKLEARN_FALLBACK"] = old


@pytest.mark.skipif(not _no_gpu(), reason="exercises the no-device failure path")
def test_fallback_contract_both_settings(monkeypatch):
    from sklearn.mixture import GaussianMixture
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    x = _rows()
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    m = cg.GPUGaussianMixture(n_components=2, random_state=5)
    with pytest.raises(_lib.B200Error):
        m.fit_predict(x)
    assert m.labels_ is None and m.using_gpu is False
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    np.random.seed(3)
    got = cg.GPUGaussianMixture(n_components=2).fit_predict(x)
    np.random.seed(3)
    ref = GaussianMixture(n_components=2, covariance_type="full", init_params="k-means++", n_init=10,
                          reg_covar=1e-4).fit_predict(x)
    np.testing.assert_array_equal(got, ref)
    got = m.fit_predict(x)
    np.testing.assert_array_equal(got, GaussianMixture(2, n_init=10, reg_covar=1e-4, random_state=5).fit_predict(x))
    assert m.using_gpu is False and m.means_ is not None


def test_golden_labels_and_centres_are_sklearn_after_the_recorded_seed(golden):
    from sklearn.mixture import GaussianMixture
    X, labels, centers = golden["X"], golden["labels"], golden["centers"]
    assert X.dtype == np.float64 and X.shape == (600, 13)
    want = {str(n): ast.literal_eval(str(v)) for n, v in zip(golden["ctor_names"], golden["ctor_values"])}
    np.random.seed(int(golden["seed"]))
    m = GaussianMixture(**want)
    np.testing.assert_array_equal(m.fit_predict(X), labels)
    np.testing.assert_array_equal(m.means_, centers)
