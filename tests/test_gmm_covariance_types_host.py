"""Host-side contracts of GPUGaussianMixtureAnyCovariance and gmm_fit(covariance_type=...) (audiomuse_ai_b200.
clustering_gpu) for the 'diag', 'tied' and 'spherical' mixtures, and of the gmm_all_covariance_types opt-in of
integration.apply.  No GPU compute is issued here."""
import ast
import os
import types
import warnings

import numpy as np
import pytest

TYPES = ("full", "tied", "diag", "spherical")


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "gmm_types_golden.npz"))


def _rows(n=120, d=4, seed=2):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.standard_normal((n // 2, d)) + 5, rng.standard_normal((n - n // 2, d)) - 5])


@pytest.mark.parametrize("cov", TYPES)
def test_validation_raises_value_error_before_the_library(monkeypatch, cov):
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
        (dict(n_components=2, init_params="kmeans"), x),
        (dict(n_components=2, init_params="random"), x),
        (dict(n_components=513), np.zeros((600, 2))),
        (dict(n_components=2), np.zeros((10, 257))),
        (dict(n_components=512, n_init=128), np.zeros((600, 2))),
    ]
    for kw, data in bad:
        with pytest.raises(ValueError):
            cg.GPUGaussianMixtureAnyCovariance(covariance_type=cov, **kw).fit_predict(data)
    with pytest.raises(ValueError, match="Expected n_samples >= n_components"):
        cg.GPUGaussianMixtureAnyCovariance(n_components=len(x) + 1, covariance_type=cov).fit_predict(x)
    for v in (np.nan, np.inf, -np.inf):
        b = x.copy()
        b[3, 1] = v
        with pytest.raises(ValueError, match="NaN or infinity"):
            cg.GPUGaussianMixtureAnyCovariance(n_components=2, covariance_type=cov).fit_predict(b)
    with pytest.raises(ValueError):
        cg.GPUGaussianMixtureAnyCovariance(n_components=2, covariance_type="banded").fit_predict(x)
    with pytest.raises(ValueError):
        cg.gmm_fit(x, 2, covariance_type="banded")
    with pytest.raises(ValueError):
        cg.gmm_fit(x, 2, covariance_type=cov, reg_covar=-1.0)


def test_the_default_class_still_fits_full_only():
    from audiomuse_ai_b200 import clustering_gpu as cg
    assert cg.GPUGaussianMixture.DEVICE_COVARIANCE_TYPES == ("full",)
    assert set(cg.GPUGaussianMixtureAnyCovariance.DEVICE_COVARIANCE_TYPES) == set(TYPES)
    assert issubclass(cg.GPUGaussianMixtureAnyCovariance, cg.GPUGaussianMixture)


@pytest.mark.parametrize("cov", ("tied", "diag", "spherical"))
@pytest.mark.parametrize("K", [1, 2, 40, 100])
def test_draws_leave_the_generator_where_sklearn_leaves_it(cov, K):
    from sklearn.mixture import GaussianMixture
    from audiomuse_ai_b200.artist_gmm import kpp_draws
    X = np.random.default_rng(K).standard_normal((max(K, 2) * 3, 2))

    def sk_fit(rs):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            GaussianMixture(K, covariance_type=cov, n_init=10, max_iter=1, reg_covar=1e-2,
                            init_params="k-means++", random_state=rs).fit(X)

    a, b = np.random.RandomState(5), np.random.RandomState(5)
    sk_fit(a)
    kpp_draws(b, K, 10)
    assert all(np.array_equal(u, v) for u, v in zip(a.get_state(), b.get_state()))
    np.random.seed(9)
    sk_fit(None)
    want = np.random.get_state()
    np.random.seed(9)
    kpp_draws(None, K, 10)
    assert all(np.array_equal(u, v) for u, v in zip(want, np.random.get_state()))


def _ref_module():
    ref_cg = types.ModuleType("tasks.clustering_gpu")
    for n in ("GPUKMeans", "GPUDBSCAN", "GPUPCA", "GPUSpectralClustering", "GPUGaussianMixture", "check_gpu_available"):
        setattr(ref_cg, n, object())
    return ref_cg


def test_apply_installs_the_class_the_flag_selects():
    from audiomuse_ai_b200 import clustering_gpu as cg, integration
    old = os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
    try:
        ref_cg = _ref_module()
        integration.apply(gaussian_mixture=ref_cg, gmm_all_covariance_types=True, allow_sklearn_fallback=False)
        assert ref_cg.GPUGaussianMixture is cg.GPUGaussianMixtureAnyCovariance
        ref_cg = _ref_module()
        integration.apply(gaussian_mixture=ref_cg, allow_sklearn_fallback=False)
        assert ref_cg.GPUGaussianMixture is cg.GPUGaussianMixture
        ref_cg = _ref_module()
        before = ref_cg.GPUGaussianMixture
        with pytest.raises(ValueError, match="gaussian_mixture="):
            integration.apply(gmm_all_covariance_types=True, allow_sklearn_fallback=False)
        with pytest.raises(ValueError, match="gaussian_mixture="):
            integration.apply(clustering=ref_cg, gmm_all_covariance_types=True, allow_sklearn_fallback=False)
        assert ref_cg.GPUGaussianMixture is before and ref_cg.GPUKMeans is not cg.GPUKMeans   # nothing was patched
        assert "B200_ALLOW_SKLEARN_FALLBACK" not in os.environ
    finally:
        os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
        if old is not None:
            os.environ["B200_ALLOW_SKLEARN_FALLBACK"] = old


@pytest.mark.skipif(not _no_gpu(), reason="exercises the no-device failure path")
@pytest.mark.parametrize("cov", ("tied", "diag", "spherical"))
def test_fallback_contract_both_settings(monkeypatch, cov):
    from sklearn.mixture import GaussianMixture
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    x = _rows()
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    m = cg.GPUGaussianMixtureAnyCovariance(n_components=2, covariance_type=cov, random_state=5)
    with pytest.raises(_lib.B200Error):
        m.fit_predict(x)
    assert m.labels_ is None and m.using_gpu is False
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    np.random.seed(3)
    g = cg.GPUGaussianMixtureAnyCovariance(n_components=2, covariance_type=cov)
    got = g.fit_predict(x)
    after = np.random.get_state()
    np.random.seed(3)
    ref = GaussianMixture(n_components=2, covariance_type=cov, init_params="k-means++", n_init=10,
                          reg_covar=1e-4)
    np.testing.assert_array_equal(got, ref.fit_predict(x))
    want = np.random.get_state()
    assert after[0] == want[0] and np.array_equal(after[1], want[1]) and after[2:] == want[2:]
    assert g.model.covariance_type == cov and g.covariances_.shape == ref.covariances_.shape
    np.testing.assert_array_equal(g.covariances_, ref.covariances_)
    got = m.fit_predict(x)
    want = GaussianMixture(2, covariance_type=cov, init_params="k-means++", n_init=10, reg_covar=1e-4,
                           random_state=5).fit_predict(x)
    np.testing.assert_array_equal(got, want)
    assert m.using_gpu is False and m.means_ is not None


@pytest.mark.parametrize("cov", ("diag", "tied", "spherical"))
def test_golden_labels_and_centres_are_sklearn_after_the_recorded_seed(golden, cov):
    from sklearn.mixture import GaussianMixture
    X, labels, centers = golden["X"], golden[f"{cov}/labels"], golden[f"{cov}/centers"]
    assert X.dtype == np.float64 and X.shape == (600, 13)
    assert str(golden[f"{cov}/class_name"]) == "GPUGaussianMixture"
    want = {str(n): ast.literal_eval(str(v)) for n, v in zip(golden[f"{cov}/ctor_names"], golden[f"{cov}/ctor_values"])}
    assert want["covariance_type"] == cov and want["random_state"] is None
    np.random.seed(int(golden[f"{cov}/seed"]))
    m = GaussianMixture(**want)
    np.testing.assert_array_equal(m.fit_predict(X), labels)
    np.testing.assert_array_equal(m.means_, centers)


@pytest.mark.parametrize("cov", ("diag", "tied", "spherical"))
def test_factory_hands_out_the_recorded_arguments(golden, monkeypatch, cov):
    from audiomuse_ai_b200 import clustering_gpu as cg
    want = {str(n): ast.literal_eval(str(v)) for n, v in zip(golden[f"{cov}/ctor_names"], golden[f"{cov}/ctor_values"])}
    monkeypatch.setattr(cg, "GMM_COVARIANCE_TYPE", cov)
    monkeypatch.setattr(cg, "GPUGaussianMixture", cg.GPUGaussianMixtureAnyCovariance)
    gpu = cg.get_clustering_model("gmm", {"n_components": int(golden["n_components"])}, use_gpu=True)
    assert type(gpu) is cg.GPUGaussianMixtureAnyCovariance and {n: getattr(gpu, n) for n in want} == want
