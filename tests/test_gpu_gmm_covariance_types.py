"""The clustering task's 'diag', 'tied' and 'spherical' Gaussian mixtures on the device (audiomuse_ai_b200.
clustering_gpu.gmm_fit(covariance_type=...) / GPUGaussianMixtureAnyCovariance, am_gmm_fit in csrc/gmm.cu) against
scikit-learn's GaussianMixture on float64 input."""
import os
import warnings

import numpy as np
import pytest

from tests.test_gpu_gmm import FULL_SETS, MARGIN_FLOOR, SEED, advanced, blobs, kpp_with_margins, scale

pytestmark = pytest.mark.gpu

TYPES = ("diag", "tied", "spherical")


def sk(X, K, cov, n_init=1, max_iter=100, tol=1e-3, reg_covar=1e-4, random_state=None):
    from sklearn.mixture import GaussianMixture
    m = GaussianMixture(n_components=K, covariance_type=cov, init_params="k-means++", n_init=n_init,
                        max_iter=max_iter, tol=tol, reg_covar=reg_covar, random_state=random_state)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        labels = m.fit_predict(X)
    return m, labels


def assert_params(f, m, X, tol):
    np.testing.assert_allclose(f.means, m.means_, rtol=0, atol=tol * scale(X))
    assert f.covariances.shape == m.covariances_.shape and f.precisions_cholesky.shape == m.precisions_cholesky_.shape
    np.testing.assert_allclose(f.covariances, m.covariances_, rtol=0, atol=tol * scale(m.covariances_))
    np.testing.assert_allclose(f.precisions_cholesky, m.precisions_cholesky_, rtol=0,
                               atol=tol * scale(m.precisions_cholesky_))


@pytest.mark.parametrize("cov", TYPES)
@pytest.mark.parametrize("d", [2, 13, 16, 17, 64, 199, 200, 256])
def test_one_iteration_matches_sklearn(cov, d):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(3 + d, 300 + d, d, 4, spread=1.0)
    K = 5
    f = cg.gmm_fit(X, K, n_init=1, max_iter=1, random_state=5, covariance_type=cov)
    m, labels = sk(X, K, cov, max_iter=1, random_state=5)
    assert f.n_iter == 1
    np.testing.assert_allclose(f.lower_bound, m.lower_bound_, rtol=1e-12, atol=0)
    np.testing.assert_allclose(f.weights, m.weights_, rtol=0, atol=1e-12)
    assert_params(f, m, X, 1e-10)
    np.testing.assert_array_equal(f.labels, labels)


@pytest.mark.parametrize("cov", TYPES)
def test_fixed_trajectory_matches_sklearn(cov):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(4, 900, 20, 6, spread=2.0)
    f = cg.gmm_fit(X, 6, n_init=1, max_iter=10, tol=0.0, random_state=3, covariance_type=cov)
    m, _ = sk(X, 6, cov, max_iter=10, tol=0.0, random_state=3)
    assert f.n_iter == m.n_iter_ == 10 and not f.converged
    np.testing.assert_allclose(f.lower_bounds, m.lower_bounds_, rtol=1e-10, atol=0)


def reference_run(X, K, cov, seed=SEED, n_init=10, tol=1e-3):
    """test_gpu_gmm.reference_run for a covariance type: scikit-learn's GaussianMixture(K, cov, n_init=10,
    random_state=seed) as its inits (init i is an n_init = 1 fit on the generator advanced by i draws_per_init(K)
    doubles), and the smallest margins of every decision: k-means++ draws and candidate potentials, |change| - tol at
    every iteration, and the best init's final bound over the next best init with another solution.
    -> (per init (model, labels), the inits equivalent to the best one, margins)"""
    from sklearn.cluster import kmeans_plusplus
    from audiomuse_ai_b200 import clustering_gpu as cg
    per = cg.draws_per_init(K)
    fits, bounds = [], []
    m = {"draw": np.inf, "potential": np.inf, "tol": np.inf, "best_init": np.inf}
    for i in range(n_init):
        idx, dm, pm = kpp_with_margins(X, K, advanced(seed, i * per))
        np.testing.assert_array_equal(idx, kmeans_plusplus(X, K, random_state=advanced(seed, i * per))[1])
        m["draw"], m["potential"] = min(m["draw"], dm), min(m["potential"], pm)
        model, labels = sk(X, K, cov, tol=tol, random_state=advanced(seed, i * per))
        lb = np.asarray(model.lower_bounds_)
        if len(lb) > 1:
            m["tol"] = min(m["tol"], float(np.min(np.abs(np.abs(np.diff(lb)) - tol) / np.abs(lb[1:]))))
        fits.append((model, labels))
        bounds.append(model.lower_bound_)
    best, top = 0, -np.inf
    for i, b in enumerate(bounds):
        if b > top or top == -np.inf:
            best, top = i, b

    def same_partition(a, b):
        return len(set(zip(a.tolist(), b.tolist()))) == len(set(a.tolist())) == len(set(b.tolist()))

    same = [i for i in range(n_init) if same_partition(fits[i][1], fits[best][1])
            and abs(bounds[i] - top) <= 1e-12 * abs(top)]
    rest = [b for i, b in enumerate(bounds) if i not in same]
    if rest:
        m["best_init"] = (top - max(rest)) / abs(top)
    return fits, same, m


@pytest.fixture(scope="module")
def full_fits():
    cache = {}

    def get(cov, name):
        if (cov, name) not in cache:
            _, N, d, K, spread, dup = next(s for s in FULL_SETS if s[0] == name)
            X = blobs(sum(map(ord, name)), N, d, K, spread=spread, dup=dup)
            cache[cov, name] = (X, K) + reference_run(X, K, cov)
        return cache[cov, name]
    return get


# 'tied' starts every init from X^T X over all rows with one-hot responsibilities, and on these two sets its inits stop
# after 3 iterations at different partitions whose final bounds lie within 1.2e-9 relative of each other: the
# best-init margin is 2.9e-10 (d13_k2) and 1.8e-10 (overlap), below MARGIN_FLOOR, and it stayed below the floor on
# d13_k2 for every random_state from 21 to 39.  There the device may pick any of those inits; its outputs are compared
# with scikit-learn's fit of the init it picked, and its bound must be within 2e-9 relative of the best.  Any other set
# below the floor fails.
BELOW_FLOOR = {("tied", "d13_k2"), ("tied", "overlap")}


@pytest.mark.parametrize("cov", TYPES)
@pytest.mark.parametrize("name", [s[0] for s in FULL_SETS])
def test_full_fit_with_the_reference_settings(full_fits, cov, name):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X, K, fits, same, margins = full_fits(cov, name)
    print(cov, name, {k: f"{v:.3g}" for k, v in margins.items()})
    near_tie = (cov, name) in BELOW_FLOOR
    assert min(margins.values()) > MARGIN_FLOOR or (near_tie and min(margins["draw"], margins["potential"],
                                                                     margins["tol"]) > MARGIN_FLOOR), margins
    f = cg.gmm_fit(X, K, n_init=10, random_state=SEED, covariance_type=cov)
    top = max(model.lower_bound_ for model, _ in fits)
    if near_tie:
        assert abs(f.lower_bound - top) <= 2e-9 * abs(top)
    else:
        assert f.best_init in same
    m, labels = fits[f.best_init]
    assert (f.n_iter, f.converged) == (m.n_iter_, m.converged_)
    np.testing.assert_array_equal(f.labels, labels)
    np.testing.assert_allclose(f.lower_bound, m.lower_bound_, rtol=1e-9, atol=0)
    np.testing.assert_allclose(f.weights, m.weights_, rtol=0, atol=1e-8)
    assert_params(f, m, X, 1e-8)


@pytest.mark.parametrize("cov", TYPES)
def test_task_shape_fixed_iterations(cov):
    from audiomuse_ai_b200 import clustering_gpu as cg
    rng = np.random.default_rng(9)
    X = rng.standard_normal((20000, 200)) + np.repeat(rng.standard_normal((60, 200)), 334, 0)[:20000]
    X = (X - X.mean(0)) / X.std(0)
    f = cg.gmm_fit(X, 60, n_init=1, max_iter=3, tol=0.0, random_state=1, covariance_type=cov)
    m, labels = sk(X, 60, cov, max_iter=3, tol=0.0, random_state=1)
    np.testing.assert_allclose(f.lower_bounds, m.lower_bounds_, rtol=1e-10, atol=0)
    assert_params(f, m, X, 1e-9)
    diff = f.labels != labels
    if diff.any():
        lr = np.sort(m._estimate_weighted_log_prob(X)[diff], axis=1)
        gap = lr[:, -1] - lr[:, -2]
        print(f"{int(diff.sum())} labels differ, top-two gaps up to {gap.max():.3g}")
        assert (gap < 1e-8).all()


def _ill_defined_rows(cov):
    """rows on which scikit-learn's fit with reg_covar = 0 raises: a zero column makes every diag and tied covariance
    singular; for spherical, most rows are zero, so a zero seed row gives a component of variance 0"""
    rng = np.random.default_rng(6)
    X = rng.standard_normal((200, 5))
    if cov == "spherical":
        X[:150] = 0.0
    else:
        X[:, 2] = 0.0
    return X


@pytest.mark.parametrize("cov", TYPES)
def test_ill_defined_raises_like_sklearn(cov):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = _ill_defined_rows(cov)
    with pytest.raises(ValueError, match="ill-defined empirical covariance"):
        sk(X, 3, cov, reg_covar=0.0, random_state=0)
    with pytest.raises(ValueError, match="ill-defined empirical covariance"):
        cg.GPUGaussianMixtureAnyCovariance(3, covariance_type=cov, reg_covar=0.0, random_state=0).fit_predict(X)


@pytest.mark.parametrize("cov", TYPES)
def test_float32_input_returns_float32_and_sklearn_labels(cov):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(5, 600, 12, 4, spread=0.3).astype(np.float32)
    g = cg.GPUGaussianMixtureAnyCovariance(4, covariance_type=cov, random_state=8)
    got = g.fit_predict(X)
    m, want = sk(X.astype(np.float64), 4, cov, n_init=10, random_state=8)
    assert g.using_gpu and g.means_.dtype == np.float32 and g.covariances_.dtype == np.float32
    assert g.precisions_cholesky_.dtype == np.float32
    assert g.covariances_.shape == m.covariances_.shape and g.precisions_cholesky_.shape == m.precisions_cholesky_.shape
    assert got.dtype == np.int64
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("cov", TYPES)
def test_two_calls_are_bit_identical(cov):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(7, 1000, 30, 8, spread=0.5)
    a = cg.gmm_fit(X, 8, n_init=10, random_state=4, covariance_type=cov)
    b = cg.gmm_fit(X, 8, n_init=10, random_state=4, covariance_type=cov)
    for n in ("weights", "means", "covariances", "precisions_cholesky", "labels"):
        np.testing.assert_array_equal(getattr(a, n), getattr(b, n))
    assert a.lower_bounds == b.lower_bounds


@pytest.mark.parametrize("cov", TYPES)
def test_global_seed_fit_replays_the_reference_task(golden_dir, monkeypatch, cov):
    """The reference's _apply_clustering_model after np.random.seed(s) with GMM_COVARIANCE_TYPE = cov
    (tests/golden/gmm_types_golden.npz): get_clustering_model with the opt-in class installed, as
    integration.apply(gaussian_mixture=..., gmm_all_covariance_types=True) installs it in the reference's module,
    gives the recorded labels and centres (means_), and leaves numpy's global generator where scikit-learn's fit
    leaves it."""
    from audiomuse_ai_b200 import clustering_gpu as cg
    g = np.load(os.path.join(golden_dir, "gmm_types_golden.npz"))
    X, seed, K = g["X"], int(g[f"{cov}/seed"]), int(g["n_components"])
    monkeypatch.setattr(cg, "GMM_COVARIANCE_TYPE", cov)
    monkeypatch.setattr(cg, "GPUGaussianMixture", cg.GPUGaussianMixtureAnyCovariance)
    np.random.seed(seed)
    model = cg.get_clustering_model("gmm", {"n_components": K}, use_gpu=True)
    labels = model.fit_predict(X)
    after = np.random.get_state()
    assert model.using_gpu and model.covariance_type == cov
    np.testing.assert_array_equal(labels, g[f"{cov}/labels"])
    centers = np.stack([model.means_[c] for c in range(len(g[f"{cov}/centers"]))])
    np.testing.assert_allclose(centers, g[f"{cov}/centers"], rtol=0, atol=1e-8 * scale(X))
    np.random.seed(seed)
    sk(X, K, cov, n_init=10)
    want = np.random.get_state()
    assert after[0] == want[0] and np.array_equal(after[1], want[1]) and after[2:] == want[2:]
