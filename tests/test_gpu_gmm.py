"""The clustering task's full-covariance Gaussian mixture on the device (audiomuse_ai_b200.clustering_gpu.gmm_fit /
GPUGaussianMixture, csrc/gmm.cu) against scikit-learn's GaussianMixture on float64 input."""
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def blobs(seed, n, d, groups, spread=0.3, dup=0):
    rng = np.random.default_rng(seed)
    c = 3.0 * rng.standard_normal((groups, d))
    X = c[np.arange(n) % groups] + spread * rng.standard_normal((n, d))
    if dup:
        X[:dup] = X[0]
    return X


def sk(X, K, n_init=1, max_iter=100, tol=1e-3, reg_covar=1e-4, random_state=None):
    from sklearn.mixture import GaussianMixture
    m = GaussianMixture(n_components=K, covariance_type="full", init_params="k-means++", n_init=n_init,
                        max_iter=max_iter, tol=tol, reg_covar=reg_covar, random_state=random_state)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        labels = m.fit_predict(X)
    return m, labels


def advanced(seed, count):
    rs = np.random.RandomState(seed)
    rs.random_sample(count)
    return rs


def scale(a):
    return max(1.0, float(np.abs(a).max()))


def test_kpp_indices_equal_sklearn_for_every_init():
    from sklearn.cluster import kmeans_plusplus
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(1, 700, 13, 9, spread=1.0)
    for K in (1, 2, 12, 40):
        f = cg.gmm_fit(X, K, n_init=4, max_iter=1, random_state=np.random.RandomState(7), intermediates=True)
        per = cg.draws_per_init(K)
        for i in range(4):
            _, want = kmeans_plusplus(X, K, random_state=advanced(7, i * per))
            np.testing.assert_array_equal(f.kpp[i], want, err_msg=f"K={K} init {i}")


def test_init_i_alone_is_sklearn_on_the_advanced_generator():
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(2, 500, 8, 5, spread=1.5)
    K = 6
    f = cg.gmm_fit(X, K, n_init=3, max_iter=4, tol=0.0, random_state=11, intermediates=True)
    per = cg.draws_per_init(K)
    for i in range(3):
        m, _ = sk(X, K, max_iter=4, tol=0.0, random_state=advanced(11, i * per))
        np.testing.assert_allclose(f.init_lower_bounds[i, :4], m.lower_bounds_, rtol=1e-10, atol=0)


@pytest.mark.parametrize("d", [2, 13, 16, 17, 64, 199, 200, 256])
def test_one_iteration_matches_sklearn(d):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(3 + d, 300 + d, d, 4, spread=1.0)
    K = 5
    f = cg.gmm_fit(X, K, n_init=1, max_iter=1, random_state=5)
    m, labels = sk(X, K, max_iter=1, random_state=5)
    assert f.n_iter == 1
    np.testing.assert_allclose(f.lower_bound, m.lower_bound_, rtol=1e-12, atol=0)
    np.testing.assert_allclose(f.weights, m.weights_, rtol=0, atol=1e-12)
    np.testing.assert_allclose(f.means, m.means_, rtol=0, atol=1e-10 * scale(X))
    np.testing.assert_allclose(f.covariances, m.covariances_, rtol=0, atol=1e-10 * scale(m.covariances_))
    np.testing.assert_allclose(f.precisions_cholesky, m.precisions_cholesky_, rtol=0,
                               atol=1e-9 * scale(m.precisions_cholesky_))
    np.testing.assert_array_equal(f.labels, labels)


def test_fixed_trajectory_matches_sklearn():
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(4, 900, 20, 6, spread=2.0)
    f = cg.gmm_fit(X, 6, n_init=1, max_iter=10, tol=0.0, random_state=3)
    m, _ = sk(X, 6, max_iter=10, tol=0.0, random_state=3)
    assert f.n_iter == m.n_iter_ == 10 and not f.converged
    np.testing.assert_allclose(f.lower_bounds, m.lower_bounds_, rtol=1e-10, atol=0)


MARGIN_FLOOR = 1e-9   # every discrete decision of the full-fit sets is at least this far (relative) from flipping
SEED = 21

FULL_SETS = [
    # name, N, d, K, spread, dup
    ("ragged_63", 63 * 3 + 1, 5, 3, 0.3, 0),
    ("ragged_129", 129, 7, 4, 0.3, 0),
    ("d2", 400, 2, 4, 0.2, 0),
    ("d13_k2", 300, 13, 2, 0.3, 0),
    ("d16", 500, 16, 5, 0.3, 0),
    ("d17", 500, 17, 5, 0.3, 0),
    ("d64", 600, 64, 6, 0.3, 0),
    ("d199", 800, 199, 4, 0.3, 0),
    ("d200", 800, 200, 4, 0.3, 0),
    ("d256", 800, 256, 3, 0.3, 0),
    ("k1", 200, 6, 1, 0.3, 0),
    ("k40", 2000, 10, 40, 0.05, 0),
    ("k100", 3000, 6, 100, 0.05, 0),
    ("n_eq_k", 2, 3, 2, 0.3, 0),
    ("overlap", 1500, 8, 5, 2.5, 0),
    ("dups", 300, 4, 3, 0.3, 60),
]


def _sq_dist(X, xsq, rows):
    """scikit-learn's _euclidean_distances(X[rows], X, Y_norm_squared=xsq, squared=True)"""
    from sklearn.utils.extmath import row_norms
    C = X[rows]
    d = -2.0 * (C @ X.T)
    d += row_norms(C, squared=True)[:, None]
    d += xsq[None, :]
    return np.maximum(d, 0.0)


def kpp_with_margins(X, K, rs):
    """scikit-learn's _kmeans_plusplus (unit weights) restated step by step, with its decision margins: each scaled
    draw's distance to the nearest cumsum boundary over the potential, and the gap between the best and the next
    candidate potential over the best (candidates that are the same vector tie exactly on the device too)"""
    from sklearn.utils.extmath import row_norms
    N = len(X)
    L = 2 + int(np.log(K))
    xsq = row_norms(X, squared=True)
    idx = [int(rs.choice(N, p=np.full(N, 1.0 / N)))]
    closest = _sq_dist(X, xsq, idx[:1])[0]
    pot = closest.sum()
    draw_m, pot_m = [np.inf], [np.inf]
    for _ in range(1, K):
        rv = rs.uniform(size=L) * pot
        cs = np.cumsum(closest)
        cand = np.searchsorted(cs, rv)
        for r, c in zip(rv, cand):
            if c < N:
                lo = cs[c - 1] if c > 0 else 0.0
                draw_m.append(min(r - lo, cs[c] - r) / pot)
        cand = np.minimum(cand, N - 1)
        dc = np.minimum(closest, _sq_dist(X, xsq, cand))
        pots = dc.sum(1)
        b = int(np.argmin(pots))
        others = [p for j, p in enumerate(pots) if not np.array_equal(X[cand[j]], X[cand[b]])]
        if others:
            pot_m.append((min(others) - pots[b]) / pots[b])
        idx.append(int(cand[b]))
        pot, closest = pots[b], dc[b]
    return np.array(idx), min(draw_m), min(pot_m)


def reference_run(X, K, seed=SEED, n_init=10, tol=1e-3):
    """scikit-learn's GaussianMixture(K, n_init=10, random_state=seed) as its inits: init i is an n_init = 1 fit on the
    generator advanced by i draws_per_init(K) doubles, and the smallest margins of every decision: k-means++ draws and candidate potentials, |change| - tol at every
    iteration, and the best init's final bound over the next best.  -> (per init (model, labels), the inits
    equivalent to the best one, margins)"""
    from sklearn.cluster import kmeans_plusplus
    from audiomuse_ai_b200 import clustering_gpu as cg
    per = cg.draws_per_init(K)
    fits, bounds = [], []
    m = {"draw": np.inf, "potential": np.inf, "tol": np.inf, "best_init": np.inf}
    for i in range(n_init):
        idx, dm, pm = kpp_with_margins(X, K, advanced(seed, i * per))
        np.testing.assert_array_equal(idx, kmeans_plusplus(X, K, random_state=advanced(seed, i * per))[1])
        m["draw"], m["potential"] = min(m["draw"], dm), min(m["potential"], pm)
        model, labels = sk(X, K, tol=tol, random_state=advanced(seed, i * per))
        lb = np.asarray(model.lower_bounds_)
        if len(lb) > 1:
            m["tol"] = min(m["tol"], float(np.min(np.abs(np.abs(np.diff(lb)) - tol) / np.abs(lb[1:]))))
        fits.append((model, labels))
        bounds.append(model.lower_bound_)
    best, top = 0, -np.inf
    for i, b in enumerate(bounds):
        if b > top or top == -np.inf:
            best, top = i, b
    # inits that reach the best init's solution (the same partition of the rows, possibly numbered differently, and
    # its bound to 1e-12) are interchangeable: the device may pick any of them, and its outputs are then that init's.
    # The margin is to the best init with another solution.
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
    out = {}
    for name, N, d, K, spread, dup in FULL_SETS:
        X = blobs(sum(map(ord, name)), N, d, K, spread=spread, dup=dup)
        out[name] = (X, K) + reference_run(X, K)
    return out


@pytest.mark.parametrize("name", [s[0] for s in FULL_SETS])
def test_full_fit_with_the_reference_settings(full_fits, name):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X, K, fits, same, margins = full_fits[name]
    print(name, {k: f"{v:.3g}" for k, v in margins.items()})
    assert min(margins.values()) > MARGIN_FLOOR, margins
    f = cg.gmm_fit(X, K, n_init=10, random_state=SEED)
    assert f.best_init in same
    m, labels = fits[f.best_init]
    assert (f.n_iter, f.converged) == (m.n_iter_, m.converged_)
    np.testing.assert_array_equal(f.labels, labels)
    np.testing.assert_allclose(f.lower_bound, m.lower_bound_, rtol=1e-9, atol=0)
    np.testing.assert_allclose(f.means, m.means_, rtol=0, atol=1e-8 * scale(X))
    np.testing.assert_allclose(f.weights, m.weights_, rtol=0, atol=1e-8)
    np.testing.assert_allclose(f.covariances, m.covariances_, rtol=0, atol=1e-8 * scale(m.covariances_))
    np.testing.assert_allclose(f.precisions_cholesky, m.precisions_cholesky_, rtol=0,
                               atol=1e-8 * scale(m.precisions_cholesky_))


def test_task_shape_fixed_iterations():
    from audiomuse_ai_b200 import clustering_gpu as cg
    rng = np.random.default_rng(9)
    X = rng.standard_normal((20000, 200)) + np.repeat(rng.standard_normal((60, 200)), 334, 0)[:20000]
    X = (X - X.mean(0)) / X.std(0)
    f = cg.gmm_fit(X, 60, n_init=1, max_iter=3, tol=0.0, random_state=1)
    m, labels = sk(X, 60, max_iter=3, tol=0.0, random_state=1)
    np.testing.assert_allclose(f.lower_bounds, m.lower_bounds_, rtol=1e-10, atol=0)
    np.testing.assert_allclose(f.means, m.means_, rtol=0, atol=1e-9 * scale(m.means_))
    np.testing.assert_allclose(f.covariances, m.covariances_, rtol=0, atol=1e-9 * scale(m.covariances_))
    np.testing.assert_allclose(f.precisions_cholesky, m.precisions_cholesky_, rtol=0,
                               atol=1e-9 * scale(m.precisions_cholesky_))
    diff = f.labels != labels
    if diff.any():
        lr = np.sort(m._estimate_weighted_log_prob(X)[diff], axis=1)
        gap = lr[:, -1] - lr[:, -2]
        print(f"{int(diff.sum())} labels differ, top-two gaps up to {gap.max():.3g}")
        assert (gap < 1e-8).all()


def test_float32_input_returns_float32_and_sklearn_labels():
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(5, 600, 12, 4, spread=0.3).astype(np.float32)
    g = cg.GPUGaussianMixture(4, random_state=8)
    got = g.fit_predict(X)
    _, want = sk(X.astype(np.float64), 4, n_init=10, random_state=8)
    assert g.using_gpu and g.means_.dtype == np.float32 and g.covariances_.dtype == np.float32
    assert got.dtype == np.int64
    np.testing.assert_array_equal(got, want)


def test_zero_reg_covar_on_a_constant_column_raises_like_sklearn():
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(6, 200, 5, 3)
    X[:, 2] = 1.0
    with pytest.raises(ValueError, match="ill-defined empirical covariance"):
        sk(X, 3, reg_covar=0.0, random_state=0)
    with pytest.raises(ValueError, match="ill-defined empirical covariance"):
        cg.GPUGaussianMixture(3, reg_covar=0.0, random_state=0).fit_predict(X)


def test_two_calls_are_bit_identical():
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = blobs(7, 1000, 30, 8, spread=0.5)
    a = cg.gmm_fit(X, 8, n_init=10, random_state=4)
    b = cg.gmm_fit(X, 8, n_init=10, random_state=4)
    for n in ("weights", "means", "covariances", "precisions_cholesky", "labels"):
        np.testing.assert_array_equal(getattr(a, n), getattr(b, n))
    assert a.lower_bounds == b.lower_bounds


def test_global_seed_fit_replays_the_reference_task(golden_dir):
    """The reference's _apply_clustering_model after np.random.seed(s) (tests/golden/gmm_golden.npz): the class the
    factory hands out, fitted with random_state=None, gives its labels and centres (means_), and leaves numpy's global
    generator where scikit-learn's fit leaves it."""
    import os
    from audiomuse_ai_b200 import clustering_gpu as cg
    g = np.load(os.path.join(golden_dir, "gmm_golden.npz"))
    X, seed = g["X"], int(g["seed"])
    np.random.seed(seed)
    model = cg.get_clustering_model("gmm", {"n_components": int(g["n_components"])}, use_gpu=True)
    labels = model.fit_predict(X)
    after = np.random.get_state()
    assert model.using_gpu
    np.testing.assert_array_equal(labels, g["labels"])
    centers = np.stack([model.means_[c] for c in range(len(g["centers"]))])
    np.testing.assert_allclose(centers, g["centers"], rtol=0, atol=1e-8 * scale(X))
    np.random.seed(seed)
    sk(X, int(g["n_components"]), n_init=10)
    want = np.random.get_state()
    assert after[0] == want[0] and np.array_equal(after[1], want[1]) and after[2:] == want[2:]
