"""The artist-similarity GMM sweep on the device (audiomuse_ai_b200.artist_gmm, csrc/artist_gmm.cu) against the float64
oracle (oracle/artist_gmm.py), against scikit-learn on float64 input, and against the reference's own float32 run
(tests/golden/artist_gmm_golden.npz)."""
import json
import os
import warnings

import numpy as np
import pytest

from oracle import artist_gmm as og

pytestmark = pytest.mark.gpu

MARGIN_FLOOR = 1e-9       # every discrete decision of the seeded sets is at least this far from flipping
# Bounds and BIC agree to 1e-10 relative.  A component that collapses onto duplicated rows has a covariance of
# reg_covar (1e-6) plus the residue of E[x^2] - mean^2 for O(1) values, so its precisions carry ~1e-16 / 1e-6 relative
# rounding whatever the summation order; on the set built for that, the bounds agree to 1e-8.
REL = {"dups": 1e-8}


def artist_rows(seed, n, d, groups=4, spread=0.8, dup=0, const=False):
    rng = np.random.default_rng(seed)
    if const:
        return np.tile(rng.standard_normal(d).astype(np.float32), (n, 1))
    c = rng.standard_normal((groups, d))
    X = c[rng.integers(0, groups, n)] + spread * rng.standard_normal((n, d))
    if dup:
        X[rng.integers(0, n, dup)] = X[rng.integers(0, n, dup)]
    return X.astype(np.float32)


def _stage_limit(d):
    from audiomuse_ai_b200 import artist_gmm as ag
    return ag.SMEM_BYTES // (4 * d)


def seeded_sets():
    """(name, rows, max_components)"""
    lim = _stage_limit(200)
    return [
        ("stage_below", artist_rows(1, lim, 200), 10),
        ("stage_above", artist_rows(2, lim + 1, 200), 10),
        ("d128", artist_rows(3, 90, 128, groups=3), 10),
        ("d256", artist_rows(4, 60, 256, groups=5, spread=1.0), 10),
        ("d512", artist_rows(5, 40, 512, groups=2), 10),
        ("k16", artist_rows(6, 96, 200, groups=8, spread=1.2), 16),
        ("dups", artist_rows(7, 50, 200, groups=3, dup=20), 10),
        ("const", artist_rows(8, 30, 200, const=True), 10),
        ("n6000", artist_rows(9, 6000, 128, groups=6, spread=1.5), 10),
        ("few_rows", artist_rows(10, 7, 200), 10),
    ]


@pytest.fixture(scope="module")
def sets():
    return seeded_sets()


@pytest.fixture(scope="module")
def device_fits(sets):
    from audiomuse_ai_b200 import artist_gmm as ag
    out = {}
    for name, X, kmax in sets:
        out[name] = ag.fit_artist_gmms([X], max_components=kmax, intermediates=True)[0]
    return out


@pytest.fixture(scope="module")
def oracle_fits(sets):
    return {name: og.select(X.astype(np.float64), max_components=kmax) for name, X, kmax in sets}


def _close_f32(dev, ref, rel):
    """float32 output of a float64 value: within half a float32 ulp of it, plus rel of the array's largest magnitude"""
    ref = np.asarray(ref, np.float64)
    tol = 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + rel * np.abs(ref).max()
    return np.all(np.abs(dev.astype(np.float64) - ref) <= tol * (1 + 1e-12))


def test_device_equals_the_oracle(sets, device_fits, oracle_fits):
    for name, X, kmax in sets:
        f, o = device_fits[name], oracle_fits[name]
        assert f.k == o["K"], name
        for K, of in o["fits"].items():
            assert f.failed[K] == of["failed"], (name, K)
            if of["failed"]:
                continue
            for i in range(og.N_INIT):
                np.testing.assert_array_equal(f.kpp[K - 1, i, :K], of["kpp"][i], err_msg=f"{name} K={K} init {i}")
                np.testing.assert_array_equal(f.labels[K - 1, i], of["labels"][i], err_msg=f"{name} K={K} init {i}")
                assert f.n_iter[K - 1, i] == of["n_iter"][i], (name, K, i)
                assert f.converged[K - 1, i] == of["converged"][i], (name, K, i)
                assert f.lower_bound[K - 1, i] == pytest.approx(of["lower_bound"][i], rel=REL.get(name, 1e-10),
                                                               abs=0), (name, K, i)
            best = 0                 # the first init with the strictly greater bound
            for i in range(1, og.N_INIT):
                if f.lower_bound[K - 1, i] > f.lower_bound[K - 1, best]:
                    best = i
            # inits that start from the same partition reach the same mixture: either may be kept
            assert og.same_partition(of["labels"][best], of["labels"][of["best_init"]]), (name, K)
            assert f.bic[K] == pytest.approx(of["bic"], rel=REL.get(name, 1e-10), abs=0), (name, K)
        b = o["best"]
        if b is not None:
            p = _match_by_means(f.means, b["means"])
            rel = 1e-9 if name not in REL else 1e-7
            assert _close_f32(f.weights, b["weights"][p], rel), name
            assert _close_f32(f.means, b["means"][p], rel), name
            assert _close_f32(f.covariances, b["covariances"][p], rel), name


def test_seeded_sets_have_no_knife_edges(oracle_fits):
    for name, o in oracle_fits.items():
        for key, v in o["margins"].items():
            assert v > MARGIN_FLOOR, (name, key, v)


def test_batch_invariance(sets, device_fits):
    """one call over every set, in shuffled order, gives each artist bit for bit its single-artist result"""
    from audiomuse_ai_b200 import artist_gmm as ag
    rows = [X for _, X, _ in sets if X.shape[1] == 200]
    names = [n for n, X, _ in sets if X.shape[1] == 200]
    order = np.random.default_rng(0).permutation(len(rows))
    batch = ag.fit_artist_gmms([rows[i] for i in order], intermediates=True)
    for j, i in enumerate(order):
        a, b = batch[j], ag.fit_artist_gmms([rows[i]], intermediates=True)[0]
        assert a.k == b.k and a.bic.keys() == b.bic.keys(), names[i]
        assert np.array_equal(np.array(list(a.bic.values())), np.array(list(b.bic.values())), equal_nan=True)
        for attr in ("lower_bound", "n_iter", "converged", "weights", "means", "covariances", "kpp", "labels"):
            x, y = getattr(a, attr), getattr(b, attr)
            assert (x is None and y is None) or np.array_equal(x, y, equal_nan=True), (names[i], attr)


def _match_by_means(m_dev, m_ref):
    from scipy.optimize import linear_sum_assignment
    cost = ((m_dev[:, None, :].astype(np.float64) - m_ref[None, :, :]) ** 2).sum(-1)
    r, c = linear_sum_assignment(cost)
    return c[np.argsort(r)]


def test_device_matches_sklearn_on_float64_input(sets, device_fits):
    from sklearn.mixture import GaussianMixture
    warnings.filterwarnings("ignore")
    for name, X, kmax in sets:
        if len(X) > 500:
            continue
        X64 = X.astype(np.float64)
        best, best_k, best_gm = np.inf, None, None
        for K in range(1, og.max_feasible(len(X), 2, kmax) + 1):
            try:
                gm = GaussianMixture(K, covariance_type="diag", max_iter=100, n_init=3, random_state=42).fit(X64)
            except ValueError:
                continue
            b = gm.bic(X64)
            if b < best:
                best, best_k, best_gm = b, K, gm
        f = device_fits[name]
        assert f.k == best_k, name
        p = _match_by_means(f.means, best_gm.means_)
        for dev, ref in ((f.weights, best_gm.weights_[p]), (f.means, best_gm.means_[p]),
                         (f.covariances, best_gm.covariances_[p])):
            assert _close_f32(dev, ref, 1e-8), name


# ------------------------------------------------------------------------------------------------ the reference's run
@pytest.fixture(scope="module")
def golden(golden_dir):
    import sys
    sys.path.insert(0, golden_dir)
    import make_artist_gmm_golden as mk
    g = np.load(os.path.join(golden_dir, "artist_gmm_golden.npz"))
    rows, emb, _ = mk.library()
    return g, emb


def _fitted(g, emb):
    """(name, rows as fetched, K, weights, means, covariances) of the artists the reference fitted"""
    out, p = [], 0
    off, idx = g["row_offsets"], g["row_index"]
    for a, name in enumerate(g["artists"]):
        K = int(g["n_components"][a])
        if K <= 0 or g["is_few_songs"][a]:
            continue
        X = emb[idx[off[a]:off[a + 1]]]
        out.append((str(name), X, K, g["weights"][p:p + K], g["means"][p:p + K], g["covariances"][p:p + K]))
        p += K
    return out


def test_device_against_the_reference_float32_run(golden):
    """the deployed float32 reference: the same K for at least 97 % of the fitted artists; where K agrees, the mean
    log-likelihood of the rows under the device's mixture is never more than 1e-5 relative below the reference's.
    It is often far above it: the float32 run stops on a worse optimum for 41 of the 79 artists (DESIGN.md)"""
    from audiomuse_ai_b200 import artist_gmm as ag
    arts = _fitted(*golden)
    fits = ag.fit_artist_gmms([X for _, X, *_ in arts])
    agree, rel = 0, []
    for (name, X, K, w, m, c), f in zip(arts, fits):
        if f.k != K:
            continue
        agree += 1
        X64 = X.astype(np.float64)
        ll = [og.score(X64, ww.astype(np.float64), mm.astype(np.float64), 1.0 / np.sqrt(cc.astype(np.float64)))
              for ww, mm, cc in ((f.weights, f.means, f.covariances), (w, m, c))]
        rel.append((ll[0] - ll[1]) / abs(ll[1]))
    assert agree >= 0.97 * len(arts), (agree, len(arts))
    assert min(rel) >= -1e-5, min(rel)


def test_drop_in_dicts_have_the_reference_shape(golden):
    """fit_artist_gmm on every golden artist's fetched rows: None where the reference stored nothing, the reference's
    keys, float32 values, weights summing to 1, shapes of K and d; few-song artists byte for byte"""
    import hashlib
    from audiomuse_ai_b200 import artist_gmm as ag
    g, emb = golden
    off, idx = g["row_offsets"], g["row_index"]
    for a, name in enumerate(g["artists"]):
        X = emb[idx[off[a]:off[a + 1]]]
        got = ag.fit_artist_gmm(str(name), [r for r in X])
        if int(g["n_components"][a]) < 0:
            assert got is None, name
            continue
        K, d = got["n_components"], got["n_features"]
        assert set(got) == {"weights", "means", "covariances", "n_components", "covariance_type", "n_features",
                            "n_tracks", "is_few_songs"}
        assert d == X.shape[1] and got["n_tracks"] == len(X) and got["covariance_type"] == "diag"
        assert len(got["weights"]) == K and np.array(got["means"]).shape == (K, d)
        assert np.array(got["covariances"]).shape == (K, d)
        assert abs(sum(got["weights"]) - 1.0) <= 1e-6
        for key in ("weights", "means", "covariances"):
            v = np.array(got[key], np.float64)
            assert got["is_few_songs"] or np.array_equal(v, v.astype(np.float32).astype(np.float64)), (name, key)
        assert got["is_few_songs"] == bool(g["is_few_songs"][a])
        if got["is_few_songs"]:
            got["tracks_hash"] = str(g["tracks_hash"][a])      # what build_and_store_artist_index adds
            assert hashlib.sha256(json.dumps(got).encode()).hexdigest() == str(g["params_sha256"][a]), name


def test_the_reference_unit_contract():
    """what the reference's own unit tests ask of the two functions, with seeded data"""
    from audiomuse_ai_b200 import artist_gmm as ag
    rng = np.random.default_rng(12)
    assert ag.select_optimal_gmm_components(rng.random((1, 128))) == 1
    assert 1 <= ag.select_optimal_gmm_components(rng.random((2, 128))) <= 2
    for n in (3, 4, 5):
        assert 1 <= ag.select_optimal_gmm_components(rng.random((n, 64))) <= n
    X = artist_rows(20, 100, 64)
    assert 1 <= ag.select_optimal_gmm_components(X) <= 20
    assert ag.select_optimal_gmm_components(X, min_components=3, max_components=5) <= 5
    assert ag.select_optimal_gmm_components(X, max_components=3) <= 3
    assert ag.select_optimal_gmm_components(X) == ag.select_optimal_gmm_components(X.copy())
    assert 1 <= ag.select_optimal_gmm_components(artist_rows(21, 50, 512)) <= 10
    one = ag.fit_artist_gmm("one", [rng.random(64).astype(np.float32)])
    assert one["n_components"] == 1 and one["is_few_songs"] and one["weights"] == [1.0]
    few = ag.fit_artist_gmm("few", list(rng.random((3, 64)).astype(np.float32)))
    assert few["n_components"] == 3 and few["is_few_songs"]
    many = ag.fit_artist_gmm("many", list(artist_rows(22, 60, 64)))
    assert not many["is_few_songs"] and many["covariance_type"] == "diag" and many["n_features"] == 64
    assert many["n_tracks"] == 60 and abs(sum(many["weights"]) - 1.0) < 1e-6
    assert np.array(many["means"]).shape == np.array(many["covariances"]).shape == (many["n_components"], 64)
    other = ag.fit_artist_gmm("other", list(artist_rows(23, 60, 64)))
    assert not np.allclose(np.array(many["means"]).mean(0), np.array(other["means"]).mean(0))
    assert ag.fit_artist_gmm("empty", []) is None
    assert ag.fit_artist_gmm("ragged", [np.ones(64, np.float32)] * 5 + [np.ones(32, np.float32)]) is None
