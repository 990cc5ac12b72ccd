"""Host-side contracts of the artist-similarity GMM sweep (audiomuse_ai_b200.artist_gmm) and of the float64 oracle it is
tested against (oracle/artist_gmm.py).  No GPU compute is issued here."""
import hashlib
import json
import os
import sys
import types
import warnings

import numpy as np
import pytest

from oracle import artist_gmm as og

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_artist_gmm_golden as mk  # noqa: E402

warnings.filterwarnings("ignore", module="sklearn")


def _artist(seed, n, d, groups=4, spread=0.8):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((groups, d))
    return (c[rng.integers(0, groups, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)


def test_draw_table_is_what_a_fit_consumes():
    """GaussianMixture(K, n_init=3, random_state=rs).fit leaves rs exactly after the table's K prefix"""
    from sklearn.mixture import GaussianMixture
    from audiomuse_ai_b200 import artist_gmm as ag
    full = ag.draw_table()
    np.testing.assert_array_equal(full[:len(og.draw_table(10))], og.draw_table(10))
    X = _artist(0, 60, 16).astype(np.float64)
    for K in range(1, 11):
        rs = np.random.RandomState(og.SEED)
        GaussianMixture(K, covariance_type="diag", max_iter=100, n_init=3, random_state=rs).fit(X)
        ref = np.random.RandomState(og.SEED)
        np.testing.assert_array_equal(ref.random_sample(3 * og.draws_per_init(K)), full[:3 * og.draws_per_init(K)])
        assert rs.random_sample() == ref.random_sample(), K


CASES = [(5, 128), (12, 200), (40, 512), (90, 200), (200, 128), (500, 200)]


@pytest.mark.parametrize("n,d", CASES)
def test_oracle_equals_sklearn_on_float64(n, d):
    from sklearn.cluster import KMeans, kmeans_plusplus
    from sklearn.mixture import GaussianMixture
    X = _artist(n * 7 + d, n, d, groups=3 + n % 4, spread=1.1).astype(np.float64)
    sel = og.select(X)
    best, best_k = np.inf, None
    Xc = X - X.mean(0)
    for K in range(1, og.max_feasible(n) + 1):
        f = sel["fits"][K]
        gm = GaussianMixture(K, covariance_type="diag", max_iter=100, n_init=3, random_state=og.SEED).fit(X)
        for i in range(og.N_INIT):
            rs = np.random.RandomState(og.SEED)
            rs.random_sample(i * og.draws_per_init(K))
            _, idx = kmeans_plusplus(Xc, K, random_state=rs)
            np.testing.assert_array_equal(idx, f["kpp"][i])
            rs = np.random.RandomState(og.SEED)
            rs.random_sample(i * og.draws_per_init(K))
            np.testing.assert_array_equal(KMeans(K, n_init=1, random_state=rs).fit(X).labels_, f["labels"][i])
        b = gm.bic(X)
        assert f["bic"] == pytest.approx(b, rel=1e-10, abs=0)
        assert f["lower_bound"][f["best_init"]] == pytest.approx(gm.lower_bound_, rel=1e-10, abs=0)
        for mine, ref in ((f["weights"], gm.weights_), (f["means"], gm.means_), (f["covariances"], gm.covariances_)):
            assert np.abs(mine - ref).max() <= 1e-9 * np.abs(ref).max()
        if b < best:
            best, best_k = b, K
    assert sel["K"] == best_k


def test_max_feasible_is_the_reference_rule():
    from audiomuse_ai_b200 import artist_gmm as ag
    for n, lo, hi, want in [(1, 2, 10, 1), (2, 2, 10, 2), (5, 2, 10, 5), (6, 2, 10, 2), (9, 2, 10, 2), (10, 2, 10, 2),
                            (15, 2, 10, 3), (49, 2, 10, 9), (50, 2, 10, 10), (5000, 2, 10, 10), (30, 4, 10, 6),
                            (8, 3, 10, 3), (5, 2, 3, 3), (100, 2, 4, 4), (3, 5, 10, 3)]:
        assert ag.max_feasible(n, lo, hi) == og.max_feasible(n, lo, hi) == want, (n, lo, hi)


@pytest.fixture
def no_device(monkeypatch):
    from audiomuse_ai_b200 import _lib

    def missing():
        raise _lib.B200Error(_lib.AM_ERR_NO_DEVICE, "no device in this test")

    monkeypatch.setattr(_lib, "load", missing)
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)


def test_failure_values_before_any_device_work(no_device):
    from audiomuse_ai_b200 import artist_gmm as ag
    assert ag.fit_artist_gmm("nobody", []) is None
    assert ag.fit_artist_gmm("ragged", [np.ones(8, np.float32), np.ones(9, np.float32)] * 4) is None
    bad = _artist(1, 30, 8)
    bad[3, 2] = np.nan
    assert ag.select_optimal_gmm_components(bad) == 2
    assert ag.select_optimal_gmm_components(bad, min_components=3) == 3
    bad[3, 2] = np.inf
    assert ag.fit_artist_gmm("inf", list(bad)) is None
    assert ag.select_optimal_gmm_components(np.ones((1, 8))) == 1
    with pytest.raises(ValueError):
        ag.fit_artist_gmms([bad])
    with pytest.raises(ValueError):
        ag.fit_artist_gmms([np.ones((5, 1025), np.float32)])
    with pytest.raises(ValueError):
        ag.fit_artist_gmms([np.ones((200, 4), np.float32)], max_components=17)


def test_no_device_raises_or_returns_none(no_device, caplog):
    from audiomuse_ai_b200 import _lib, artist_gmm as ag
    X = _artist(2, 20, 8)
    with pytest.raises(_lib.B200Error):
        ag.select_optimal_gmm_components(X)
    assert ag.fit_artist_gmm("someone", list(X)) is None
    assert "someone" in caplog.text


def test_few_song_artists_are_the_reference_byte_for_byte(no_device):
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "artist_gmm_golden.npz"))
    from audiomuse_ai_b200 import artist_gmm as ag
    _, emb, _ = mk.library()
    assert hashlib.sha256(emb.tobytes()).hexdigest() == str(g["library_sha256"])
    off, idx = g["row_offsets"], g["row_index"]
    few = np.flatnonzero(g["is_few_songs"])
    assert len(few) >= 20 and set(g["n_components"][few]) == {1, 2, 3, 4}
    for a in few:
        got = ag.fit_artist_gmm(str(g["artists"][a]), list(emb[idx[off[a]:off[a + 1]]]))
        got["tracks_hash"] = str(g["tracks_hash"][a])
        assert hashlib.sha256(json.dumps(got).encode()).hexdigest() == str(g["params_sha256"][a])


def test_golden_library_covers_the_cases():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "artist_gmm_golden.npz"))
    rows, emb, null = mk.library()
    sizes = np.diff(g["row_offsets"])
    assert sizes.max() > 2000 and len(null) > 0 and (sizes < 5).sum() >= 20
    const = emb[[i for i, r in enumerate(rows) if r[0] == f"Artist {mk.CONST_ARTIST:03d}"]]
    assert (const == const[0]).all()
    assert json.loads(str(g["artist_map_json"])) == {str(i): str(a) for i, a in enumerate(g["artists"])
                                                     if g["n_components"][i] > 0}


def test_oracle_agrees_with_the_reference_float32_choice_of_k():
    """The reference runs scikit-learn in float32; the float64 oracle chose the same K for all 79 fitted golden
    artists (DESIGN.md).  The bar is 97 %."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "artist_gmm_golden.npz"))
    _, emb, _ = mk.library()
    off, idx = g["row_offsets"], g["row_index"]
    agree = total = 0
    for a in range(len(g["artists"])):
        K = int(g["n_components"][a])
        if K <= 0 or g["is_few_songs"][a]:
            continue
        total += 1
        agree += og.select(emb[idx[off[a]:off[a + 1]]].astype(np.float64))["K"] == K
    assert total == 79 and agree >= 0.97 * total, (agree, total)


def test_integration_patches_the_module_and_the_fallback_calls_the_originals(monkeypatch, no_device):
    from audiomuse_ai_b200 import artist_gmm as ag, integration
    calls = []
    mod = types.ModuleType("tasks.artist_gmm_manager")
    mod.fit_artist_gmm = lambda name, emb: calls.append(("fit", name)) or {"orig": True}
    mod.select_optimal_gmm_components = lambda e, lo=2, hi=10: calls.append(("select", len(e))) or 7
    monkeypatch.setattr(ag, "_originals", {})
    integration.apply(artist_gmm_manager=mod, allow_sklearn_fallback=False)
    assert mod.fit_artist_gmm is ag.fit_artist_gmm
    assert mod.select_optimal_gmm_components is ag.select_optimal_gmm_components
    integration.apply(artist_gmm_manager=mod, allow_sklearn_fallback=False)     # twice: the originals stay captured
    X = _artist(3, 20, 8)
    assert mod.fit_artist_gmm("a", list(X)) is None and calls == []
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    assert mod.select_optimal_gmm_components(X) == 7
    assert mod.fit_artist_gmm("a", list(X)) == {"orig": True}
    assert calls == [("select", 20), ("fit", "a")]
