"""am_knn_similar and am_knn_farthest on the GPU: the reference's recorded requests
(tests/golden/similar_tracks_golden.npz) through the drop-ins and through integration.apply, seeded 100 k-row
libraries against the float64 oracle (oracle/similar_tracks.py), candidate lists longer than 4,096, and repeat calls."""
import sys
import types

import numpy as np
import pytest

from audiomuse_ai_b200 import integration, similar_tracks as st, voyager_compat as vc
from oracle import knn as oknn
from oracle import similar_tracks as osim
from tests.golden import make_similar_tracks_golden as gen
from tests.test_gpu_song_path import _index, _library
from tests.test_similar_tracks_host import FAR_BOUND, fake_modules, run
from tests.test_song_path_host import KNN_BOUND, thr_bound

pytestmark = pytest.mark.gpu

SPACES = {"cosine": (vc.Space.Cosine, oknn.COSINE), "euclidean": (vc.Space.Euclidean, oknn.EUCLIDEAN),
          "ip": (vc.Space.InnerProduct, oknn.INNER_PRODUCT)}


def _golden_index(c, indexes):
    key = (c["library"], c["space"])
    if key not in indexes:
        indexes[key] = _index(gen.library(c["library"]), c["space"], gen.stored_rows(*key))
    return indexes[key]


def test_golden_requests_through_the_dropins(monkeypatch):
    indexes = {}
    for c in gen.load():
        got, _ = run(c, _golden_index(c, indexes), monkeypatch)
        assert got == c["result"], c["name"]


def test_golden_requests_through_integration_apply(monkeypatch):
    indexes = {}
    for c in gen.load():
        def through_apply(kind):
            def make(vm):
                app_voyager = types.ModuleType("app_voyager")
                integration.apply(similar=vm, app_voyager=app_voyager)
                return getattr(app_voyager, {"by_id": "find_nearest_neighbors_by_id",
                                             "by_vector": "find_nearest_neighbors_by_vector",
                                             "max": "get_max_distance_for_id"}[kind])
            return make
        got, _ = run(c, _golden_index(c, indexes), monkeypatch, fns={k: through_apply(k) for k in
                                                                      ("by_id", "by_vector", "max")})
        assert got == c["result"], c["name"]


def _table(N, seed):
    """Metadata for a large library: artists, duplicate titles, None authors and varied other_features."""
    rng = np.random.default_rng(seed)
    t = {}
    for i in range(N):
        t[f"item{i}"] = {"item_id": f"item{i}", "title": f"Song {i - (i % 41 == 1)}",
                         "author": None if i % 97 == 3 else f"Artist {int(rng.integers(0, N // 8))}",
                         "other_features": gen.other_features(i, rng)}
    return t


def _check_lists(got, want, name):
    assert [r["item_id"] for r in got] == [r["item_id"] for r in want], name
    assert got == want, name


@pytest.mark.parametrize("N,d,space", [(100_000, 512, "cosine"), (100_000, 200, "euclidean")])
def test_large_libraries_match_the_oracle(N, d, space, monkeypatch):
    x = _library(d, N, d)
    rows = oknn.normalize_rows(x) if space == "cosine" else x
    idx = _index(x, space, rows)
    table = _table(N, d)
    checked = 0
    for lookback, cap, thr_c, thr_e, mood_thr in ((1, 3, 0.05, 4.0, 0.15), (1, 1, 0.3, 9.0, 0.3), (0, 0, 0.05, 4.0, 0.15)):
        cfg = dict(gen.BASE, VOYAGER_METRIC="angular" if space == "cosine" else "euclidean", LOOKBACK=lookback,
                   MAX_SONGS_PER_ARTIST=cap, THRESHOLD_COSINE=thr_c, THRESHOLD_EUCLIDEAN=thr_e,
                   MOOD_SIMILARITY_THRESHOLD=mood_thr)
        vm, ah = fake_modules(idx, table, cfg)
        monkeypatch.setitem(sys.modules, "app_helper", ah)
        by_id, by_vec = st.make_find_nearest_neighbors_by_id(vm), st.make_find_nearest_neighbors_by_vector(vm)
        for j, (n, ed, mood) in enumerate(((10, True, True), (100, True, True), (200, False, True), (25, True, False))):
            target = f"item{(7919 * (j + 1) + lookback) % N}"
            want, fgap, kgap = osim.by_id(rows, space, table, cfg, target, n, ed, mood)
            if fgap > thr_bound(cfg) and kgap > KNN_BOUND:
                _check_lists(by_id(target, n=n, eliminate_duplicates=ed, mood_similarity=mood, radius_similarity=False),
                             want, (space, target))
                checked += 1
            vec = (rows[(104729 * (j + 1)) % N] + 0.05 * np.random.default_rng(j).standard_normal(d)).astype(np.float32)
            want, fgap, kgap = osim.by_vector(rows, space, table, cfg, vec, n, ed)
            if fgap > thr_bound(cfg) and kgap > KNN_BOUND:
                _check_lists(by_vec(vec, n=n, eliminate_duplicates=ed), want, (space, "vector", j))
                checked += 1
    assert checked >= 16


@pytest.mark.parametrize("space", ["cosine", "euclidean", "ip"])
@pytest.mark.parametrize("N,d", [(100_000, 200), (100_000, 512)])
def test_farthest_matches_the_oracle(N, d, space):
    x = _library(d + 1, N, d)
    vspace, ometric = SPACES[space]
    idx = vc.Index(vspace, num_dimensions=d)
    idx.add_items(x, ids=np.arange(N))
    rows = oknn.normalize_rows(x) if space == "cosine" else x
    for t in (0, 12345, N - 1, N - 50 - 1):   # the last rows are copies of the first ones
        want, gap = osim.max_distance(rows, space, f"item{t}", metric=ometric)
        dist, far = idx.farthest(t)
        assert gap > FAR_BOUND, (space, t)
        assert (dist, f"item{far}") == (want["max_distance"], want["farthest_item_id"]), (space, t)
        # the value the query path returns for that row
        ids, dists = idx.query(idx.get_vector(t), k=N)
        assert float(dists[list(ids).index(far)]) == dist


def test_farthest_agrees_with_the_full_query_loop():
    """The reference's loop over query(k=len) on a library with exact duplicates at the far end."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((5000, 64)).astype(np.float32)
    x[4000:4010] = -x[0] * 3
    for space in ("cosine", "euclidean", "ip"):
        idx = vc.Index(SPACES[space][0], num_dimensions=64)
        idx.add_items(x, ids=np.arange(len(x)))
        for t in (0, 1, 4005):
            ids, dists = idx.query(idx.get_vector(t), k=len(x))
            best, far = float("-inf"), None
            for i, dd in zip(ids, dists):
                if int(i) != t and dd > best:
                    best, far = dd, int(i)
            assert idx.farthest(t) == (float(best), far), (space, t)
    one = vc.Index(vc.Space.Cosine, num_dimensions=64)
    one.add_items(x[:1])
    assert one.farthest(0) == (0.0, None)


def test_candidate_lists_longer_than_4096(monkeypatch):
    N, d = 100_000, 200
    x = _library(7, N, d)
    rows = oknn.normalize_rows(x)
    idx = _index(x, "cosine", rows)
    table = _table(N, 7)
    cfg = dict(gen.BASE, THRESHOLD_COSINE=0.05, MAX_SONGS_PER_ARTIST=2)
    vm, ah = fake_modules(idx, table, cfg)
    monkeypatch.setitem(sys.modules, "app_helper", ah)
    calls = []
    similar = idx.similar

    def counted(*a, **k):
        calls.append(len(a[3]))
        return similar(*a, **k)

    idx.similar = counted
    try:
        vec = (rows[11] + 0.05 * np.random.default_rng(3).standard_normal(d)).astype(np.float32)
        want, fgap, kgap = osim.by_vector(rows, "cosine", table, cfg, vec, 1000, True)
        assert fgap > thr_bound(cfg) and kgap > KNN_BOUND
        _check_lists(st.make_find_nearest_neighbors_by_vector(vm)(vec, n=1000, eliminate_duplicates=True), want, "vec")
        want, fgap, kgap = osim.by_id(rows, "cosine", table, cfg, "item12", 500, True, True)
        assert fgap > thr_bound(cfg) and kgap > KNN_BOUND
        _check_lists(st.make_find_nearest_neighbors_by_id(vm)("item12", n=500, eliminate_duplicates=True,
                                                              mood_similarity=True, radius_similarity=False),
                     want, "id")
    finally:
        del idx.similar
    assert calls[0] == 5000 and calls[1] == 4501 - 1


def test_two_calls_are_bit_identical(monkeypatch):
    c = next(c for c in gen.load() if c["name"] == "id_n500_mood")
    idx = _index(gen.library(c["library"]), c["space"], gen.stored_rows(c["library"], c["space"]))
    a, _ = run(c, idx, monkeypatch)
    b, _ = run(c, idx, monkeypatch)
    assert a == b == c["result"]
    x = _library(9, 100_000, 200)
    big = vc.Index(vc.Space.Euclidean, num_dimensions=200)
    big.add_items(x)
    assert big.farthest(77) == big.farthest(77)
