"""am_knn_radius_walk on the GPU: the reference's playlists (tests/golden/radius_walk_golden.npz) through the
integration drop-in, and seeded pools against the float64 oracle (oracle/radius_walk.py)."""
import threading

import numpy as np
import pytest

from oracle import radius_walk as orw
from tests.golden import make_radius_walk_golden as gen

pytestmark = pytest.mark.gpu

GAP = 1e-6


def _close(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    assert np.all(np.abs(got[fin] - want[fin]) <= 2e-6 + 1e-6 * np.abs(want[fin]))


def _index(rows):
    """The walk reads the stored rows whatever the index space: a Euclidean-space index stores them as given."""
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Euclidean, num_dimensions=rows.shape[1])
    idx.add_items(rows, ids=np.arange(len(rows)))
    return idx


def test_golden_cases_through_the_dropin():
    import types

    from audiomuse_ai_b200 import integration
    cases = gen.load()
    indexes, exact = {}, 0
    for case in cases:
        key = (case["library"], case["space"])
        if key not in indexes:
            rows = gen.stored_rows(*key)
            indexes[key] = (rows, _index(rows))
        rows, idx = indexes[key]
        anchor_calls = []

        def cached_vector(item_id, idx=idx, calls=anchor_calls):
            calls.append(item_id)
            return idx.get_vector(int(item_id[4:]))

        vm = types.SimpleNamespace(voyager_index=idx, MAX_SONGS_PER_ARTIST=case["max_songs_per_artist"],
                                   VOYAGER_METRIC=case["metric"], _get_cached_vector=cached_vector)
        w = case["walk_in"]
        cd = [{"item_id": f"item{v}", "row": v, "title": None, "author": a} for v, a in zip(w["vid"], w["author"])]
        _, walk = integration.make_radius_walk(vm)
        out = walk(case["target"], case["n"], cd, None, case["eliminate_duplicates"])
        assert anchor_calls == [case["target"]]          # the anchor only: no per-candidate vector fetch
        got = [int(r["item_id"][4:]) for r in out]
        if min(case["sort_gap"], case["score_gap"]) > GAP:
            want = case["walk_out"]["vid"]
            exact += 1
        else:
            r = orw.radius_walk([rows[v] for v in w["vid"]], rows[int(case["target"][4:])], w["author"], case["n"],
                                case["eliminate_duplicates"], case["max_songs_per_artist"], case["metric"],
                                mode="float64")
            want = [w["vid"][p] for p in r["positions"]]
        assert got == want, case["name"]
        if got == case["walk_out"]["vid"]:
            _close([r["distance"] for r in out], case["walk_out"]["distance"])
    assert exact >= 15


def _pool(seed, N, d, k, zero_row=False, missing=False):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((32, d)).astype(np.float32)
    X = (base[rng.integers(0, 32, N)] + 0.5 * rng.standard_normal((N, d)).astype(np.float32)).astype(np.float32)
    if zero_row:
        X[7] = 0.0
    ids = rng.choice(N, size=k, replace=False).astype(np.int64)
    if zero_row:
        ids[3] = 7
    anchor = X[int(rng.integers(0, N))].copy()
    if missing:
        ids[5] = N + 10
    return X, anchor, ids


POOLS = [  # seed, N, d, n, metric, eliminate_duplicates, cap, artists ("random" / "one"), zero row, missing id
    (1, 6000, 200, 10, "angular", True, 3, "random", True, True),
    (2, 6000, 512, 100, "angular", True, 3, "random", False, False),
    (3, 6000, 200, 100, "euclidean", True, 1, "random", False, True),
    (4, 20000, 512, 2000, "angular", True, 3, "random", True, False),
    (5, 20000, 200, 2000, "euclidean", False, 3, "random", False, False),
    (6, 6000, 512, 100, "angular", True, 0, "one", False, False),
    (7, 6000, 200, 100, "euclidean", True, 1, "one", False, False),
    (8, 6000, 512, 100, "angular", True, 3, "one", False, False),
    (9, 6000, 200, 60, "angular", False, 3, "one", False, False),
]


@pytest.mark.parametrize("seed,N,d,n,metric,ed,cap,artist_kind,zero_row,missing", POOLS)
def test_seeded_pools_match_the_float64_oracle(seed, N, d, n, metric, ed, cap, artist_kind, zero_row, missing):
    k = n + max(20, 3 * n) + 1
    X, anchor, ids = _pool(seed, N, d, k, zero_row, missing)
    rng = np.random.default_rng(100 + seed)
    artists = (rng.integers(-1, max(25, n), k).astype(np.int32) if artist_kind == "random"
               else np.zeros(k, np.int32))
    idx = _index(X)
    pos, dist = idx.radius_walk(anchor, ids, artists, n, ed, cap, metric)
    vecs = [X[i] if i < N else None for i in ids]
    r = orw.radius_walk(vecs, anchor, _authors(artists), n, ed, cap, metric, mode="float64")
    assert r["sort_gap"] > 1e-12 and r["score_gap"] > 1e-12
    assert pos.tolist() == r["positions"]
    _close(dist, r["distances"])
    if artist_kind == "one" and ed and cap > 0:
        assert len(pos) == min(cap, 3)     # the first song, one per bucket in the next two buckets, never past the cap


def _authors(artists):
    return [f"artist {a}" if a >= 0 else None for a in np.asarray(artists).tolist()]


def test_zero_vector_is_never_walked_to():
    """A zero vector is at +inf from everything under the angular metric: it sorts last and its score is never below
    +inf, so the reference's walk never takes it."""
    X, anchor, ids = _pool(11, 2000, 200, 41, zero_row=True)
    pos, _ = _index(X).radius_walk(anchor, ids, np.full(41, -1, np.int32), 41, False, 3, "angular")
    assert len(pos) == 40 and 3 not in pos.tolist()


def test_two_calls_are_bit_identical_and_threads_get_their_own_answers():
    X, anchor, ids = _pool(21, 8000, 512, 401)
    idx = _index(X)
    rng = np.random.default_rng(3)
    jobs = []
    for t in range(4):
        sub = rng.permutation(ids)
        art = rng.integers(-1, 12, len(sub)).astype(np.int32)
        jobs.append((sub, art, [10, 25, 100, 200][t]))
    single = [idx.radius_walk(anchor, s, a, n, True, 3, "angular") for s, a, n in jobs]
    again = [idx.radius_walk(anchor, s, a, n, True, 3, "angular") for s, a, n in jobs]
    for (p1, d1), (p2, d2) in zip(single, again):
        assert np.array_equal(p1, p2) and np.array_equal(d1.view(np.int64), d2.view(np.int64))
    results, errors = [None] * 4, []

    def worker(t):
        try:
            s, a, n = jobs[t]
            for _ in range(5):
                results[t] = idx.radius_walk(anchor, s, a, n, True, 3, "angular")
                assert np.array_equal(results[t][0], single[t][0])
                assert np.array_equal(results[t][1].view(np.int64), single[t][1].view(np.int64))
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
