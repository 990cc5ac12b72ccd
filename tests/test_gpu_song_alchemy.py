"""am_knn_alchemy on the GPU: the reference's Song Alchemy requests (tests/golden/song_alchemy_golden.npz) through the
drop-in and through integration.apply, seeded 100 k-row libraries against the float64 oracle
(oracle/song_alchemy.py), and repeat calls."""
import math
import types

import numpy as np
import pytest

from oracle import song_alchemy as osa
from tests import ref_harness as rh
from tests.golden import make_song_alchemy_golden as gen
from tests.test_gpu_song_path import _index, _library
from tests.test_song_alchemy_host import DECISION_BOUND, helper_modules, modules, run  # noqa: F401
from tests.test_song_path_host import KNN_BOUND, thr_bound

pytestmark = pytest.mark.gpu

# Both sides compute the centroid distances in float64 from the same float32 rows, in different summation orders: the
# cosine differs by a few ulps (1e-15 covers d <= 512), which arccos / pi turns into 1e-15 / (pi sin(pi t)) at a
# distance t.  Every recorded distance is far enough from 0 and 1 for that to stay below 1e-13.
DIST_ATOL = 1e-12


def dist_tol(d, metric):
    if metric != "angular":
        return DIST_ATOL
    return DIST_ATOL + 1e-15 / (math.pi * max(math.sin(math.pi * d), 1e-300))


def assert_same_answer(got, want, metric, name):
    """The dicts are equal but for the distances, which agree within dist_tol."""
    assert [r["item_id"] for r in got["results"]] == [r["item_id"] for r in want["results"]], name
    assert [r["item_id"] for r in got["filtered_out"]] == [r["item_id"] for r in want["filtered_out"]], name
    for g, w in zip(got["results"], want["results"]):
        assert abs(g["distance"] - w["distance"]) <= dist_tol(w["distance"], metric), (name, g["item_id"])
        g["distance"] = w["distance"]
    assert got == want, name


class Counted:
    """Counts the device index's query and alchemy calls."""

    def __init__(self, idx):
        self.idx, self.query, self.alchemy = idx, 0, 0

    def __enter__(self):
        query, alchemy = self.idx.query, self.idx.alchemy

        def counted_query(*a, **k):
            self.query += 1
            return query(*a, **k)

        def counted_alchemy(*a, **k):
            self.alchemy += 1
            return alchemy(*a, **k)

        self.idx.query, self.idx.alchemy = counted_query, counted_alchemy
        return self

    def __exit__(self, *exc):
        del self.idx.query, self.idx.alchemy


def _golden_index(c, indexes):
    key = (c["library"], c["space"])
    if key not in indexes:
        indexes[key] = _index(gen.library(c["library"]), c["space"], gen.stored_rows(*key))
    return indexes[key]


def test_golden_requests_through_the_dropin(helper_modules):  # noqa: F811
    indexes = {}
    for c in gen.load():
        idx = _golden_index(c, indexes)
        with Counted(idx) as calls:
            got = run(c, idx, helper_modules)
        assert_same_answer(got, c["result"], c["config"]["PATH_DISTANCE_METRIC"], c["name"])
        if c["result"]["results"]:
            by_id = any(k.startswith("find_nearest_neighbors_by_id") for k in c["calls"])
            assert (calls.query, calls.alchemy) == (0 if by_id else 1, 1), c["name"]


def test_golden_requests_through_integration_apply(helper_modules):  # noqa: F811
    import sys

    from audiomuse_ai_b200 import integration
    indexes = {}
    for c in gen.load()[::4]:
        idx = _golden_index(c, indexes)
        sa, vm, ah, aha = modules(c, idx)
        helper_modules(ah, aha)
        sys.modules[vm.__name__] = vm
        try:
            app = types.ModuleType("app_alchemy")
            sa.find_nearest_neighbors_by_id.__module__ = vm.__name__
            integration.apply(alchemy=sa, app_alchemy=app)
            got = run(c, idx, helper_modules, fn=app.song_alchemy)
        finally:
            del sys.modules[vm.__name__]
        assert_same_answer(got, c["result"], c["config"]["PATH_DISTANCE_METRIC"], c["name"])


def _alchemy_cfg(space, n, lookback, cap, sub_thr):
    from audiomuse_ai_b200 import _lib
    return _lib.AlchemyCfg(voyager_metric=0 if space == "cosine" else 1, path_metric=0 if space == "cosine" else 1,
                           filter_lookback=lookback, filter_batch=50, voyager_cap=cap, n=n, skip_chain=0,
                           filter_threshold=0.01 if space == "cosine" else 0.15, subtract_threshold=sub_thr)


@pytest.mark.parametrize("N,d,space", [(100_000, 512, "cosine"), (100_000, 200, "euclidean")])
def test_large_libraries_match_the_oracle(N, d, space):
    from audiomuse_ai_b200 import song_path as sp
    from oracle import knn as oknn
    x = _library(d, N, d)
    rows = oknn.normalize_rows(x) if space == "cosine" else x
    idx = _index(x, space, rows)
    table = rh.make_score_table(N, seed=d)
    for i in range(0, N, 97):
        table[f"item{i}"]["author"] = None if i % 2 else ""
    rng = np.random.default_rng(N + d)
    metric = "angular" if space == "cosine" else "euclidean"
    checked = 0
    for n_results, with_sub, lookback, cap in ((10, False, 1, 3), (100, True, 1, 3), (200, True, 1, 1),
                                               (200, False, 0, 0), (100, True, 3, 0)):
        add = [int(v) for v in rng.choice(N, 3, replace=False)]
        add_c = rows[add].astype(np.float64).mean(axis=0)
        sub_c = rows[int(rng.integers(N))].astype(np.float64) if with_sub else None
        sub_thr = 0.0
        if with_sub:   # angular: the default; euclidean: the median distance, so that both decisions occur
            sub_thr = 0.2 if space == "cosine" else float(np.median(np.linalg.norm(rows[:2000] - sub_c, axis=1)))
        n = 3 * n_results
        k = sp.query_size(n, True, N)
        listed, knn_gap = osa.knn_list(rows, space, add_c, k)
        keyed = osa.keys(table, listed)
        cfg = {"VOYAGER_METRIC": "angular" if space == "cosine" else "euclidean", "THRESHOLD_COSINE": 0.01,
               "THRESHOLD_EUCLIDEAN": 0.15, "LOOKBACK": lookback, "BATCH": 50, "MAX_SONGS_PER_ARTIST": cap,
               "ELIMINATE_DUPLICATES": True}
        excl = {f"item{a}" for a in add}
        o = osa.candidates(rows, keyed, cfg, metric, add_c, sub_c, sub_thr, listed, excl, n, False)
        ids = idx.query(np.asarray(add_c, np.float32), k)[0].astype(np.int64)
        items = [f"item{i}" for i in ids]
        sig, raw = dense_keys(table, items)
        pos, status, dsub, dadd, got_rows = idx.alchemy(_alchemy_cfg(space, n, lookback, cap, sub_thr), add_c, sub_c,
                                                        ids, sig[0], raw[0], sig[1], sorted(add), rows=True)
        margins = (knn_gap > KNN_BOUND and o["filter_gap"] > thr_bound(cfg) and o["sub_gap"] > DECISION_BOUND)
        if not margins:
            continue
        checked += 1
        assert items == listed
        chain = [items[p] for p in pos]
        assert chain == o["chain"], (n_results, with_sub, lookback, cap)
        assert [items[p] for p, s in zip(pos, status) if s == 1][:n] == o["kept"]
        assert [items[p] for p, s in zip(pos, status) if s == 2] == o["filtered_out"]
        assert all(s == 0 for p, s in zip(pos, status) if items[p] in excl)
        for p, s, ds, da in zip(pos, status, dsub, dadd):
            it = items[p]
            if s == 1:
                assert abs(da - o["distances"][it]) <= dist_tol(o["distances"][it], metric)
            if s and sub_c is not None:
                assert abs(ds - o["dsub"][it]) <= dist_tol(o["dsub"][it], metric)
            if s:
                assert np.array_equal(got_rows[list(pos).index(p)], rows[int(it[4:])])
    assert checked >= 4


def dense_keys(table, items):
    """The drop-in's dense keys: ((signature keys, their count), (raw-author keys, their count))."""
    from audiomuse_ai_b200 import song_path as sp
    sig, raw = sp.Keys(), sp.Keys()
    s = [sig(sp.signature(table[i])) if i in table else -1 for i in items]
    r = [raw(table[i]["author"]) if i in table and table[i].get("author") else -1 for i in items]
    return (s, len(sig)), (r, len(raw))


def test_two_calls_are_bit_identical():
    c = next(c for c in gen.load() if c["name"] == "n200_sub")
    rows = gen.stored_rows(c["library"], c["space"])
    idx = _index(gen.library(c["library"]), c["space"], rows)
    table = gen.score_table(c["library"])
    add_c, sub_c = rows[41].astype(np.float64), rows[950].astype(np.float64)
    ids = idx.query(np.asarray(add_c, np.float32), 3000)[0].astype(np.int64)
    sig, raw = dense_keys(table, [f"item{i}" for i in ids])
    outs = [idx.alchemy(_alchemy_cfg("cosine", 600, 1, 3, 0.2), add_c, sub_c, ids, sig[0], raw[0], sig[1], [41, 950],
                        rows=True) for _ in range(2)]
    assert len(outs[0][0]) > 500
    for a, b in zip(*outs):
        assert a.dtype == b.dtype and a.tobytes() == b.tobytes()
