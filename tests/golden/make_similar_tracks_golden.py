#!/usr/bin/env python
"""Goldens of the reference's plain similar-tracks requests, so that the tests need no reference checkout.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_similar_tracks_golden.py
    # writes tests/golden/similar_tracks_golden.npz

Runs the reference's find_nearest_neighbors_by_id (radius_similarity off), find_nearest_neighbors_by_vector and
get_max_distance_for_id (tasks/voyager_manager.py:1372-1702), UNMODIFIED, over the Song Path goldens' seeded libraries
and metadata table (duplicate rows, case and whitespace title variants, None and "" authors), with other_features
strings that vary: all six moods, some keys only, extra keys and spaces, malformed values ("danceable:abc"), "" and
None.  A recording brute-force index answers the queries.  Per case it records the configuration, the request and the
returned list or dict, checked against the float64 oracle (oracle/similar_tracks.py), and the oracle's deciding gaps.
Item ids are "item<index id>".

Above BATCH_SIZE_VECTOR_OPS (50) candidates the reference's mood filter computes its batches on a thread pool and
collects them with as_completed, which yields the futures in set order: its own output order is then not
deterministic.  This generator replaces vm._get_thread_pool and vm.as_completed with in-order versions (each batch
runs when it is submitted, and the futures come back in submission order), so the recorded lists keep k-NN order, the
order the drop-in and the oracle keep.

Cases cover both VOYAGER_METRICs, lookback 0 and 1, lists longer than 50 (the batched filter window and the mood
filter's threaded branch), caps 0, 1 and 3, eliminate_duplicates and mood_similarity on and off, n in {1, 10, 100,
500}, a library smaller than the query, a target without mood features, and max-distance targets whose farthest rows
tie: exact duplicate rows, and rows at the same float32 distance but different float64 ones.
"""
import json
import os
import sys
from concurrent.futures import Future

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402
from tests.golden import make_radius_walk_golden as rwg  # noqa: E402
from tests.golden import make_song_path_golden as spg  # noqa: E402

GOLDEN = os.path.join(HERE, "similar_tracks_golden.npz")
D = spg.D
LIBRARIES = dict(spg.LIBRARIES, ties=(40, 63), single=(1, 64))
MOODS = ["danceable", "aggressive", "happy", "party", "relaxed", "sad"]


def library(name):
    """The Song Path libraries; "ties": row 0 with rows 2 and 3 at -row 0 and row 1 at -row 0 plus 1e-4 in one
    coordinate (its squared euclidean distance to row 0 rounds to the same float32 as theirs), the rest near row 0;
    "single": one row."""
    if name in spg.LIBRARIES:
        return spg.library(name)
    n, seed = LIBRARIES[name]
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, D)).astype(np.float32)
    if name == "ties":
        e = np.zeros(D, np.float32)
        e[0] = 1.0
        x = (e + 0.1 * rng.standard_normal((n, D))).astype(np.float32)
        x[0] = e
        x[1] = -e
        x[1, 1] = 1e-4
        x[2] = x[3] = -e
    return x


def stored_rows(name, space):
    x = library(name)
    if space == "cosine":
        from oracle import knn as oknn
        return oknn.normalize_rows(x)
    return x


def other_features(i, rng):
    """Row i's other_features: all six moods near 0.5 (most rows), some keys only, extra keys and spaces, a malformed
    value, "" or None."""
    vals = np.round(0.5 + 0.12 * rng.standard_normal(6), 4)
    full = ",".join(f"{k}:{v}" for k, v in zip(MOODS, vals))
    if i % 31 == 7:
        return None
    if i % 29 == 11:
        return ""
    if i % 23 == 13:
        return "danceable:abc,happy:0.5"
    if i % 13 == 4:
        return ",".join(f"{k}:{v}" for k, v in zip(MOODS[::2], vals[::2]))
    if i % 11 == 6:
        return f" tempo_class : 0.3 ,{full.replace(',', ' , ')}, no_colon_here"
    return full


def score_table(name):
    n, seed = LIBRARIES[name]
    t = spg.score_table(name) if name in spg.LIBRARIES else rh.make_score_table(n, seed)
    rng = np.random.default_rng(seed + 1000)
    for i in range(n):
        t[f"item{i}"]["other_features"] = other_features(i, rng)
    return t


def query_vector(lib, space, row, seed):
    """A float32 vector near stored row `row`."""
    x = stored_rows(lib, space).astype(np.float64)
    return (x[row % len(x)] + 0.05 * np.random.default_rng(seed).standard_normal(D)).astype(np.float32)


BASE = {"VOYAGER_METRIC": "angular", "THRESHOLD_COSINE": 0.01, "THRESHOLD_EUCLIDEAN": 0.15, "LOOKBACK": 1,
        "BATCH": 50, "MAX_SONGS_PER_ARTIST": 3, "ELIMINATE_DUPLICATES": True, "MOOD_SIMILARITY_ENABLE": False,
        "MOOD_SIMILARITY_THRESHOLD": 0.15}


def C(**kw):
    return dict(BASE, **kw)


EUC = dict(VOYAGER_METRIC="euclidean")
# kind, name, library, space, config, request
CASES = [
    ("by_id", "id_n10", "main", "cosine", C(), dict(target="item10", n=10)),
    ("by_id", "id_n1", "main", "cosine", C(), dict(target="item11", n=1)),
    ("by_id", "id_n100_mood", "main", "cosine", C(), dict(target="item12", n=100, mood_similarity=True)),
    ("by_id", "id_n100_mood_config", "main", "cosine", C(MOOD_SIMILARITY_ENABLE=True), dict(target="item9", n=100)),
    ("by_id", "id_n500_mood", "main", "cosine", C(), dict(target="item14", n=500, mood_similarity=True)),
    ("by_id", "id_n500", "main", "cosine", C(), dict(target="item15", n=500)),
    ("by_id", "id_n100_nodedupe", "main", "cosine", C(), dict(target="item16", n=100, eliminate_duplicates=False)),
    ("by_id", "id_n100_nodedupe_mood", "main", "cosine", C(MOOD_SIMILARITY_THRESHOLD=0.3),
     dict(target="item17", n=100, eliminate_duplicates=False, mood_similarity=True)),
    ("by_id", "id_mood_off_explicit", "main", "cosine", C(MOOD_SIMILARITY_ENABLE=True),
     dict(target="item18", n=10, mood_similarity=False)),
    ("by_id", "id_target_without_moods", "main", "cosine", C(), dict(target="item38", n=100, mood_similarity=True)),
    ("by_id", "id_target_malformed_moods", "main", "cosine", C(), dict(target="item36", n=10, mood_similarity=True)),
    ("by_id", "id_lookback0", "main", "cosine", C(LOOKBACK=0), dict(target="item19", n=100, mood_similarity=True)),
    ("by_id", "id_cap0", "main", "cosine", C(MAX_SONGS_PER_ARTIST=0), dict(target="item20", n=100)),
    ("by_id", "id_cap1", "main", "cosine", C(MAX_SONGS_PER_ARTIST=1), dict(target="item2401", n=100)),
    ("by_id", "id_dup_rows", "main", "cosine", C(), dict(target="item105", n=100)),
    ("by_id", "id_wide_thr", "main", "cosine", C(THRESHOLD_COSINE=0.2, MAX_SONGS_PER_ARTIST=1),
     dict(target="item21", n=100, mood_similarity=True)),
    ("by_id", "id_euc", "main", "euclidean", C(**EUC), dict(target="item50", n=10)),
    ("by_id", "id_euc_n100_mood", "main", "euclidean", C(**EUC, THRESHOLD_EUCLIDEAN=3.0),
     dict(target="item51", n=100, mood_similarity=True)),
    ("by_id", "id_euc_n500_cap1", "main", "euclidean", C(**EUC, MAX_SONGS_PER_ARTIST=1, THRESHOLD_EUCLIDEAN=3.0),
     dict(target="item52", n=500)),
    ("by_id", "id_euc_lookback0_nodedupe", "main", "euclidean", C(**EUC, LOOKBACK=0),
     dict(target="item53", n=100, eliminate_duplicates=False)),
    ("by_id", "id_small", "small", "cosine", C(), dict(target="item1", n=100, mood_similarity=True)),
    ("by_id", "id_small_n10", "small", "euclidean", C(**EUC), dict(target="item2", n=10)),
    ("by_id", "id_unknown", "small", "cosine", C(), dict(target="item999", n=10)),
    ("by_vector", "vec_n10", "main", "cosine", C(), dict(row=30, seed=1, n=10)),
    ("by_vector", "vec_n1", "main", "cosine", C(), dict(row=31, seed=2, n=1)),
    ("by_vector", "vec_n100", "main", "cosine", C(), dict(row=32, seed=3, n=100)),
    ("by_vector", "vec_n500", "main", "cosine", C(), dict(row=33, seed=4, n=500)),
    ("by_vector", "vec_n100_nodedupe", "main", "cosine", C(), dict(row=34, seed=5, n=100, eliminate_duplicates=False)),
    ("by_vector", "vec_cap0", "main", "cosine", C(MAX_SONGS_PER_ARTIST=0), dict(row=35, seed=6, n=100)),
    ("by_vector", "vec_cap1_wide", "main", "cosine", C(MAX_SONGS_PER_ARTIST=1, THRESHOLD_COSINE=0.2),
     dict(row=2410, seed=7, n=100)),
    ("by_vector", "vec_lookback0", "main", "cosine", C(LOOKBACK=0), dict(row=36, seed=8, n=100)),
    ("by_vector", "vec_dup_rows", "main", "cosine", C(), dict(row=110, seed=9, n=100)),
    ("by_vector", "vec_euc", "main", "euclidean", C(**EUC), dict(row=60, seed=10, n=10)),
    ("by_vector", "vec_euc_n500", "main", "euclidean", C(**EUC, THRESHOLD_EUCLIDEAN=3.0), dict(row=61, seed=11, n=500)),
    ("by_vector", "vec_euc_cap1_nodedupe", "main", "euclidean", C(**EUC, MAX_SONGS_PER_ARTIST=1),
     dict(row=62, seed=12, n=100, eliminate_duplicates=False)),
    ("by_vector", "vec_small", "small", "cosine", C(), dict(row=3, seed=13, n=100)),
    ("max", "max_cos", "main", "cosine", C(), dict(target="item10")),
    ("max", "max_cos_dup", "main", "cosine", C(), dict(target="item2000")),
    ("max", "max_euc", "main", "euclidean", C(**EUC), dict(target="item50")),
    ("max", "max_small", "small", "cosine", C(), dict(target="item5")),
    ("max", "max_ties_euc", "ties", "euclidean", C(**EUC), dict(target="item0")),
    ("max", "max_ties_cos", "ties", "cosine", C(), dict(target="item0")),
    ("max", "max_single", "single", "cosine", C(), dict(target="item0")),
    ("max", "max_unknown", "small", "cosine", C(), dict(target="item999")),
]


class _Cursor(rh.FakeCursor):
    """rh.FakeCursor, plus the mood filter's read of its target's other_features (voyager_manager.py:729)."""

    def execute(self, sql, params=None):
        if " ".join(sql.split()) == "SELECT other_features FROM score WHERE item_id = %s":
            r = self.db.score.get(params[0])
            self._rows = [rh.DictRow({"other_features": r.get("other_features")})] if r else []
            return
        super().execute(sql, params)


class _DB(rh.FakeDB):
    def cursor(self, cursor_factory=None, **kw):
        return _Cursor(self, cursor_factory is not None)


class _Now:
    """A thread pool that runs each batch when it is submitted."""

    def submit(self, fn, *a, **k):
        f = Future()
        f.set_result(fn(*a, **k))
        return f


def configure(vm, cfg):
    vm.VOYAGER_METRIC = cfg["VOYAGER_METRIC"]
    vm.DUPLICATE_DISTANCE_THRESHOLD_COSINE = cfg["THRESHOLD_COSINE"]
    vm.DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN = cfg["THRESHOLD_EUCLIDEAN"]
    vm.DUPLICATE_DISTANCE_CHECK_LOOKBACK = cfg["LOOKBACK"]
    vm.BATCH_SIZE_VECTOR_OPS = cfg["BATCH"]
    vm.MAX_SONGS_PER_ARTIST = cfg["MAX_SONGS_PER_ARTIST"]
    vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT = cfg["ELIMINATE_DUPLICATES"]
    vm.MOOD_SIMILARITY_ENABLE = cfg["MOOD_SIMILARITY_ENABLE"]
    vm.MOOD_SIMILARITY_THRESHOLD = cfg["MOOD_SIMILARITY_THRESHOLD"]
    vm.SIMILARITY_RADIUS_DEFAULT = False


def run_oracle(osim, case):
    """The oracle's answer and gaps for a recorded (or to be recorded) case."""
    kind, lib, space, cfg, req = case["kind"], case["library"], case["space"], case["config"], case["request"]
    rows, table = stored_rows(lib, space), score_table(lib)
    if kind == "by_id":
        out, fg, kg = osim.by_id(rows, space, table, cfg, req["target"], req["n"], req.get("eliminate_duplicates"),
                                 req.get("mood_similarity"))
        return {"result": out, "filter_gap": fg, "knn_gap": kg}
    if kind == "by_vector":
        out, fg, kg = osim.by_vector(rows, space, table, cfg, np.asarray(req["vector"], np.float32), req["n"],
                                     req.get("eliminate_duplicates"))
        return {"result": out, "filter_gap": fg, "knn_gap": kg}
    if int(req["target"][4:]) >= len(rows):
        return {"result": None, "far_gap": np.inf}
    out, gap = osim.max_distance(rows, space, req["target"])
    return {"result": out, "far_gap": gap}


def main():
    db = _DB()
    ref = rh.load_reference(rwg.types_voyager(), db)
    vm = ref.vm
    vm._get_thread_pool = lambda: _Now()
    vm.as_completed = lambda futures: iter(list(futures))
    from oracle import similar_tracks as osim
    cases = []
    for kind, name, lib, space, cfg, req in CASES:
        rows = stored_rows(lib, space)
        db.score = score_table(lib)
        vm.voyager_index = (rh.RecordingIndex(library(lib)) if space == "cosine"
                            else rwg.EuclideanRecordingIndex(rows))
        assert np.array_equal(vm.voyager_index.rows, rows)
        vm.id_map = {i: f"item{i}" for i in range(len(rows))}
        vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
        configure(vm, cfg)
        vm._get_cached_vector.cache_clear()
        req = dict(req)
        if kind == "by_id":
            out = vm.find_nearest_neighbors_by_id(req["target"], n=req["n"],
                                                  eliminate_duplicates=req.get("eliminate_duplicates"),
                                                  mood_similarity=req.get("mood_similarity"), radius_similarity=False)
        elif kind == "by_vector":
            req["vector"] = [float(v) for v in query_vector(lib, space, req.pop("row"), req.pop("seed"))]
            out = vm.find_nearest_neighbors_by_vector(np.asarray(req["vector"], np.float32), n=req["n"],
                                                      eliminate_duplicates=req.get("eliminate_duplicates"))
        else:
            out = vm.get_max_distance_for_id(req["target"])
        case = {"kind": kind, "name": name, "library": lib, "space": space, "config": cfg, "request": req,
                "result": out}
        o = run_oracle(osim, case)
        assert o.pop("result") == out, name
        case.update(o)
        cases.append(case)
        size = len(out) if isinstance(out, list) else out
        print(f"{name:28s} {str(size):60s} {({k: f'{v:.2e}' for k, v in o.items()})}")
    np.savez_compressed(GOLDEN, meta=np.array(json.dumps(cases)))


def load(path=GOLDEN):
    return json.loads(str(np.load(path)["meta"]))


if __name__ == "__main__":
    main()
