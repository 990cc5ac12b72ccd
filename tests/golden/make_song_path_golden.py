#!/usr/bin/env python
"""Goldens of the reference's Song Path, so that the tests need no reference checkout.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_song_path_golden.py
    # writes tests/golden/song_path_golden.npz

Runs the reference's find_path_between_songs (tasks/path_manager.py:320-557), UNMODIFIED, over seeded libraries, a
recording brute-force index and an in-memory metadata table, and records per case: the configuration, the float32
vector and k of every index.query its jobs made, the job sequence (k, num_to_find and the songs found, merges
included), the two heuristic neighbour lists, the final ids in order and the total distance, and the float64
oracle's (oracle/song_path.py) smallest deciding gaps.  Item ids are "item<index id>".

Cases cover Lreq in {3, 5, 25, 60}, path_fix_size on and off, both PATH_DISTANCE_METRICs and VOYAGER_METRICs,
MAX_SONGS_PER_ARTIST in {0, 1, 3}, DUPLICATE_DISTANCE_CHECK_LOOKBACK in {0, 1, 3}, eliminate_duplicates on and off,
exact duplicate rows, titles repeated under case and whitespace variants, None and "" authors, a single-artist region
and wide duplicate thresholds that make jobs fail and merge (the last one included), and a library smaller than
the query size.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402
from tests.golden import make_radius_walk_golden as rwg  # noqa: E402

GOLDEN = os.path.join(HERE, "song_path_golden.npz")
D = 64
LIBRARIES = {"main": (3000, 61), "small": (40, 62)}
BATCH = 50   # voyager_manager.BATCH_SIZE_VECTOR_OPS


def library(name):
    """Seeded [N, 64] float32 embeddings in 30 clusters; rows 2000-2029 are exact copies of rows 100-129 (main)."""
    n, seed = LIBRARIES[name]
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((30, D)).astype(np.float32)
    x = (base[rng.integers(0, 30, n)] + 0.5 * rng.standard_normal((n, D)).astype(np.float32)).astype(np.float32)
    if n > 2030:
        x[2000:2030] = x[100:130]
    return x


def stored_rows(name, space):
    """The rows the index stores: unit-normalised for the cosine space."""
    x = library(name)
    if space == "cosine":
        from oracle import knn as oknn
        return oknn.normalize_rows(x)
    return x


def score_table(name):
    """rh.make_score_table, plus: prolific artists, None and "" authors, every 19th title repeating its neighbour's
    under case and whitespace changes, and rows 2400-2599 all by one artist (a region the artist caps starve)."""
    n, seed = LIBRARIES[name]
    t = rh.make_score_table(n, seed)
    for i in range(n):
        r = t[f"item{i}"]
        if 2400 <= i < 2600:
            r["author"] = "Single Artist"
        elif i % 7 == 0:
            r["author"] = "Prolific A"
        elif i % 11 == 0:
            r["author"] = "prolific a "
        elif i % 23 == 5:
            r["author"] = None
        elif i % 29 == 3:
            r["author"] = ""
        if i % 19 == 2 and i > 0:
            prev = t[f"item{i - 1}"]
            r["title"] = "  " + prev["title"].upper() + " "
            r["author"] = None if prev["author"] is None else prev["author"].lower() + "  "
    return t


# name, library, space, PATH_DISTANCE_METRIC, Lreq, path_fix_size, MAX_SONGS_PER_ARTIST, LOOKBACK,
# eliminate_duplicates, THRESHOLD_COSINE, THRESHOLD_EUCLIDEAN, start, end
CASES = [
    ("ang_l3", "main", "cosine", "angular", 3, False, 3, 1, True, 0.01, 0.15, "item10", "item20"),
    ("ang_l5_fix", "main", "cosine", "angular", 5, True, 3, 1, True, 0.01, 0.15, "item11", "item21"),
    ("ang_l25", "main", "cosine", "angular", 25, False, 3, 1, True, 0.01, 0.15, "item12", "item22"),
    ("ang_l25_fix", "main", "cosine", "angular", 25, True, 3, 1, True, 0.01, 0.15, "item13", "item23"),
    ("ang_l60_fix", "main", "cosine", "angular", 60, True, 3, 1, True, 0.01, 0.15, "item14", "item24"),
    ("ang_l60", "main", "cosine", "angular", 60, False, 3, 1, True, 0.01, 0.15, "item15", "item25"),
    ("ang_l25_fix_cap0", "main", "cosine", "angular", 25, True, 0, 1, True, 0.01, 0.15, "item16", "item26"),
    ("ang_l25_fix_cap1", "main", "cosine", "angular", 25, True, 1, 1, True, 0.01, 0.15, "item17", "item27"),
    ("ang_l25_lb0", "main", "cosine", "angular", 25, True, 3, 0, True, 0.01, 0.15, "item18", "item28"),
    ("ang_l25_lb3", "main", "cosine", "angular", 25, True, 3, 3, True, 0.01, 0.15, "item19", "item29"),
    ("ang_l25_nodedupe", "main", "cosine", "angular", 25, True, 3, 1, False, 0.01, 0.15, "item30", "item40"),
    ("ang_l25_nodedupe_cap1", "main", "cosine", "angular", 25, False, 1, 1, False, 0.01, 0.15, "item31", "item41"),
    ("ang_dup_rows", "main", "cosine", "angular", 25, True, 3, 1, True, 0.01, 0.15, "item105", "item2010"),
    ("ang_single_artist_fix", "main", "cosine", "angular", 25, True, 1, 1, True, 0.01, 0.15, "item2400", "item2599"),
    ("ang_single_artist", "main", "cosine", "angular", 25, False, 1, 1, True, 0.01, 0.15, "item2401", "item2598"),
    ("ang_wide_thr_fix", "main", "cosine", "angular", 25, True, 3, 3, True, 0.19, 0.15, "item32", "item42"),
    ("ang_wide_thr_l60_fix", "main", "cosine", "angular", 60, True, 1, 3, True, 0.21, 0.15, "item33", "item43"),
    ("ang_path_euclid", "main", "cosine", "euclidean", 25, True, 3, 1, True, 0.01, 0.15, "item34", "item44"),
    ("ang_path_euclid_wide", "main", "cosine", "euclidean", 25, True, 3, 3, True, 0.01, 0.9, "item35", "item45"),
    ("euc_l3", "main", "euclidean", "euclidean", 3, True, 3, 1, True, 0.01, 0.15, "item50", "item60"),
    ("euc_l25", "main", "euclidean", "euclidean", 25, False, 3, 1, True, 0.01, 0.15, "item51", "item61"),
    ("euc_l25_fix", "main", "euclidean", "euclidean", 25, True, 3, 1, True, 0.01, 0.15, "item52", "item62"),
    ("euc_l60_fix_cap1", "main", "euclidean", "euclidean", 60, True, 1, 3, True, 0.01, 0.15, "item53", "item63"),
    ("euc_path_angular", "main", "euclidean", "angular", 25, True, 3, 1, True, 0.01, 0.15, "item54", "item64"),
    ("euc_wide_thr_fix", "main", "euclidean", "euclidean", 25, True, 3, 3, True, 0.01, 3.0, "item55", "item65"),
    ("euc_nodedupe_lb0", "main", "euclidean", "angular", 25, False, 0, 0, False, 0.01, 0.15, "item56", "item66"),
    ("small_fix", "small", "cosine", "angular", 25, True, 3, 1, True, 0.01, 0.15, "item1", "item2"),
    ("small", "small", "cosine", "angular", 5, False, 3, 1, True, 0.01, 0.15, "item3", "item4"),
    ("small_euc_fix", "small", "euclidean", "euclidean", 25, True, 1, 1, True, 0.01, 0.15, "item5", "item6"),
]


class EuclideanRecordingIndex(rwg.EuclideanRecordingIndex):
    """voyager's Euclidean space over the stored rows, recording its queries like rh.RecordingIndex."""

    def query(self, vector, k):
        ids, dist = super().query(vector, k)
        self.trace.append({"op": "query", "vector": np.asarray(vector, dtype=np.float32).copy(), "k": int(k)})
        return ids, dist


def case_config(case):
    name, lib, space, pmetric, Lreq, fix, cap, lookback, ed, thr_cos, thr_euc, start, end = case
    return {"VOYAGER_METRIC": "angular" if space == "cosine" else "euclidean", "PATH_DISTANCE_METRIC": pmetric,
            "MAX_SONGS_PER_ARTIST": cap, "LOOKBACK": lookback, "THRESHOLD_COSINE": thr_cos,
            "THRESHOLD_EUCLIDEAN": thr_euc, "ELIMINATE_DUPLICATES": ed, "BATCH": BATCH}


def configure(vm, pm, cfg):
    """The configuration both modules read at call time."""
    for mod in (vm, pm):
        mod.MAX_SONGS_PER_ARTIST = cfg["MAX_SONGS_PER_ARTIST"]
        mod.DUPLICATE_DISTANCE_CHECK_LOOKBACK = cfg["LOOKBACK"]
        mod.DUPLICATE_DISTANCE_THRESHOLD_COSINE = cfg["THRESHOLD_COSINE"]
        mod.DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN = cfg["THRESHOLD_EUCLIDEAN"]
        mod.VOYAGER_METRIC = cfg["VOYAGER_METRIC"]
    vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT = cfg["ELIMINATE_DUPLICATES"]
    vm.BATCH_SIZE_VECTOR_OPS = cfg["BATCH"]
    pm.PATH_DISTANCE_METRIC = cfg["PATH_DISTANCE_METRIC"]


def main():
    db = rh.FakeDB()
    ref = rh.load_reference(rwg.types_voyager(), db)
    vm = ref.vm
    pm = rh._load("tasks.path_manager", "tasks/path_manager.py")
    sys.modules["app_helper"].get_tracks_by_ids = lambda ids: [dict(db.score[i]) for i in ids if i in db.score]
    rec = {}
    orig_job, orig_nb = pm._find_best_songs_for_job, pm.find_nearest_neighbors_by_id

    def rec_job(centroid_vec, *a, k_search=10, num_to_find=1, **kw):
        t0 = len(vm.voyager_index.trace)
        out = orig_job(centroid_vec, *a, k_search=k_search, num_to_find=num_to_find, **kw)
        rec["queries"] += [(e["vector"], e["k"]) for e in vm.voyager_index.trace[t0:] if e["op"] == "query"]
        rec["jobs"].append((k_search, num_to_find, [s["item_id"] for s in out]))
        return out

    def rec_nb(item_id, **kw):
        out = orig_nb(item_id, **kw)
        rec["neighbours"].append([n["item_id"] for n in out or []])
        return out

    pm._find_best_songs_for_job, pm.find_nearest_neighbors_by_id = rec_job, rec_nb
    from oracle import song_path as osp
    cases = []
    for case in CASES:
        name, lib, space, pmetric, Lreq, fix, cap, lookback, ed, thr_cos, thr_euc, start, end = case
        cfg = case_config(case)
        rows = stored_rows(lib, space)
        db.score = score_table(lib)
        vm.voyager_index = rh.RecordingIndex(library(lib)) if space == "cosine" else EuclideanRecordingIndex(rows)
        assert np.array_equal(vm.voyager_index.rows, rows)
        vm.id_map = {i: f"item{i}" for i in range(len(rows))}
        vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
        configure(vm, pm, cfg)
        vm._get_cached_vector.cache_clear()
        rec.update(queries=[], jobs=[], neighbours=[])
        details, total = pm.find_path_between_songs(start, end, Lreq, path_fix_size=fix)
        path = [d["item_id"] for d in details]
        o = osp.song_path(rows, space, db.score, cfg, start, end, Lreq, fix, *rec["neighbours"])
        assert o["path"] == path and o["jobs"] == rec["jobs"], name
        assert len(o["queries"]) == len(rec["queries"]) and all(
            np.array_equal(a[0], b[0]) and a[1] == b[1] for a, b in zip(o["queries"], rec["queries"])), name
        cases.append({"name": name, "library": lib, "space": space, "config": cfg, "Lreq": Lreq, "path_fix_size": fix,
                      "start": start, "end": end, "neighbours": rec["neighbours"], "jobs": rec["jobs"], "path": path,
                      "total": float(total), "thr_gap": o["thr_gap"], "knn_gap": o["knn_gap"],
                      "queries": rec["queries"]})
        merges = sum(1 for k, need, f in rec["jobs"] if not f)
        print(f"{name:24s} {len(path):3d} of {Lreq:3d} songs, {len(rec['jobs']):3d} jobs, {merges:2d} failed, "
              f"total {float(total):.5f}, gaps thr {o['thr_gap']:.2e} knn {o['knn_gap']:.2e}")
    save(cases)


def save(cases):
    """One compressed .npz: the cases as a JSON string, each case's query vectors f32[nq, d] beside it."""
    out = {}
    meta = []
    for i, c in enumerate(cases):
        out[f"{i}_queries"] = np.array([q for q, _ in c["queries"]], dtype=np.float32).reshape(-1, D)
        meta.append(dict({k: v for k, v in c.items() if k != "queries"}, query_k=[int(k) for _, k in c["queries"]]))
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(GOLDEN, **out)


def load(path=GOLDEN):
    """The cases as main() recorded them; "queries" is the list of (f32 vector, k)."""
    g = np.load(path)
    cases = json.loads(str(g["meta"]))
    for i, c in enumerate(cases):
        c["queries"] = list(zip(g[f"{i}_queries"], c.pop("query_k")))
        c["jobs"] = [(k, need, list(f)) for k, need, f in c["jobs"]]
    return cases


if __name__ == "__main__":
    main()
