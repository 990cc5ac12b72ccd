#!/usr/bin/env python
"""Goldens of the reference's similar-tracks radius walk, so that the tests need no reference checkout.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_radius_walk_golden.py
    # writes tests/golden/radius_walk_golden.npz

Runs the reference's find_nearest_neighbors_by_id(..., radius_similarity=True) (tasks/voyager_manager.py:1372-1491),
UNMODIFIED, over seeded libraries and an in-memory metadata table with prolific artists and None / "" authors, and
records what its two walk functions saw and returned: _radius_walk_get_candidates (:842-938, the candidate ids it
received and kept) and _execute_radius_walk (:941-1367, its candidate list in order -- index id, author, anchor
distance -- and its playlist).  Item ids are "item<index id>", so only index ids are stored.  Cases cover n in
{1, 10, 25, 49, 50, 51, 100, 200}, eliminate_duplicates on and off, MAX_SONGS_PER_ARTIST in {0, 1, 3}, the angular and euclidean metrics, a pool
smaller than n, exact duplicate rows (they tie on the anchor distance) and a candidate missing from reverse_id_map.
Each case also stores the smallest float64 gap that decided an ordering (oracle/radius_walk.py in float64 mode):
between neighbours of the anchor-distance sort and between each greedy step's best score and its runner-up.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402

GOLDEN = os.path.join(HERE, "radius_walk_golden.npz")
D = 200
LIBRARIES = {"main": (2400, 51), "small": (150, 52)}


def library(name):
    """Seeded [N, 200] float32 embeddings: clusters, and rows 2000-2029 exact copies of rows 100-129 (main only)."""
    n, seed = LIBRARIES[name]
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((40, D)).astype(np.float32)
    x = (base[rng.integers(0, 40, n)] + 0.45 * rng.standard_normal((n, D)).astype(np.float32)).astype(np.float32)
    if n > 2030:
        x[2000:2030] = x[100:130]
    return x


def stored_rows(name, space):
    """The rows the index stores: unit-normalised for the cosine space (as voyager and RecordingIndex store them)."""
    x = library(name)
    if space == "cosine":
        from oracle import knn as oknn
        return oknn.normalize_rows(x)
    return x


def score_table(name):
    """rh.make_score_table plus two prolific artists and falsy authors (None and "")."""
    n, seed = LIBRARIES[name]
    t = rh.make_score_table(n, seed)
    for i in range(n):
        r = t[f"item{i}"]
        if i % 7 == 0:
            r["author"] = "Prolific A"
        elif i % 11 == 0:
            r["author"] = "Prolific B"
        elif i % 23 == 5:
            r["author"] = None
        elif i % 29 == 3:
            r["author"] = ""
    return t


# name, library, index space, VOYAGER_METRIC, n, eliminate_duplicates, MAX_SONGS_PER_ARTIST, lookback, target, missing
CASES = [
    ("cos_n1", "main", "cosine", "angular", 1, True, 3, 1, "item300", None),
    ("cos_n10", "main", "cosine", "angular", 10, True, 3, 1, "item301", None),
    ("cos_n25", "main", "cosine", "angular", 25, True, 3, 1, "item302", None),
    ("cos_n49", "main", "cosine", "angular", 49, True, 3, 1, "item303", None),
    ("cos_n50", "main", "cosine", "angular", 50, True, 3, 1, "item304", None),
    ("cos_n51", "main", "cosine", "angular", 51, True, 3, 1, "item305", None),
    ("cos_n100", "main", "cosine", "angular", 100, True, 3, 1, "item306", None),
    ("cos_n200", "main", "cosine", "angular", 200, True, 3, 1, "item307", None),
    ("cos_n25_nodedupe", "main", "cosine", "angular", 25, False, 3, 1, "item308", None),
    ("cos_n100_nodedupe", "main", "cosine", "angular", 100, False, 3, 1, "item309", None),
    ("cos_n50_cap0", "main", "cosine", "angular", 50, True, 0, 1, "item310", None),
    ("cos_n51_cap1", "main", "cosine", "angular", 51, True, 1, 1, "item311", None),
    ("cos_n100_cap1", "main", "cosine", "angular", 100, True, 1, 1, "item312", None),
    ("cos_n100_duplicate_rows", "main", "cosine", "angular", 100, True, 3, 0, "item105", None),
    ("cos_n200_duplicate_rows_nodedupe", "main", "cosine", "angular", 200, False, 3, 0, "item2010", None),
    ("cos_n25_missing_id", "main", "cosine", "angular", 25, True, 3, 0, "item313", 4),
    ("cos_small_pool", "small", "cosine", "angular", 200, True, 3, 1, "item7", None),
    ("euc_n10", "main", "euclidean", "euclidean", 10, True, 3, 1, "item400", None),
    ("euc_n51_cap1", "main", "euclidean", "euclidean", 51, True, 1, 1, "item401", None),
    ("euc_n50_nodedupe", "main", "euclidean", "euclidean", 50, False, 3, 1, "item402", None),
    ("euc_n100", "main", "euclidean", "euclidean", 100, True, 3, 1, "item403", None),
    ("euc_n200", "main", "euclidean", "euclidean", 200, True, 3, 1, "item404", None),
    ("euc_small_pool", "small", "euclidean", "euclidean", 100, True, 3, 1, "item8", None),
]


class EuclideanRecordingIndex(rh.RecordingIndex):
    """voyager's Euclidean space: raw stored rows, exact ascending L2 order (lower id first on ties)."""

    def __init__(self, rows):
        super().__init__(rows)
        self.rows = np.asarray(rows, dtype=np.float32)

    def query(self, vector, k):
        q = np.asarray(vector, dtype=np.float32)
        ids, dist = self._oknn.topk(self.rows, q[np.newaxis, :], int(k), metric=self._oknn.EUCLIDEAN)
        return ids[0].astype(np.uint64), dist[0].astype(np.float32)


def case_gaps(rows, target_vid, walk_in, metric, n, ed, cap):
    from oracle import radius_walk as orw
    r = orw.radius_walk([rows[v] for v in walk_in["vid"]], rows[target_vid], walk_in["author"], n, ed, cap, metric,
                        mode="float64")
    return r["sort_gap"], r["score_gap"]


def main():
    db = rh.FakeDB()
    ref = rh.load_reference(types_voyager(), db)
    vm = ref.vm
    seen = {}

    orig_cand, orig_walk = vm._radius_walk_get_candidates, vm._execute_radius_walk

    def vid(item_id):   # item ids are "item<index id>"
        return int(item_id[4:])

    def rec_cand(**kw):
        out = orig_cand(**kw)
        seen["cand_in"] = [vid(r["item_id"]) for r in kw["initial_results"]]
        seen["cand_out"] = [vid(c["item_id"]) for c in out]
        return out

    def rec_walk(**kw):
        cd = kw["candidate_data"]   # the walk sorts it in place: record it first
        seen["walk_in"] = {"vid": [vid(c["item_id"]) for c in cd], "author": [c["author"] for c in cd],
                           "dist_anchor": [c["dist_anchor"] for c in cd]}
        out = orig_walk(**kw)
        seen["walk_out"] = {"vid": [vid(r["item_id"]) for r in out], "distance": [r["distance"] for r in out]}
        return out

    vm._radius_walk_get_candidates, vm._execute_radius_walk = rec_cand, rec_walk
    cases = []
    for name, lib, space, metric, n, ed, cap, lookback, target, missing in CASES:
        rows = stored_rows(lib, space)
        db.score = score_table(lib)
        vm.voyager_index = rh.RecordingIndex(library(lib)) if space == "cosine" else EuclideanRecordingIndex(rows)
        assert np.array_equal(vm.voyager_index.rows, rows)
        vm.id_map = {i: f"item{i}" for i in range(len(rows))}
        vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
        vm.VOYAGER_METRIC, vm.MAX_SONGS_PER_ARTIST, vm.DUPLICATE_DISTANCE_CHECK_LOOKBACK = metric, cap, lookback
        vm._get_cached_vector.cache_clear()
        dropped = None
        if missing is not None:   # one pool member loses its reverse_id_map entry: no vector, dropped from the pool
            seen.clear()
            vm.find_nearest_neighbors_by_id(target, n=n, eliminate_duplicates=ed, mood_similarity=False,
                                            radius_similarity=True)
            dropped = seen["cand_out"][missing]
            del vm.reverse_id_map[f"item{dropped}"]
            vm._get_cached_vector.cache_clear()
        seen.clear()
        answer = vm.find_nearest_neighbors_by_id(target, n=n, eliminate_duplicates=ed, mood_similarity=False,
                                                 radius_similarity=True)
        assert [vid(r["item_id"]) for r in answer] == seen["walk_out"]["vid"]
        if dropped is not None:
            assert dropped in seen["cand_in"] and dropped not in seen["cand_out"]
        sort_gap, score_gap = case_gaps(rows, vid(target), seen["walk_in"], metric, n, ed, cap)
        cases.append({"name": name, "library": lib, "space": space, "metric": metric, "n": n,
                      "eliminate_duplicates": ed, "max_songs_per_artist": cap, "lookback": lookback,
                      "target": target, "dropped": dropped, "cand_in": seen["cand_in"], "cand_out": seen["cand_out"],
                      "walk_in": seen["walk_in"], "walk_out": seen["walk_out"],
                      "sort_gap": sort_gap, "score_gap": score_gap})
        print(f"{name:34s} pool {len(seen['walk_in']['vid']):4d} -> {len(answer):3d} songs, "
              f"gaps {sort_gap:.3g} / {score_gap:.3g}")
    save(cases)


_ARRAYS = (("cand_in", None), ("cand_out", None), ("walk_in", "vid"), ("walk_in", "dist_anchor"), ("walk_out", "vid"),
           ("walk_out", "distance"))


def save(cases):
    """One compressed .npz: the case parameters as a JSON string, the per-case lists as arrays; authors as indices
    into one name table, -1 for None."""
    names = sorted({a for c in cases for a in c["walk_in"]["author"] if a is not None})
    code = {a: i for i, a in enumerate(names)}
    out = {"authors": np.array(names, dtype=str)}
    meta = []
    for i, c in enumerate(cases):
        meta.append({k: v for k, v in c.items() if k not in ("cand_in", "cand_out", "walk_in", "walk_out")})
        for outer, inner in _ARRAYS:
            v = c[outer] if inner is None else c[outer][inner]
            out[f"{i}_{outer}_{inner or ''}"] = np.asarray(v, dtype=np.float64 if "dist" in (inner or "") else np.int64)
        out[f"{i}_walk_in_author"] = np.array([-1 if a is None else code[a] for a in c["walk_in"]["author"]], np.int64)
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(GOLDEN, **out)


def load(path=GOLDEN):
    """The cases as main() recorded them: lists of index ids, authors (None / str) and float distances."""
    g = np.load(path)
    names = g["authors"].tolist()
    cases = []
    for i, c in enumerate(json.loads(str(g["meta"]))):
        c = dict(c, walk_in={}, walk_out={})
        for outer, inner in _ARRAYS:
            v = g[f"{i}_{outer}_{inner or ''}"].tolist()
            if inner is None:
                c[outer] = v
            else:
                c[outer][inner] = v
        c["walk_in"]["author"] = [None if a < 0 else names[a] for a in g[f"{i}_walk_in_author"].tolist()]
        cases.append(c)
    return cases


def types_voyager():
    import types
    m = types.ModuleType("voyager")

    class RecallError(RuntimeError):
        pass

    m.RecallError = RecallError
    m.Space = types.SimpleNamespace(Cosine=2, Euclidean=0, InnerProduct=1)
    m.Index = rh.RecordingIndex
    return m


if __name__ == "__main__":
    main()
