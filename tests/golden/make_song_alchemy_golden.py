#!/usr/bin/env python
"""Goldens of the reference's Song Alchemy, so that the tests need no reference checkout.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_song_alchemy_golden.py
    # writes tests/golden/song_alchemy_golden.npz

Runs the reference's song_alchemy (tasks/song_alchemy.py:371-1115), UNMODIFIED, over the Song Path goldens' seeded
libraries and metadata table (duplicate rows, case and whitespace title variants, None and "" authors, a
single-artist region), a recording brute-force index, and this module's artist GMMs, anchors, mood centroids, main
map and artist-component projections.  Per case it records the configuration and request, the `random` and
`np.random` seeds, the index queries, the full return dict, and every call of the reference helpers the drop-in calls
too (centroids, GMM components, mood vectors and labels, find_nearest_neighbors_by_id, and the two local projections
with a hash of their input vectors), so that the tests can replay them.  It also records the float64 oracle's
(oracle/song_alchemy.py) candidate distances and deciding gaps.  Item ids are "item<index id>".

Cases cover song, artist, anchor and mood items on both sides, the legacy id lists, the single-song temperature-0
branch, temperatures 0, 0.5 and 1, both PATH_DISTANCE_METRICs and VOYAGER_METRICs, lookback 0 and 1, caps 0, 1 and 3,
eliminate_duplicates on and off, n in {1, 10, 100, 200}, a library smaller than the query, and a main map that is
absent, partial (with >= 4 vectors to project locally, so that the discriminant projection runs) or complete.
"""
import hashlib
import json
import os
import random
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402
from tests.golden import make_radius_walk_golden as rwg  # noqa: E402
from tests.golden import make_song_path_golden as spg  # noqa: E402

GOLDEN = os.path.join(HERE, "song_alchemy_golden.npz")
D = spg.D
library, stored_rows, score_table = spg.library, spg.stored_rows, spg.score_table

ARTISTS = {"art3": ("Artist 3", [100, 400, 700]), "art5": ("Artist 5", [1500])}   # GMM components near these rows
ANCHORS = {"anc1": ("Calm", [200, 201, 202]), "anc2": ("Loud", [1800, 1801])}
MOODS = {"happy": [300, 900], "sad": [1200, 2700]}


def _vec(lib, space, rows, seed):
    """A float64 vector near the mean of `rows` of the stored library (clipped to what the library has)."""
    x = stored_rows(lib, space).astype(np.float64)
    rows = [r % len(x) for r in rows]
    return x[rows].mean(axis=0) + 0.05 * np.random.default_rng(seed).standard_normal(D)


def artist_gmm(lib, space):
    return {name: {"means": [_vec(lib, space, [r], r).tolist() for r in rows],
                   "weights": ([0.5, 0.3, 0.2] if len(rows) == 3 else [1.0]), "is_single_track": len(rows) == 1}
            for name, rows in ARTISTS.values()}


def artist_name(artist_id):
    return ARTISTS[artist_id][0] if artist_id in ARTISTS else None


def anchor(lib, space, anchor_id):
    if anchor_id not in ANCHORS:
        return None
    name, rows = ANCHORS[anchor_id]
    return {"id": anchor_id, "name": name, "centroid": _vec(lib, space, rows, 7).tolist(), "created_at": None}


def moods(lib, space):
    return {m: {"centroids": [{"centroid": _vec(lib, space, [r], r + 1).tolist()} for r in rows]}
            for m, rows in MOODS.items()}


def main_map(lib, kind):
    """load_map_projection('main_map'): None, every item but those at rows divisible by 3, or every item."""
    n = spg.LIBRARIES[lib][0]
    if kind == "none":
        return None, None
    ids = [f"item{i}" for i in range(n) if kind == "full" or i % 3]
    return ids, np.random.default_rng(n).uniform(-1, 1, (len(ids), 2)).astype(np.float32)


def artist_projection_cache():
    """Components 0 and 2 of art3 and the only one of art5 (art3's component 1 is not in the cache)."""
    cmap = [{"artist_id": "art3", "component_idx": 0}, {"artist_id": "art3", "component_idx": 2},
            {"artist_id": "art5", "component_idx": 0}]
    return {"component_map": cmap, "projection": np.array([[0.25, -0.5], [-0.75, 0.125], [0.5, 0.5]])}


def S(i):
    return {"type": "song", "id": f"item{i}"}


DEFAULTS = dict(library="main", space="cosine", pmetric="angular", n=10, temperature=1.0, cap=3, lookback=1, ed=True,
                map="partial", add=None, sub=None, add_ids=None, sub_ids=None, subtract_distance=None)
CASES = [
    dict(name="songs_t1", add=[S(10), S(11)]),
    dict(name="song_sub_song_t05", add=[S(12)], sub=[S(900)], n=100, temperature=0.5),
    dict(name="single_song_t0", add=[S(13)], temperature=0.0),
    dict(name="single_song_t0_sub", add=[S(14)], sub=[S(901)], temperature=0.0, n=100),
    dict(name="artist_add_t05", add=[{"type": "artist", "id": "art3"}], temperature=0.5),
    dict(name="anchor_mood_both_sides", add=[{"type": "anchor", "id": "anc1"}, {"type": "mood", "id": "happy:0"}],
         sub=[{"type": "mood", "id": "sad:1"}, {"type": "anchor", "id": "anc2"}], n=100),
    dict(name="songs_t0_sub_artist", add=[S(20), S(21)], sub=[{"type": "artist", "id": "art5"}], n=100,
         temperature=0.0),
    dict(name="everything", add=[S(22), {"type": "artist", "id": "art5"}, {"type": "anchor", "id": "anc2"},
                                 {"type": "mood", "id": "sad:0"}],
         sub=[S(1203), {"type": "artist", "id": "art3"}, {"type": "mood", "id": "happy:1"},
              {"type": "anchor", "id": "anc1"}], n=100, temperature=0.5),
    dict(name="euc", space="euclidean", pmetric="euclidean", add=[S(30)], sub=[S(600)], n=100),
    dict(name="euc_path_angular", space="euclidean", pmetric="angular", add=[S(31)], sub=[S(601)], n=100,
         temperature=0.0),
    dict(name="cos_path_euclidean", pmetric="euclidean", add=[S(32)], sub=[S(602)], subtract_distance=1.2, n=100),
    dict(name="euc_single_song_t0", space="euclidean", pmetric="euclidean", add=[S(33)], temperature=0.0, n=100),
    dict(name="lookback0", lookback=0, add=[S(34)], n=100),
    dict(name="cap0", cap=0, add=[S(35)], n=100),
    dict(name="cap1", cap=1, add=[S(36)], n=100),
    dict(name="nodedupe", ed=False, add=[S(37)], sub=[S(603)], n=100),
    dict(name="nodedupe_cap1_t0", ed=False, cap=1, add=[S(38), S(39)], n=100, temperature=0.0),
    dict(name="n1", add=[S(40)], n=1),
    dict(name="n200_sub", add=[S(41)], sub=[S(950)], n=200),
    dict(name="n200_t0", add=[S(2401), S(2402)], n=200, temperature=0.0),
    dict(name="single_artist_cap1", add=[S(2403)], cap=1, n=100),
    dict(name="dup_rows", add=[S(105)], n=10),
    dict(name="legacy_ids", add_ids=["item50"], sub_ids=["item700"], n=10),
    dict(name="small", library="small", add=[S(1)], n=10),
    dict(name="small_n100_sub", library="small", add=[S(2)], sub=[S(3)], n=100, temperature=0.0),
    dict(name="map_none_discriminant", map="none", add=[S(42), S(43)], sub=[S(604), S(605)], n=10),
    dict(name="map_partial_discriminant", add=[S(45), S(48)], sub=[S(606), S(609)], n=100),
    dict(name="map_full", map="full", add=[S(46)], sub=[S(607)], n=100),
    dict(name="map_none_pca", map="none", add=[{"type": "mood", "id": "happy:1"}], n=10),
    dict(name="no_centroid", add=[{"type": "anchor", "id": "anc_missing"}, {"type": "mood", "id": "calm:9"}]),
]
CASES = [dict(DEFAULTS, **c) for c in CASES]
THRESHOLD_COSINE, THRESHOLD_EUCLIDEAN, BATCH = 0.01, 0.15, 50


def case_config(c):
    """What voyager_manager and config hold for the case (oracle/song_alchemy.py's cfg)."""
    return {"VOYAGER_METRIC": "angular" if c["space"] == "cosine" else "euclidean",
            "PATH_DISTANCE_METRIC": c["pmetric"], "MAX_SONGS_PER_ARTIST": c["cap"], "LOOKBACK": c["lookback"],
            "THRESHOLD_COSINE": THRESHOLD_COSINE, "THRESHOLD_EUCLIDEAN": THRESHOLD_EUCLIDEAN,
            "ELIMINATE_DUPLICATES": c["ed"], "BATCH": BATCH}


def configure(vm, config, cfg):
    spg.configure(vm, types.SimpleNamespace(), cfg)
    config.PATH_DISTANCE_METRIC = cfg["PATH_DISTANCE_METRIC"]
    config.ALCHEMY_DEFAULT_N_RESULTS, config.ALCHEMY_MAX_N_RESULTS, config.ALCHEMY_TEMPERATURE = 100, 200, 1.0
    config.ALCHEMY_SUBTRACT_DISTANCE_ANGULAR, config.ALCHEMY_SUBTRACT_DISTANCE_EUCLIDEAN = 0.2, 5.0


def vectors_key(*lists):
    """sha256 of the float64 bytes of each list of vectors, in order: what the replay of a projection checks."""
    h = hashlib.sha256()
    for vs in lists:
        h.update(np.asarray(np.vstack(vs) if len(vs) else np.zeros((0, D)), dtype=np.float64).tobytes())
        h.update(b"|")
    return h.hexdigest()


def jsonable(x):
    """The return dict as JSON holds it: tuples become lists, numpy scalars plain floats."""
    return json.loads(json.dumps(x, default=lambda o: o.tolist() if hasattr(o, "tolist") else str(o)))


RECORDED = ("_compute_centroid_from_items", "_get_artist_gmm_vectors_and_weights", "_get_mood_centroid_vector",
            "_get_mood_label", "find_nearest_neighbors_by_id", "_project_with_discriminant", "_project_to_2d")


def call_key(name, args, kwargs):
    if name in ("_project_with_discriminant", "_project_to_2d"):
        return name + ":" + vectors_key(*args)
    return name + ":" + json.dumps([args, kwargs], sort_keys=True)


def main():
    db = rh.FakeDB()
    ref = rh.load_reference(rwg.types_voyager(), db)
    vm, config = ref.vm, ref.config
    ah = sys.modules["app_helper"]
    ah.load_map_projection = lambda name: (None, None)
    gmm_mod = rh._stub("tasks.artist_gmm_manager", artist_gmm_params=None, reverse_artist_map=None)
    rh._stub("app_helper_artist", get_artist_name_by_id=artist_name)
    sa = rh._load("tasks.song_alchemy", "tasks/song_alchemy.py")
    from oracle import song_alchemy as osa

    calls = {}

    def recording(name, fn):
        def wrapper(*args, **kwargs):
            key = call_key(name, args, kwargs)
            try:
                out = fn(*args, **kwargs)
            except Exception as e:
                calls[key] = {"raises": f"{type(e).__name__}: {e}"}
                raise
            if name == "find_nearest_neighbors_by_id":
                calls[key] = {"value": [r["item_id"] for r in out or []]}
            else:
                calls[key] = {"value": jsonable(out)}
            return out
        return wrapper

    for name in RECORDED:
        setattr(sa, name, recording(name, getattr(sa, name)))
    mood_file = tempfile.NamedTemporaryFile("w", suffix=".json", delete=False)
    cases = []
    try:
        for i, c in enumerate(CASES):
            lib, space = c["library"], c["space"]
            cfg = case_config(c)
            rows = stored_rows(lib, space)
            db.score = score_table(lib)
            vm.voyager_index = (rh.RecordingIndex(library(lib)) if space == "cosine"
                                else spg.EuclideanRecordingIndex(rows))
            assert np.array_equal(vm.voyager_index.rows, rows)
            vm.id_map = {k: f"item{k}" for k in range(len(rows))}
            vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
            configure(vm, config, cfg)
            vm._get_cached_vector.cache_clear()
            gmm_mod.artist_gmm_params, gmm_mod.reverse_artist_map = artist_gmm(lib, space), {}
            gmm_mod.load_artist_index_for_querying = lambda: None
            ah.get_alchemy_anchor_by_id = lambda a, lib=lib, space=space: anchor(lib, space, a)
            ah.ARTIST_PROJECTION_CACHE = artist_projection_cache()
            ah.load_map_projection = sa.load_map_projection = lambda name, kind=c["map"], lib=lib: main_map(lib, kind)
            mood_file.seek(0)
            mood_file.truncate()
            json.dump(moods(lib, space), mood_file)
            mood_file.flush()
            config.MOOD_CENTROIDS_FILE = mood_file.name
            calls.clear()
            random.seed(1000 + i)
            np.random.seed(2000 + i)
            t0 = len(vm.voyager_index.trace)
            out = sa.song_alchemy(add_items=c["add"], subtract_items=c["sub"], add_ids=c["add_ids"],
                                  subtract_ids=c["sub_ids"], n_results=c["n"], subtract_distance=c["subtract_distance"],
                                  temperature=c["temperature"])
            queries = [(e["vector"], e["k"]) for e in vm.voyager_index.trace[t0:] if e["op"] == "query"]
            rec = dict(c, config=cfg, random_seed=1000 + i, np_random_seed=2000 + i, result=jsonable(out),
                       calls=dict(calls), queries=queries)
            rec.update(check_with_oracle(osa, rows, db.score, rec))
            cases.append(rec)
            res = out["results"]
            print(f"{c['name']:26s} {len(res):3d} results, {len(out['filtered_out']):3d} filtered out, "
                  f"projection {out.get('projection')!s:12s} gaps filter {rec['filter_gap']:.2e} sub "
                  f"{rec['sub_gap']:.2e} knn {rec['knn_gap']:.2e} sample {rec['sample_gap']:.2e}")
    finally:
        os.unlink(mood_file.name)
    save(cases)


def request_centroids(rec):
    """The add and subtract centroids the reference computed, from the recorded helper calls."""
    def items(side):
        its, ids = rec[side], rec[side + "_ids"]
        return [{"type": "song", "id": i} for i in ids] if its is None and ids is not None else its

    def centroid(its):
        if not its:
            return None
        v = rec["calls"][call_key("_compute_centroid_from_items", (its,), {})]["value"]
        return None if v is None else np.array(v, dtype=float)

    return items("add"), items("sub"), centroid(items("add")), centroid(items("sub"))


def oracle_request(osa, rows, table, rec):
    """The oracle's answer to the recorded request: (candidates() dict or None, knn_gap)."""
    add, sub, add_c, sub_c = request_centroids(rec)
    if add_c is None:
        return None, np.inf
    n = rec["n"] * 3
    cfg = rec["config"]
    thr = rec["subtract_distance"]
    if thr is None:
        thr = 0.2 if cfg["PATH_DISTANCE_METRIC"] == "angular" else 5.0
    own = {it["id"] for it in add + (sub or []) if it.get("type") == "song"}
    nb_key = call_key("find_nearest_neighbors_by_id", (add[0]["id"],), {"n": rec["n"]}) if add else None
    if rec["temperature"] == 0.0 and len(add) == 1 and add[0].get("type") == "song" and nb_key in rec["calls"]:
        listed, skip, knn_gap = rec["calls"][nb_key]["value"], True, np.inf
    else:
        from audiomuse_ai_b200 import song_path as sp
        k = sp.query_size(n, cfg["ELIMINATE_DUPLICATES"], len(rows))
        listed, knn_gap = osa.knn_list(rows, rec["space"], add_c, k) if k > 0 else ([], np.inf)
        skip = False
    o = osa.candidates(rows, osa.keys(table, listed), cfg, cfg["PATH_DISTANCE_METRIC"], add_c, sub_c, thr, listed, own, n, skip)
    return o, knn_gap


def check_with_oracle(osa, rows, table, rec):
    """Asserts the oracle's kept / filtered-out lists, distances and sampled order against the recorded return dict;
    returns what the golden keeps of it."""
    o, knn_gap = oracle_request(osa, rows, table, rec)
    res = rec["result"]
    if o is None or not o["chain"]:
        assert res["results"] == [] and res["filtered_out"] == [], rec["name"]
        return {"candidates": [], "distances": [], "filter_gap": np.inf, "sub_gap": np.inf, "knn_gap": knn_gap,
                "sample_gap": np.inf}
    ids = [i for i in o["kept"] if i in table]
    order, sample_gap = osa.sample(ids, o["distances"], rec["temperature"], rec["n"], rec["random_seed"])
    assert [r["item_id"] for r in res["results"]] == order, rec["name"]
    assert all(r["distance"] == o["distances"][r["item_id"]] for r in res["results"]), rec["name"]
    assert [r["item_id"] for r in res["filtered_out"]] == o["filtered_out"], rec["name"]
    return {"candidates": ids, "distances": [o["distances"][i] for i in ids], "filter_gap": o["filter_gap"],
            "sub_gap": o["sub_gap"], "knn_gap": knn_gap, "sample_gap": sample_gap}


def save(cases):
    """One compressed .npz: the cases as a JSON string (inf as null), each case's query vectors f32[nq, d] beside it."""
    out, meta = {}, []
    for i, c in enumerate(cases):
        out[f"{i}_queries"] = np.array([q for q, _ in c["queries"]], dtype=np.float32).reshape(-1, D)
        m = {k: v for k, v in c.items() if k != "queries"}
        m["query_k"] = [int(k) for _, k in c["queries"]]
        for g in ("filter_gap", "sub_gap", "knn_gap", "sample_gap"):
            m[g] = None if not np.isfinite(m[g]) else float(m[g])
        meta.append(m)
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(GOLDEN, **out)


def load(path=GOLDEN):
    """The cases as main() recorded them; "queries" is the list of (f32 vector, k), a gap of None is +inf."""
    g = np.load(path)
    cases = json.loads(str(g["meta"]))
    for i, c in enumerate(cases):
        c["queries"] = list(zip(g[f"{i}_queries"], c.pop("query_k")))
        for k in ("filter_gap", "sub_gap", "knn_gap", "sample_gap"):
            c[k] = np.inf if c[k] is None else c[k]
    return cases


if __name__ == "__main__":
    main()
