"""Per-request latency of Song Alchemy: the device drop-in (alchemy.make_song_alchemy: one query, one details read,
one am_knn_alchemy call) against the reference's candidate path over this repository's index, restated here with the
reference's round trips: the by-vector query, the distance filter on get_vector (behind an LRU cache of 1000 vectors
that lives across requests, like _get_cached_vector), one details read, the quadratic same-song dedupe on normalised
strings, the raw-author cap, then one get_vector per candidate for the subtract filter, again for the projection and
again for the displayed distances, one details read per list, and the same temperature sampling.  Both sides see the
same centroids (the mean of two add songs, one subtract song), a main map that covers every item (each side turns it
into its item -> coordinate dict per request, as the reference does; no local projection runs) and the same `random`
seed.  Libraries of 100 k x 512 (cosine) and 100 k x 200
(euclidean) with in-memory metadata standing in for SQL; n in {10, 100, 200}, with and without a subtract song.  A host
clock around each request (both end in a device synchronise), after a warm-up; median and p99 over --calls requests
cycling through 20 requests (the reference takes seconds per request at n = 200), and the two sides' playlists compared
on each.  Prints the card and its power limit, then
one JSON line per (library, n, subtract).

    python tools/song_alchemy_bench.py [--calls 20]
"""
import argparse
import functools
import json
import os
import random
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import alchemy as al, song_path as sp, voyager_compat as vc  # noqa: E402
from oracle import knn as oknn  # noqa: E402
from tests import ref_harness as rh  # noqa: E402
from tools.radius_walk_bench import card, stats  # noqa: E402

N_CFG = dict(VOYAGER_METRIC=None, DUPLICATE_DISTANCE_CHECK_LOOKBACK=1, BATCH_SIZE_VECTOR_OPS=50,
             DUPLICATE_DISTANCE_THRESHOLD_COSINE=0.01, DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN=0.15,
             MAX_SONGS_PER_ARTIST=3, SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT=True)


def centroid_distance(c, v, metric):
    if metric == "angular":
        cs = np.clip(np.dot(c / (np.linalg.norm(c) or 1.0), v / (np.linalg.norm(v) or 1.0)), -1.0, 1.0)
        return float(np.arccos(cs) / np.pi)
    return float(np.linalg.norm(c - v))


def reference_request(idx, vec, table, metric, add_ids, sub_ids, n, thr, main_map):
    """song_alchemy's candidate path as the reference runs it over the index; returns the result ids."""
    details = lambda ids: {i: dict(table[i]) for i in ids if i in table}  # noqa: E731  (one SQL read)
    norm = lambda s: s.strip().lower() if s else ""  # noqa: E731
    add_c = np.mean([np.array(vec(i), dtype=float) for i in add_ids], axis=0)
    sub_c = np.mean([np.array(vec(i), dtype=float) for i in sub_ids], axis=0) if sub_ids else None
    vdist = oknn.direct_cosine_distance if metric == "angular" else oknn.direct_euclidean_distance
    vthr = N_CFG["DUPLICATE_DISTANCE_THRESHOLD_COSINE" if metric == "angular" else "DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN"]
    k = sp.query_size(3 * n, True, len(idx))
    items = [f"item{int(i)}" for i in idx.query(np.asarray(add_c, np.float32), k)[0]]
    kept = []
    for i, it in enumerate(items):
        if len(items) > 50 and i % 50 == 0:
            base = len(kept)
        window = kept[max(0, (base if len(items) > 50 else len(kept)) - 1):]
        if not any(vdist(vec(it), vec(o)) < vthr for o in window):
            kept.append(it)
    det = details(kept)
    unique, added = [], []
    for it in kept:
        d = det.get(it)
        if not d:
            continue
        if not any(norm(d["title"]) == norm(a["title"]) and norm(d["author"]) == norm(a["author"]) for a in added):
            unique.append(it)
            added.append(d)
    counts, neighbours = {}, []
    for it in unique:
        a = det[it]["author"]
        if a and counts.get(a, 0) < 3:
            neighbours.append(it)
            counts[a] = counts.get(a, 0) + 1
    own = set(add_ids) | set(sub_ids)
    cands = [it for it in neighbours[:3 * n] if it not in own]
    filtered_out = []
    if sub_c is not None:
        keep = []
        for it in cands:
            (keep if centroid_distance(sub_c, np.array(vec(it), dtype=float), metric) >= thr else filtered_out).append(it)
        cands = keep
    proj_vectors = [np.array(vec(it), dtype=float) for it in cands + filtered_out]  # built even when the map has all
    assert len(proj_vectors) == len(cands) + len(filtered_out)
    to_coord = {str(i): (float(c[0]), float(c[1])) for i, c in zip(main_map[0], main_map[1].tolist())}
    coords = {it: to_coord.get(it) for it in cands + filtered_out}
    distances = {it: centroid_distance(add_c, np.array(vec(it), dtype=float), metric) for it in cands}
    det = details(cands)
    chosen = al.sample([c for c in cands if c in det], distances, 1.0, n)
    for it in chosen:
        det[it].update(distance=distances[it], embedding_2d=coords[it])
    details(filtered_out)
    return chosen


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    for d, space in ((512, "cosine"), (200, "euclidean")):
        N = 100_000
        metric = "angular" if space == "cosine" else "euclidean"
        rng = np.random.default_rng(d)
        base = rng.standard_normal((64, d)).astype(np.float32)
        x = (base[rng.integers(0, 64, N)] + 0.6 * rng.standard_normal((N, d)).astype(np.float32)).astype(np.float32)
        idx = vc.Index(vc.Space.Cosine if space == "cosine" else vc.Space.Euclidean, num_dimensions=d)
        idx.add_items(x, ids=np.arange(N))
        table = rh.make_score_table(N, seed=d)
        main_map = ([f"item{i}" for i in range(N)], rng.uniform(-1, 1, (N, 2)).astype(np.float32))
        vec = functools.lru_cache(maxsize=1000)(lambda item: idx.get_vector(int(item[4:])))
        stored = lambda item: idx.get_vector(int(item[4:]))  # noqa: E731
        requests = [([f"item{int(a)}" for a in rng.choice(N, 2, replace=False)], f"item{int(rng.integers(N))}")
                    for _ in range(20)]
        vm = types.SimpleNamespace(voyager_index=idx, id_map={i: f"item{i}" for i in range(N)}, **N_CFG)
        vm.VOYAGER_METRIC = metric
        vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
        thr = 0.2 if metric == "angular" else float(np.median(np.linalg.norm(x[:1000] - x[1000], axis=1)))
        sa = types.SimpleNamespace(
            config=types.SimpleNamespace(PATH_DISTANCE_METRIC=metric, ALCHEMY_DEFAULT_N_RESULTS=100,
                                         ALCHEMY_MAX_N_RESULTS=200, ALCHEMY_TEMPERATURE=1.0,
                                         ALCHEMY_SUBTRACT_DISTANCE_ANGULAR=thr, ALCHEMY_SUBTRACT_DISTANCE_EUCLIDEAN=thr),
            get_vector_by_id=stored,
            _compute_centroid_from_items=lambda items: np.mean([np.array(stored(i["id"]), dtype=float)
                                                                for i in items], axis=0),
            get_score_data_by_ids=lambda ids: [dict(table[i]) for i in ids if i in table],
            load_map_projection=lambda name: main_map)
        sys.modules["app_helper"] = types.SimpleNamespace(ARTIST_PROJECTION_CACHE=None)
        device = al.make_song_alchemy(sa, vm)
        for n in (10, 100, 200):
            for with_sub in (False, True):
                def run_device(r):
                    random.seed(7)
                    out = device(add_items=[{"type": "song", "id": i} for i in r[0]],
                                 subtract_items=[{"type": "song", "id": r[1]}] if with_sub else None, n_results=n,
                                 temperature=1.0)
                    torch.cuda.synchronize()
                    return [o["item_id"] for o in out["results"]]

                def run_ref(r):
                    random.seed(7)
                    out = reference_request(idx, vec, table, metric, r[0], [r[1]] if with_sub else [], n, thr, main_map)
                    torch.cuda.synchronize()
                    return out

                row = {"library": f"{N}x{d}", "space": space, "n": n, "subtract": with_sub}
                outs = {}
                for side, fn in (("device", run_device), ("reference", run_ref)):
                    for w in range(args.warmup):
                        fn(requests[w % len(requests)])
                    ts, outs[side] = [], []
                    for c in range(args.calls):
                        t0 = time.perf_counter()
                        outs[side].append(fn(requests[c % len(requests)]))
                        ts.append(time.perf_counter() - t0)
                    row[side] = stats(ts)
                row["same_playlist"] = f"{sum(a == b for a, b in zip(outs['device'], outs['reference']))}/{args.calls}"
                row["speedup_median"] = round(row["reference"]["median_ms"] / row["device"]["median_ms"], 1)
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
