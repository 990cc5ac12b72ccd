"""Per-request latency of the similar-tracks radius walk: the device drop-in pair (integration.make_radius_walk:
candidate step + am_knn_radius_walk) against the reference's Python walk (oracle/radius_walk.py in "reference" mode,
the reference's own float32 get_direct_distance calls) fed by one get_vector per candidate, as
_radius_walk_get_candidates does over this repository's index.  Libraries of 100 k x 512 and 100 k x 200 with
in-memory metadata standing in for SQL (the title/artist and mood filters are SQL and out of scope: identity here).
n in {10, 25, 100, 200}; the pool is the reference's k = n + max(20, 3n) + 1 nearest neighbours of the anchor.
A host clock around each call (both end in a device synchronise), after a warm-up; median and p99 over >= 200 calls.
Prints the card and its power limit, then one JSON line per (library, n).

    python tools/radius_walk_bench.py [--calls 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import corpus, integration, voyager_compat as vc  # noqa: E402
from oracle import radius_walk as orw  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - reported as such
        power = f"unavailable ({e})"
    return name, power


def stats(ts):
    ts = np.asarray(ts) * 1e3
    return {"median_ms": round(float(np.median(ts)), 4), "p99_ms": round(float(np.percentile(ts, 99)), 4),
            "calls": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    n_items = 100_000
    rng = np.random.default_rng(7)
    n_artists = n_items // 12
    meta = {f"item{i}": {"item_id": f"item{i}", "title": f"Song {i}", "author": f"Artist {int(a)}"}
            for i, a in enumerate(rng.integers(0, n_artists, n_items))}
    sys.modules["app_helper"] = types.SimpleNamespace(
        get_score_data_by_ids=lambda ids: [meta[i] for i in ids if i in meta])
    for d in (512, 200):
        x = corpus.knn_library(n_items, d, 1234 + d)
        idx = vc.Index(vc.Space.Cosine, num_dimensions=d)
        idx.add_items(x)
        vm = types.SimpleNamespace(
            voyager_index=idx, reverse_id_map={f"item{i}": i for i in range(n_items)}, MAX_SONGS_PER_ARTIST=3,
            VOYAGER_METRIC="angular", MOOD_SIMILARITY_ENABLE=False,
            _filter_by_distance=lambda res, db: res, _deduplicate_and_filter_neighbors=lambda res, db, det: res,
            _filter_by_mood_similarity=lambda res, tid, db: res,
            _get_cached_vector=lambda item: idx.get_vector(int(item[4:])))
        cand_fn, walk_fn = integration.make_radius_walk(vm)
        for n in (10, 25, 100, 200):
            k = n + max(20, 3 * n) + 1
            anchors = rng.integers(0, n_items, args.calls + args.warmup)
            requests = []
            for a in anchors:
                ids, dist = idx.query(idx.get_vector(int(a)), k)
                requests.append((f"item{a}", [{"item_id": f"item{int(i)}", "distance": float(s)}
                                              for i, s in zip(ids, dist) if int(i) != a]))

            def device(req):
                target, initial = req
                cd = cand_fn(target, None, initial, None, {}, True, mood_similarity=False)
                return walk_fn(target, n, cd, None, True)

            def reference(req):
                target, initial = req
                anchor = idx.get_vector(int(target[4:]))
                vecs = [idx.get_vector(int(r["item_id"][4:])) for r in initial]   # _get_cached_vector per candidate
                authors = [meta[r["item_id"]]["author"] for r in initial]
                return orw.radius_walk(vecs, anchor, authors, n, True, 3, "angular", mode="reference")

            res = {}
            for label, fn in (("device", device), ("reference_python", reference)):
                for req in requests[:args.warmup]:
                    fn(req)
                ts = []
                for req in requests[args.warmup:]:
                    t0 = time.perf_counter()
                    fn(req)
                    ts.append(time.perf_counter() - t0)
                res[label] = stats(ts)
            same = 0
            for req in requests[args.warmup:args.warmup + 20]:   # the two answer the same on the timed inputs
                got = [r["item_id"] for r in device(req)]
                ref = reference(req)
                same += got == [req[1][p]["item_id"] for p in ref["positions"]]
            print(json.dumps({"library": f"{n_items}x{d}", "n": n, "k": k, **res,
                              "speedup_median": round(res["reference_python"]["median_ms"] / res["device"]["median_ms"], 1),
                              "same_playlist_of_20": same}), flush=True)


if __name__ == "__main__":
    main()
