"""Per-request latency of the plain similar-tracks requests: the device drop-ins (similar_tracks.make_*: one query, one
details read and one am_knn_similar call; one am_knn_farthest call for the maximum) against the reference's functions
restated over this repository's index with the reference's round trips: find_nearest_neighbors_by_id's query, the
distance filter on get_vector (behind an LRU cache of 1000 vectors that lives across requests, like
_get_cached_vector), the details reads, the seeded name dedupe, the mood filter parsing other_features, the raw-author
cap; find_nearest_neighbors_by_vector's quadratic same-song scan; get_max_distance_for_id's query(k=len(index)) and
its Python loop over every row.  Libraries of 100 k x 512 (cosine) and 100 k x 200 (euclidean) with in-memory metadata
standing in for SQL; n in {10, 25, 100, 200}, duplicate elimination and mood on and off.  A host clock around each
request (both end in a device synchronise), after a warm-up; median and p99 over --calls requests cycling through 20
targets, and the two sides' answers compared on each.  Prints the card and its power limit, then one JSON line per
(library, request, n, options).

    python tools/similar_tracks_bench.py [--calls 20]
"""
import argparse
import functools
import json
import os
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import similar_tracks as st, voyager_compat as vc  # noqa: E402
from oracle import knn as oknn  # noqa: E402
from tests import ref_harness as rh  # noqa: E402
from tests.golden import make_similar_tracks_golden as gen  # noqa: E402
from tools.radius_walk_bench import card, stats  # noqa: E402


def norm(s):
    return s.strip().lower() if s else ""


class Reference:
    """The reference's three functions over the index, as voyager_manager.py:1372-1702 runs them."""

    def __init__(self, vm, table):
        self.vm, self.table = vm, table
        self.vec = functools.lru_cache(maxsize=1000)(lambda item: vm.voyager_index.get_vector(vm.reverse_id_map[item]))

    def details(self, ids):   # one SQL read
        return {i: dict(self.table[i]) for i in ids if i in self.table}

    def filter(self, items):
        vm = self.vm
        dist = oknn.direct_cosine_distance if vm.VOYAGER_METRIC == "angular" else oknn.direct_euclidean_distance
        thr = (vm.DUPLICATE_DISTANCE_THRESHOLD_COSINE if vm.VOYAGER_METRIC == "angular"
               else vm.DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN)
        self.details([s["item_id"] for s in items])
        kept, batched, base = [], len(items) > 50, 0
        for i, s in enumerate(items):
            if batched and i % 50 == 0:
                base = len(kept)
            v = self.vec(s["item_id"])
            if not any(dist(v, self.vec(o["item_id"])) < thr for o in kept[max(0, (base if batched else len(kept)) - 1):]):
                kept.append(s)
        return kept

    def cap(self, songs, det):
        counts, out = {}, []
        for s in songs:
            a = det.get(s["item_id"], {}).get("author")
            if a and counts.get(a, 0) < self.vm.MAX_SONGS_PER_ARTIST:
                out.append(s)
                counts[a] = counts.get(a, 0) + 1
        return out

    def by_id(self, target, n, ed, mood):
        vm = self.vm
        tdet = self.details([target])[target]
        q = vm.voyager_index.get_vector(vm.reverse_id_map[target])
        k = st.by_id_query_size(n, ed, False, mood, len(vm.voyager_index))
        ids, dists = vm.voyager_index.query(q, k=k)
        init = [{"item_id": vm.id_map[int(i)], "distance": float(d)} for i, d in zip(ids, dists)
                if vm.id_map[int(i)] != target]
        kept = [s for s in self.filter([{"item_id": target, "distance": 0.0}] + init) if s["item_id"] != target]
        det = self.details([s["item_id"] for s in kept])
        seen, unique = {(norm(tdet["title"]), norm(tdet["author"]))}, []
        for s in kept:
            d = det.get(s["item_id"])
            if d and (norm(d["title"]), norm(d["author"])) not in seen:
                seen.add((norm(d["title"]), norm(d["author"])))
                unique.append(s)
        if mood:
            tf = st.parse_mood_features(tdet["other_features"]) if tdet.get("other_features") else {}
            if tf:
                feats = {i: st.parse_mood_features(d["other_features"])
                         for i, d in self.details([s["item_id"] for s in unique]).items() if d.get("other_features")}
                moody = []
                for s in unique:
                    f = feats.get(s["item_id"])
                    if f:
                        md = sum(abs(tf.get(m, 0.0) - f.get(m, 0.0)) for m in st.MOOD_FEATURES) / 6
                        if md <= vm.MOOD_SIMILARITY_THRESHOLD:
                            moody.append(dict(s, mood_distance=md))
                unique = moody
        if ed:
            unique = self.cap(unique, self.details([s["item_id"] for s in unique]))
        return unique[:n]

    def by_vector(self, vec, n, ed):
        vm = self.vm
        ids, dists = vm.voyager_index.query(vec, k=st.query_size(n, ed, len(vm.voyager_index)))
        kept = self.filter([{"item_id": vm.id_map[int(i)], "distance": float(d)} for i, d in zip(ids, dists)])
        det = self.details([s["item_id"] for s in kept])
        unique, added = [], []
        for s in kept:
            d = det.get(s["item_id"])
            if d and not any(norm(d["title"]) == norm(a["title"]) and norm(d["author"]) == norm(a["author"])
                             for a in added):
                unique.append(s)
                added.append(d)
        return (self.cap(unique, det) if ed else unique)[:n]

    def max_distance(self, target):
        vm = self.vm
        tv = vm.reverse_id_map[target]
        nbrs, dists = vm.voyager_index.query(vm.voyager_index.get_vector(tv), k=len(vm.voyager_index))
        best, far = float("-inf"), None
        for v, d in zip(nbrs, dists):
            if v != tv and d > best:
                best, far = d, v
        return {"max_distance": float(best), "farthest_item_id": vm.id_map.get(int(far))}


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
        rng = np.random.default_rng(d)
        base = rng.standard_normal((64, d)).astype(np.float32)
        x = (base[rng.integers(0, 64, N)] + 0.6 * rng.standard_normal((N, d)).astype(np.float32)).astype(np.float32)
        idx = vc.Index(vc.Space.Cosine if space == "cosine" else vc.Space.Euclidean, num_dimensions=d)
        idx.add_items(x, ids=np.arange(N))
        table = rh.make_score_table(N, seed=d)
        frng = np.random.default_rng(d + 1)
        for i in range(N):
            table[f"item{i}"]["other_features"] = gen.other_features(i, frng)
        vm = types.SimpleNamespace(voyager=vc, voyager_index=idx, id_map={i: f"item{i}" for i in range(N)})
        vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
        gen.configure(vm, dict(gen.BASE, VOYAGER_METRIC="angular" if space == "cosine" else "euclidean",
                               THRESHOLD_EUCLIDEAN=0.15))
        sys.modules["app_helper"] = types.SimpleNamespace(
            get_score_data_by_ids=lambda ids: [dict(table[i]) for i in ids if i in table], get_db=lambda: None)
        ref = Reference(vm, table)
        dev = {"by_id": st.make_find_nearest_neighbors_by_id(vm), "by_vector": st.make_find_nearest_neighbors_by_vector(vm),
               "max": st.make_get_max_distance_for_id(vm)}
        targets = [f"item{int(t)}" for t in rng.choice(N, 20, replace=False)]
        vectors = [(x[int(t)] + 0.05 * rng.standard_normal(d)).astype(np.float32) for t in rng.choice(N, 20)]
        runs = []
        for n in (10, 25, 100, 200):
            for ed in (True, False):
                for mood in (False, True):
                    runs.append(("by_id", dict(n=n, eliminate_duplicates=ed, mood_similarity=mood),
                                 lambda t, n=n, ed=ed, mood=mood: dev["by_id"](t, n=n, eliminate_duplicates=ed,
                                                                                mood_similarity=mood,
                                                                                radius_similarity=False),
                                 lambda t, n=n, ed=ed, mood=mood: ref.by_id(t, n, ed, mood)))
                runs.append(("by_vector", dict(n=n, eliminate_duplicates=ed),
                             lambda v, n=n, ed=ed: dev["by_vector"](v, n=n, eliminate_duplicates=ed),
                             lambda v, n=n, ed=ed: ref.by_vector(v, n, ed)))
        runs.append(("max_distance", {}, dev["max"], ref.max_distance))
        for kind, opts, run_dev, run_ref in runs:
            inputs = vectors if kind == "by_vector" else targets
            row = {"library": f"{N}x{d}", "space": space, "request": kind, **opts}
            outs = {}
            for side, fn in (("device", run_dev), ("reference", run_ref)):
                for w in range(args.warmup):
                    fn(inputs[w % len(inputs)])
                torch.cuda.synchronize()
                ts, outs[side] = [], []
                for c in range(args.calls):
                    t0 = time.perf_counter()
                    outs[side].append(fn(inputs[c % len(inputs)]))
                    torch.cuda.synchronize()
                    ts.append(time.perf_counter() - t0)
                row[side] = stats(ts)
            row["same_answer"] = f"{sum(a == b for a, b in zip(outs['device'], outs['reference']))}/{args.calls}"
            row["speedup_median"] = round(row["reference"]["median_ms"] / row["device"]["median_ms"], 1)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
