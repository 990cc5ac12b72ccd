"""Per-request latency of the Song Path: the device drop-in (song_path.make_song_path: one batched query, one details
read, one am_knn_song_path call) against the reference's per-job Python over this repository's index, restated here
with the reference's round trips: per job one index.query, one get_vector per candidate the distance filter looks at
(cached, like _get_cached_vector), two details reads, one get_vector per candidate the acceptance reaches, the
reference's float32 distance helpers, and one get_vector per path song for the total.  Libraries of 100 k x 512
(cosine) and 100 k x 200 (euclidean) with in-memory metadata standing in for SQL; Lreq in {10, 25, 100}, path_fix_size
off and on; the heuristic's two find_nearest_neighbors_by_id calls are the same top-25 lists on both sides and not
timed.  A host clock around each request (both end in a device synchronise), after a warm-up; median and p99 over
--calls requests cycling through 20 (start, end) pairs, and the two sides' paths compared on each pair.  Prints the card
and its power limit, then one JSON line per (library, Lreq, path_fix_size).

    python tools/song_path_bench.py [--calls 200]
"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import song_path as sp, voyager_compat as vc  # noqa: E402
from oracle import knn as oknn  # noqa: E402
from tests import ref_harness as rh  # noqa: E402
from tests.golden import make_song_path_golden as gen  # noqa: E402
from tools.radius_walk_bench import card, stats  # noqa: E402


def angular32(a, b):
    """path_manager.get_angular_distance on float32 rows."""
    na, nb = np.linalg.norm(a), np.linalg.norm(b)
    if na == 0 or nb == 0:
        return float("inf")
    return np.arccos(np.clip(np.dot(a / na, b / nb), -1.0, 1.0)) / np.pi


def reference_request(idx, table, cfg, start, end, Lreq, fix, nb):
    """find_path_between_songs as the reference runs it over the index, job by job."""
    cache = {}

    def vec(item):
        if item not in cache:
            cache[item] = idx.get_vector(int(item[4:]))
        return cache[item]

    vdist = oknn.direct_cosine_distance if cfg["VOYAGER_METRIC"] == "angular" else oknn.direct_euclidean_distance
    pdist = angular32 if cfg["PATH_DISTANCE_METRIC"] == "angular" else (lambda a, b: np.linalg.norm(a - b))
    vthr = cfg["THRESHOLD_COSINE"] if cfg["VOYAGER_METRIC"] == "angular" else cfg["THRESHOLD_EUCLIDEAN"]
    pthr = cfg["THRESHOLD_COSINE"] if cfg["PATH_DISTANCE_METRIC"] == "angular" else cfg["THRESHOLD_EUCLIDEAN"]
    lb, cap, ed = cfg["LOOKBACK"], cfg["MAX_SONGS_PER_ARTIST"], cfg["ELIMINATE_DUPLICATES"]
    details = lambda ids: {i: dict(table[i]) for i in ids if i in table}  # noqa: E731  (one SQL read)
    start_vec, end_vec = idx.get_vector(int(start[4:])), idx.get_vector(int(end[4:]))
    used, used_sig, counts = {start, end}, {sp.signature(table[start]), sp.signature(table[end])}, {}
    for a in (sp.normalize(table[start]["author"]), sp.normalize(table[end]["author"])):
        if a:
            counts[a] = counts.get(a, 0) + 1
    path = [(start, start_vec)]

    def job(v, k, need):
        size = sp.query_size(k, ed, len(idx))
        items = [f"item{int(i)}" for i in idx.query(np.asarray(v, np.float32), size)[0]]
        kept = []
        for i, it in enumerate(items):
            if lb <= 0:
                kept = items
                break
            if len(items) > 50 and i % 50 == 0:
                base = len(kept)
            window = kept[max(0, (base if len(items) > 50 else len(kept)) - lb):]
            if not any(vdist(vec(it), vec(o)) < vthr for o in window):
                kept.append(it)
        det = details(kept)
        seen, out, acounts = set(), [], {}
        for it in kept:
            d = det.get(it)
            if d is None or sp.signature(d) in seen:
                continue
            seen.add(sp.signature(d))
            if ed and cap > 0:
                if not d["author"] or acounts.get(d["author"], 0) >= cap:
                    continue
                acounts[d["author"]] = acounts.get(d["author"], 0) + 1
            out.append(it)
        det = details(out[:k])
        found = []
        for it in out[:k]:
            if len(found) >= need:
                break
            d = det.get(it)
            a = sp.normalize(d["author"])
            if it in used or sp.signature(d) in used_sig or (cap > 0 and counts.get(a, 0) >= cap):
                continue
            cv = idx.get_vector(int(it[4:]))
            if lb > 0 and any(pdist(cv, pv) < pthr for _, pv in path[-lb:]):
                continue
            if lb > 0 and any(pdist(cv, pv) < pthr for _, pv in found[-lb:]):
                continue
            found.append((it, cv))
            used.add(it)
            used_sig.add(sp.signature(d))
            counts[a] = counts.get(a, 0) + 1
        if len(found) < need:
            for it, _ in found:
                used.discard(it)
                used_sig.discard(sp.signature(table[it]))
                a = sp.normalize(table[it]["author"])
                counts[a] = max(0, counts.get(a, 0) - 1)
            return []
        return found

    metric = cfg["PATH_DISTANCE_METRIC"]
    inter = sp.interpolate_centroids(start_vec, end_vec, Lreq, metric)[1:-1]
    jobs = sp.plan_jobs(inter, sp.initial_job_count(Lreq - 2, *nb), fix)
    i = 0
    while i < len(jobs):
        found = job(jobs[i]["vector"], jobs[i]["k"], jobs[i]["need"])
        if found or not fix:
            path += found
            i += 1
        elif i + 1 >= len(jobs):
            break
        else:
            sp.merge_jobs(jobs, i, inter, metric)
    ids = list(dict.fromkeys([p for p, _ in path] + [end]))
    vecs = [idx.get_vector(int(p[4:])) for p in ids]
    return ids, float(sum(pdist(a, b) for a, b in zip(vecs, vecs[1:])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
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
        pairs = [tuple(f"item{int(v)}" for v in rng.choice(N, 2, replace=False)) for _ in range(20)]
        nbs = {}
        for s, e in pairs:
            q = idx.get_vectors([int(s[4:]), int(e[4:])])
            nbs[(s, e)] = [[f"item{int(i)}" for i in r] for r in idx.query(q, 25)[0]]
        for Lreq in (10, 25, 100):
            for fix in (False, True):
                cfg = gen.case_config(("", "", space, "angular" if space == "cosine" else "euclidean", Lreq, fix, 3, 1,
                                       True, 0.01, 0.15, "", ""))
                vm = types.SimpleNamespace(voyager_index=idx, id_map={i: f"item{i}" for i in range(N)})
                vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
                pm = types.SimpleNamespace()
                gen.configure(vm, pm, cfg)
                pm.PATH_CANDIDATES_PER_STEP = 25
                pm.get_vector_by_id = lambda item: idx.get_vector(int(item[4:]))
                pm._create_path_from_ids = lambda ids: [dict(table[i]) for i in dict.fromkeys(ids) if i in table]
                sys.modules["app_helper"] = types.SimpleNamespace(
                    get_score_data_by_ids=lambda ids: [dict(table[i]) for i in ids if i in table])
                device = sp.make_song_path(vm, pm)

                def run_device(s, e):
                    nb = iter(nbs[(s, e)])
                    pm.find_nearest_neighbors_by_id = lambda item_id, n=10: [{"item_id": i} for i in next(nb)]
                    details, total = device(s, e, Lreq, path_fix_size=fix)
                    torch.cuda.synchronize()
                    return [dd["item_id"] for dd in details], total

                def run_ref(s, e):
                    out = reference_request(idx, table, cfg, s, e, Lreq, fix, nbs[(s, e)])
                    torch.cuda.synchronize()
                    return out

                same = sum(run_device(*p)[0] == run_ref(*p)[0] for p in pairs)
                row = {"library": f"{N}x{d}", "space": space, "Lreq": Lreq, "path_fix_size": fix,
                       "same_path": f"{same}/{len(pairs)}"}
                for side, fn in (("device", run_device), ("reference", run_ref)):
                    for w in range(args.warmup):
                        fn(*pairs[w % len(pairs)])
                    ts = []
                    for c in range(args.calls):
                        t0 = time.perf_counter()
                        fn(*pairs[c % len(pairs)])
                        ts.append(time.perf_counter() - t0)
                    row[side] = stats(ts)
                row["speedup_median"] = round(row["reference"]["median_ms"] / row["device"]["median_ms"], 1)
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
