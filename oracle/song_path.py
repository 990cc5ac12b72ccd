"""Oracle: the Song Path request (tasks/path_manager.py:320-557) in float64.  TEST INFRASTRUCTURE ONLY.

Restates find_path_between_songs over an in-memory library (the index's stored rows, item "item<i>" at row i) and a
metadata table, one job at a time as the reference runs them: the k-NN query of each job (exact float64 distance,
ties by lower row), the by-vector chain of find_nearest_neighbors_by_vector (voyager_manager.py:1589-1657), the
acceptance of _find_best_songs_for_job (path_manager.py:180-317), the merge on failure and the total distance.  Every
distance is computed in float64 from the stored float32 rows; the reference computes them in float32.  The job
planning (centroids, buckets, merges) is the package's own (audiomuse_ai_b200.song_path), which the goldens pin
bit for bit through the recorded query vectors.

Besides the answer it reports the smallest gap that decided it: `thr_gap`, the closest any compared distance came to
its threshold, and `knn_gap`, the closest two neighbours came that a job's prefix keeps apart (the prefix boundary,
and consecutive candidates inside the prefix; exact ties are broken by row in every implementation and not counted).
"""
from __future__ import annotations

import numpy as np

from audiomuse_ai_b200 import song_path as sp
from oracle import knn as oknn


def direct(a, b, metric):
    """get_direct_distance / get_distance in float64: 'euclidean' ||a - b||, 'cosine' 1 - cos, 'angle'
    arccos(cos) / pi; +inf when either row is zero."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if metric == "euclidean":
        return float(np.linalg.norm(a - b))
    den = np.linalg.norm(a) * np.linalg.norm(b)
    if den == 0:
        return float("inf")
    c = float(np.clip(np.dot(a, b) / den, -1.0, 1.0))
    return 1.0 - c if metric == "cosine" else float(np.arccos(c) / np.pi)


def song_path(rows, space, table, cfg, start, end, Lreq, path_fix_size, start_neighbours, end_neighbours):
    """rows: f32[N, d] stored rows; space: 'cosine' or 'euclidean' (the index's k-NN distance); table: item id ->
    details dict; cfg: VOYAGER_METRIC, PATH_DISTANCE_METRIC, MAX_SONGS_PER_ARTIST, LOOKBACK, THRESHOLD_COSINE,
    THRESHOLD_EUCLIDEAN, ELIMINATE_DUPLICATES, BATCH; start_neighbours / end_neighbours: the item ids the heuristic's
    two find_nearest_neighbors_by_id calls return.  Returns a dict: path (item ids), total, queries [(f32 vector, k)],
    jobs [(k, need, found item ids)], thr_gap, knn_gap."""
    rows = np.asarray(rows, np.float32)
    N = len(rows)
    x64 = rows.astype(np.float64)
    row = lambda item: int(item[4:])  # noqa: E731
    vmet = "cosine" if cfg["VOYAGER_METRIC"] == "angular" else "euclidean"
    pmet = "angle" if cfg["PATH_DISTANCE_METRIC"] == "angular" else "euclidean"
    vthr = cfg["THRESHOLD_COSINE"] if vmet == "cosine" else cfg["THRESHOLD_EUCLIDEAN"]
    pthr = cfg["THRESHOLD_COSINE"] if pmet == "angle" else cfg["THRESHOLD_EUCLIDEAN"]
    lookback, cap, ed, batch = cfg["LOOKBACK"], cfg["MAX_SONGS_PER_ARTIST"], cfg["ELIMINATE_DUPLICATES"], cfg["BATCH"]
    out = {"queries": [], "jobs": [], "thr_gap": np.inf, "knn_gap": np.inf}

    def below(a, b, metric, thr):
        dd = direct(x64[a], x64[b], metric)
        if np.isfinite(dd):
            out["thr_gap"] = min(out["thr_gap"], abs(dd - thr))
        return dd < thr

    def knn(vec, k):
        q = np.asarray(vec, np.float32)
        out["queries"].append((q, k))
        dist = oknn.exact_scores_f64(rows, q[None, :], oknn.COSINE if space == "cosine" else oknn.EUCLIDEAN)[0]
        order = np.lexsort((np.arange(N), dist))
        ds = dist[order]
        inner = np.diff(ds[:k])
        if k < N:
            inner = np.append(inner, ds[k] - ds[k - 1])
        inner = inner[inner > 0]
        if len(inner):
            out["knn_gap"] = min(out["knn_gap"], float(inner.min()))
        return [f"item{r}" for r in order[:k]]

    def by_vector(vec, n):
        size = sp.query_size(n, ed, N)
        items = knn(vec, size) if size > 0 else []
        if lookback > 0:   # _filter_by_distance: lists longer than the batch see the window as of their batch's start
            kept, batched, base = [], len(items) > batch, 0
            for i, it in enumerate(items):
                if batched and i % batch == 0:
                    base = len(kept)
                window = kept[max(0, (base if batched else len(kept)) - lookback):]
                if not any(below(row(it), row(o), vmet, vthr) for o in window):
                    kept.append(it)
            items = kept
        seen, unique = set(), []
        for it in items:
            d = table.get(it)
            if d is None or sp.signature(d) in seen:
                continue
            seen.add(sp.signature(d))
            unique.append(it)
        if ed and cap is not None and cap > 0:
            counts, capped = {}, []
            for it in unique:
                a = table[it].get("author")
                if a and counts.get(a, 0) < cap:
                    capped.append(it)
                    counts[a] = counts.get(a, 0) + 1
            unique = capped
        return unique[:n]

    sd, edd = table[start], table[end]
    used, used_sig, counts = {start, end}, {sp.signature(sd), sp.signature(edd)}, {}
    for d in (sd, edd):
        a = sp.normalize(d.get("author"))
        if a:
            counts[a] = counts.get(a, 0) + 1
    path = [start]

    def run_job(vec, k, need):
        found = []
        for it in by_vector(vec, k):
            if len(found) >= need:
                break
            d = table.get(it)
            if it in used or d is None or sp.signature(d) in used_sig:
                continue
            a = sp.normalize(d.get("author"))
            if cap is not None and cap > 0 and counts.get(a, 0) >= cap:
                continue
            if lookback > 0 and any(below(row(it), row(p), pmet, pthr) for p in path[-lookback:]):
                continue
            if lookback > 0 and any(below(row(it), row(p), pmet, pthr) for p in found[-lookback:]):
                continue
            found.append(it)
            used.add(it)
            used_sig.add(sp.signature(d))
            counts[a] = counts.get(a, 0) + 1
        if len(found) < need:
            for it in found:
                used.discard(it)
                used_sig.discard(sp.signature(table[it]))
                a = sp.normalize(table[it].get("author"))
                counts[a] = max(0, counts.get(a, 0) - 1)
            found = []
        out["jobs"].append((k, need, list(found)))
        return found

    m = Lreq - 2
    if m > 0:
        metric = cfg["PATH_DISTANCE_METRIC"]
        inter = sp.interpolate_centroids(rows[row(start)], rows[row(end)], Lreq, metric)[1:-1]
        jobs = sp.plan_jobs(inter, sp.initial_job_count(m, start_neighbours, end_neighbours), path_fix_size)
        i = 0
        while i < len(jobs):
            found = run_job(jobs[i]["vector"], jobs[i]["k"], jobs[i]["need"])
            if found or not path_fix_size:
                path += found
                i += 1
            elif i + 1 >= len(jobs):
                break
            else:
                sp.merge_jobs(jobs, i, inter, metric)
    path.append(end)
    out["path"] = list(dict.fromkeys(path))
    out["total"] = sum(direct(x64[row(a)], x64[row(b)], pmet) for a, b in zip(out["path"], out["path"][1:]))
    return out
