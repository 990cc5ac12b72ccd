"""Oracle: the plain similar-tracks requests of tasks/voyager_manager.py in float64.  TEST INFRASTRUCTURE ONLY.

Restates, over an in-memory library (the index's stored rows, item "item<i>" at row i) and a metadata table (item id ->
its score row: title, author, other_features), with no database:
  * find_nearest_neighbors_by_id without the radius walk (:1372-1545): the k-NN query of the target's stored row
    (exact float64 distance, ties by lower row, returned as float32), the target prepended to the distance filter and
    taken out again, the name dedupe seeded with the target's signature, the mood filter, the raw-author cap, [:n];
  * find_nearest_neighbors_by_vector (:1547-1657): the query, the distance filter, the name dedupe, the cap, [:n];
  * get_max_distance_for_id (:1660-1702): the first strict maximum of the float32 distances of query(k=N) in the
    query's order, skipping the target.
The filter's distances are float64 where the reference's are float32; the mood distances are the reference's own sum in
Python floats, so they agree bit for bit.

Besides the answer it reports the gaps that decided it: `filter_gap` (closest any filter distance came to its
threshold), `knn_gap` (closest two neighbours came that the query keeps apart) and, for the maximum, `far_gap` (closest
a float64 distance came to the float32 rounding boundary below the maximum, or to another distance at that maximum).
"""
from __future__ import annotations

import numpy as np

from audiomuse_ai_b200 import song_path as sp
from oracle import knn as oknn
from oracle import song_path as osp

MOOD_FEATURES = ["danceable", "aggressive", "happy", "party", "relaxed", "sad"]


def parse_mood(s):
    """_parse_mood_features (:824-838)."""
    try:
        out = {}
        for pair in s.split(","):
            if ":" in pair:
                k, v = pair.split(":", 1)
                out[k.strip()] = float(v.strip())
        return out
    except Exception:
        return {}


def knn(rows, space, vec, k):
    """query(vec, k): [(row, float32 distance)] in (float64 distance, row) order, and the knn gap."""
    q = np.asarray(vec, np.float32)
    dist = oknn.exact_scores_f64(rows, q[None, :], oknn.COSINE if space == "cosine" else oknn.EUCLIDEAN)[0]
    order = np.lexsort((np.arange(len(rows)), dist))
    ds = dist[order]
    inner = np.diff(ds[:k])
    if k < len(rows):
        inner = np.append(inner, ds[k] - ds[k - 1])
    inner = inner[inner > 0]
    return [(int(r), float(np.float32(dist[r]))) for r in order[:k]], float(inner.min()) if len(inner) else np.inf


def _filter(x64, cfg, rows_in_order):
    """_filter_by_distance over stored rows (None: no vector); returns (kept positions, filter_gap)."""
    vmet = "cosine" if cfg["VOYAGER_METRIC"] == "angular" else "euclidean"
    thr = cfg["THRESHOLD_COSINE"] if vmet == "cosine" else cfg["THRESHOLD_EUCLIDEAN"]
    lookback, batch = cfg["LOOKBACK"], cfg["BATCH"]
    if lookback <= 0:
        return list(range(len(rows_in_order))), np.inf
    gap = np.inf
    kept, batched, base = [], len(rows_in_order) > batch, 0
    for i, r in enumerate(rows_in_order):
        if batched and i % batch == 0:
            base = len(kept)
        if r is None:
            continue
        close = False
        for p in kept[max(0, (base if batched else len(kept)) - lookback):]:
            dd = osp.direct(x64[r], x64[rows_in_order[p]], vmet)
            if np.isfinite(dd):
                gap = min(gap, abs(dd - thr))
            close = close or dd < thr
        if not close:
            kept.append(i)
    return kept, gap


def _chain(rows, table, cfg, items, n, ed, seed=None, target_features=None):
    """The stages after the query over `items` [(item id, float32 distance)]: filter (a by-id target is items[0]),
    dedupe, mood (target_features: the target's parsed features, None: no stage), cap, [:n]."""
    x64 = np.asarray(rows, np.float32).astype(np.float64)
    row = lambda i: int(i[4:]) if 0 <= int(i[4:]) < len(rows) else None  # noqa: E731
    kept, gap = _filter(x64, cfg, [row(i) for i, _ in items])
    songs = [items[p] for p in kept]
    if seed is not None:
        songs = [s for s in songs if s[0] != seed]
    seen = set() if seed is None else {sp.signature(table[seed])}
    unique = []
    for it, d in songs:
        if it not in table:
            continue
        s = sp.signature(table[it])
        if s not in seen:
            seen.add(s)
            unique.append({"item_id": it, "distance": d})
    if target_features is not None:
        moody = []
        for r in unique:
            of = table[r["item_id"]].get("other_features")
            f = parse_mood(of) if of else {}
            if not f:
                continue
            md = sum(abs(target_features.get(k, 0.0) - f.get(k, 0.0)) for k in MOOD_FEATURES) / len(MOOD_FEATURES)
            if md <= cfg["MOOD_SIMILARITY_THRESHOLD"]:
                moody.append(dict(r, mood_distance=md))
        unique = moody
    cap = cfg["MAX_SONGS_PER_ARTIST"]
    if ed and cap is not None and cap > 0:
        counts, out = {}, []
        for r in unique:
            a = table[r["item_id"]].get("author")
            if not a:
                continue
            if counts.get(a, 0) < cap:
                out.append(r)
                counts[a] = counts.get(a, 0) + 1
        unique = out
    return unique[:n], gap


def by_id(rows, space, table, cfg, target, n=10, eliminate_duplicates=None, mood_similarity=None):
    """find_nearest_neighbors_by_id(target, n, eliminate_duplicates, mood_similarity, radius_similarity=False).
    cfg: VOYAGER_METRIC, THRESHOLD_COSINE, THRESHOLD_EUCLIDEAN, LOOKBACK, BATCH, MAX_SONGS_PER_ARTIST,
    ELIMINATE_DUPLICATES, MOOD_SIMILARITY_ENABLE, MOOD_SIMILARITY_THRESHOLD.  Returns (the dicts, filter_gap,
    knn_gap)."""
    ed = cfg["ELIMINATE_DUPLICATES"] if eliminate_duplicates is None else eliminate_duplicates
    if target not in table:
        return [], np.inf, np.inf
    k = n + (max(20, int(n * 3)) if ed else max(3, int(n * 0.20))) + 1
    if mood_similarity:
        k = n + max(20, int(n * (8 if ed else 4))) + 1
    k = min(k, len(rows))
    found, kgap = knn(rows, space, rows[int(target[4:])], k) if k > 1 else ([], np.inf)
    items = [(f"item{r}", d) for r, d in found if f"item{r}" != target]
    mood = cfg["MOOD_SIMILARITY_ENABLE"] if mood_similarity is None else mood_similarity
    tf = None
    if mood:
        of = table[target].get("other_features")
        tf = (parse_mood(of) if of else {}) or None
    out, gap = _chain(rows, table, cfg, [(target, 0.0)] + items, n, ed, seed=target, target_features=tf)
    return out, gap, kgap


def by_vector(rows, space, table, cfg, vec, n=100, eliminate_duplicates=None):
    """find_nearest_neighbors_by_vector(vec, n, eliminate_duplicates): (the dicts, filter_gap, knn_gap)."""
    ed = cfg["ELIMINATE_DUPLICATES"] if eliminate_duplicates is None else eliminate_duplicates
    k = min(n + int(n * 4) if ed else n + int(n * 0.2), len(rows))
    found, kgap = knn(rows, space, vec, k) if k > 0 else ([], np.inf)
    out, gap = _chain(rows, table, cfg, [(f"item{r}", d) for r, d in found], n, ed)
    return out, gap, kgap


def max_distance(rows, space, target, metric=None):
    """get_max_distance_for_id(target): ({max_distance, farthest_item_id}, far_gap).  metric: an oknn metric
    (default: the space's)."""
    t = int(target[4:])
    if metric is None:
        metric = oknn.COSINE if space == "cosine" else oknn.EUCLIDEAN
    dd = oknn.exact_scores_f64(rows, np.asarray(rows[t], np.float32)[None, :], metric)[0]
    f = dd.astype(np.float32)
    mask = np.arange(len(rows)) != t
    if not mask.any():
        return {"max_distance": 0.0, "farthest_item_id": None}, np.inf
    fmax = f[mask].max()
    at = np.flatnonzero(mask & (f == fmax))
    best = at[np.lexsort((at, dd[at]))[0]]
    below = float(np.nextafter(fmax, np.float32(-np.inf)))
    boundary = (float(fmax) + below) / 2.0            # a float64 distance below this rounds under the maximum
    others = dd[at[at != best]]
    gaps = [abs(dd[mask] - boundary).min()] + ([np.abs(others - dd[best]).min()] if len(others) else [])
    same = others[others == dd[best]]
    gaps = [g for g in gaps if g > 0] if len(same) else gaps   # exact ties are broken by row everywhere
    return {"max_distance": float(fmax), "farthest_item_id": f"item{best}"}, float(min(gaps)) if gaps else np.inf


def similar_keys(rows, cfg, target_row, target_sig, cand_rows, cand_sig, cand_raw, n, mood=None, mood_ok=None,
                 target_mood=None):
    """am_knn_similar restated over its inputs (the keys a drop-in built): cfg an am_similar_cfg-like object (metric,
    filter_lookback, filter_batch, cap, filter_threshold, mood_threshold).  Returns (positions, mood distances or
    None)."""
    x64 = np.asarray(rows, np.float32).astype(np.float64)
    ocfg = {"VOYAGER_METRIC": "angular" if cfg.metric == 0 else "euclidean", "THRESHOLD_COSINE": cfg.filter_threshold,
            "THRESHOLD_EUCLIDEAN": cfg.filter_threshold, "LOOKBACK": cfg.filter_lookback, "BATCH": cfg.filter_batch}
    by_id = target_row is not None and target_row >= 0
    lst = ([int(target_row)] if by_id else []) + [int(r) if 0 <= r < len(rows) else None for r in cand_rows]
    kept, _ = _filter(x64, ocfg, lst)
    seen = {target_sig} if target_sig >= 0 else set()
    counts, pos, md = {}, [], []
    for i in kept:
        p = i - by_id
        if p < 0:
            continue
        s = cand_sig[p]
        if s < 0 or s in seen:
            continue
        seen.add(s)
        d = None
        if mood is not None:
            if not mood_ok[p]:
                continue
            d = sum(abs(float(t) - float(c)) for t, c in zip(target_mood, mood[p])) / 6   # Python's own sum
            if not d <= cfg.mood_threshold:
                continue
        if cfg.cap > 0:
            a = cand_raw[p]
            if a < 0 or counts.get(a, 0) >= cfg.cap:
                continue
            counts[a] = counts.get(a, 0) + 1
        pos.append(p)
        md.append(d)
        if len(pos) >= n:
            break
    return np.array(pos, dtype=np.int32), (None if mood is None else np.array(md, dtype=np.float64))
