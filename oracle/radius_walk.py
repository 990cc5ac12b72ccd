"""Oracle: the similar-tracks radius walk, tasks/voyager_manager.py:941-1367 (_execute_radius_walk), restated line by
line over arrays.  TEST INFRASTRUCTURE ONLY.

The candidates come in the order _radius_walk_get_candidates (:842-938) leaves them: vectors[i] is the stored vector
of candidate i (None when it is not in the index: the reference drops it, :920-921), authors[i] its author (any value;
only truthiness and equality matter, as in the reference).  Two arithmetic modes:

  * "reference": the reference's own numpy float32 get_direct_distance calls (:99-142, oracle/knn.py), one pair at a
    time, so that every anchor distance and every score is the reference's bit for bit;
  * "float64": the same walk on float64 distances from the float32 vectors, the arithmetic of am_knn_radius_walk.

Besides the walk, the result carries the smallest gap (in the mode's arithmetic) that decided an ordering: between
neighbours of the anchor-distance sort, and between each greedy step's best score and its runner-up.  Exact ties (duplicate rows) are
not counted: they tie in every arithmetic and fall to the input order in the reference and on the device alike.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import knn as oknn

BUCKET_SIZE = 50   # voyager_manager.py:956


def distance64(v1, v2, metric: str) -> float:
    """get_direct_distance (voyager_manager.py:99-142) in float64 from the float32 vectors."""
    if v1 is None or v2 is None:
        return math.inf
    a = np.asarray(v1, dtype=np.float32).astype(np.float64)
    b = np.asarray(v2, dtype=np.float32).astype(np.float64)
    if metric != "angular":
        return float(np.sqrt(np.sum((a - b) ** 2)))
    den = math.sqrt(float(np.dot(a, a))) * math.sqrt(float(np.dot(b, b)))
    if den == 0.0:
        return math.inf
    return 1.0 - min(1.0, max(-1.0, float(np.dot(a, b)) / den))


def distance_ref(v1, v2, metric: str) -> float:
    """get_direct_distance as the reference computes it (numpy float32)."""
    if metric == "angular":
        return oknn.direct_cosine_distance(v1, v2)
    return oknn.direct_euclidean_distance(v1, v2)


def radius_walk(vectors, anchor, authors, n: int, eliminate_duplicates: bool, max_songs_per_artist, metric: str,
                mode: str = "reference"):
    """Returns {"positions": candidate positions in walk order, "distances": their anchor distances (the mode's),
    "sort_gap": ..., "score_gap": ...}.  max_songs_per_artist: config.MAX_SONGS_PER_ARTIST (None disables the artist
    rules, like <= 0); metric: config.VOYAGER_METRIC."""
    if mode not in ("reference", "float64"):
        raise ValueError(mode)
    dist = distance_ref if mode == "reference" else (lambda a, b, m: distance64(a, b, m))
    cap = max_songs_per_artist
    out = {"positions": [], "distances": [], "sort_gap": math.inf, "score_gap": math.inf}

    # _radius_walk_get_candidates :918-935: candidates with a vector, float32 vectors, distance to the anchor
    candidate_data = []
    for pos, vec in enumerate(vectors):
        if vec is None:
            continue
        v = np.asarray(vec).astype(np.float32)
        candidate_data.append({"item_id": pos, "vector": v, "dist_anchor": dist(v, anchor, metric),
                               "author": authors[pos]})
    if not candidate_data or n <= 0:
        return out

    # Step 1 (:968-993): stable sort by the anchor distance, buckets of 50 with the distance as float32
    candidate_data.sort(key=lambda x: x["dist_anchor"])
    keys = [c["dist_anchor"] for c in candidate_data]
    out["sort_gap"] = min((b - a for a, b in zip(keys, keys[1:]) if math.isfinite(b) and a != b), default=math.inf)
    num_buckets = int(math.ceil(len(candidate_data) / BUCKET_SIZE))
    buckets = []
    for i in range(num_buckets):
        b = candidate_data[i * BUCKET_SIZE:(i + 1) * BUCKET_SIZE]
        buckets.append({"items": b, "ids": [c["item_id"] for c in b],
                        "dist_anchor": np.array([c["dist_anchor"] for c in b], dtype=np.float32)})

    # Step 2 (:1001-1052): the first song, its artist counted globally only
    first_song = candidate_data[0]
    playlist_ids = [first_song["item_id"]]
    used_ids = {first_song["item_id"]}
    selected_vectors = {first_song["item_id"]: first_song["vector"]}
    artist_counts = {}
    if first_song["author"]:
        artist_counts[first_song["author"]] = 1
    artist_bucket_counts = {}
    rules = bool(eliminate_duplicates and cap is not None and cap > 0)
    score_gaps = []

    def refused(author, bucket_artist_set):
        """:1120-1136 / :1188-1211"""
        if not rules or not author:
            return False
        if author in bucket_artist_set:
            return True
        if artist_bucket_counts.get(author, 0) >= 2 and artist_counts.get(author, 0) < cap:
            return True
        return artist_counts.get(author, 0) >= cap

    def take(bucket_items, i, bucket_artist_set):
        """:1141-1161 / :1232-1253"""
        cid = bucket_items[i]["item_id"]
        used_ids.add(cid)
        if len(playlist_ids) < n:
            playlist_ids.append(cid)
        selected_vectors[cid] = bucket_items[i]["vector"]
        if eliminate_duplicates:
            a = bucket_items[i]["author"]
            if a:
                artist_counts[a] = artist_counts.get(a, 0) + 1
                if a not in bucket_artist_set:
                    bucket_artist_set.add(a)
                    artist_bucket_counts[a] = artist_bucket_counts.get(a, 0) + 1

    def walk_single_bucket(bucket_index, start_item_id=None):
        """:1071-1258"""
        bucket = buckets[bucket_index]
        items, cand_ids, cand_anchor = bucket["items"], bucket["ids"], bucket["dist_anchor"]
        remaining = [True] * len(cand_ids)
        bucket_artist_set = set()
        cur_idx = None
        if start_item_id is not None and start_item_id in cand_ids:
            si = cand_ids.index(start_item_id)
            if remaining[si] and cand_ids[si] not in used_ids:
                cur_idx = si
        if cur_idx is None:
            cur_idx = next((i for i, cid in enumerate(cand_ids) if remaining[i] and cid not in used_ids), None)
        if cur_idx is None:
            return
        if cand_ids[cur_idx] not in used_ids and not refused(items[cur_idx]["author"], bucket_artist_set):
            remaining[cur_idx] = False
            take(items, cur_idx, bucket_artist_set)
        else:
            remaining[cur_idx] = False
        while True:
            avail = [i for i, r in enumerate(remaining) if r and cand_ids[i] not in used_ids]
            if not avail:
                break
            cur_vec = selected_vectors[playlist_ids[-1]]
            best_i, best_score = None, float("inf")
            scores = []
            for i in avail:
                if refused(items[i]["author"], bucket_artist_set):
                    continue
                dist_prev = dist(items[i]["vector"], cur_vec, metric)
                score = 0.7 * dist_prev + 0.3 * float(cand_anchor[i])
                scores.append(score)
                if score < best_score:
                    best_score, best_i = score, i
            if best_i is None:
                break
            distinct = sorted(set(x for x in scores if math.isfinite(x)))
            if len(distinct) > 1:
                score_gaps.append(distinct[1] - distinct[0])
            remaining[best_i] = False
            take(items, best_i, bucket_artist_set)

    # Step 3 (:1261-1281): buckets in order until the playlist holds n songs
    buckets_to_check = min(num_buckets, max(3, int(math.ceil(n / BUCKET_SIZE))))
    processed = 0
    while len(playlist_ids) < n and processed < num_buckets:
        for bi in range(processed, min(num_buckets, buckets_to_check)):
            walk_single_bucket(bi, start_item_id=playlist_ids[0] if bi == 0 else None)
            processed += 1
            if len(playlist_ids) >= n:
                break
        if len(playlist_ids) < n and buckets_to_check < num_buckets:
            buckets_to_check = min(num_buckets, max(buckets_to_check + 1, buckets_to_check * 2))

    # _avoid_triple_adjacent (:1287-1318)
    id_to_author = {c["item_id"]: c["author"] for c in candidate_data}
    ids = playlist_ids
    i = 0
    while i <= len(ids) - 3:
        a1, a2, a3 = (id_to_author.get(ids[i + t]) for t in range(3))
        if a1 and a1 == a2 == a3:
            j = next((j for j in range(i + 3, len(ids)) if id_to_author.get(ids[j]) != a1), None)
            if j is not None:
                ids[i + 2], ids[j] = ids[j], ids[i + 2]
                continue
        i += 1

    dist_anchor_map = {c["item_id"]: c["dist_anchor"] for c in candidate_data}
    out["positions"] = ids[:n]
    out["distances"] = [dist_anchor_map[i] for i in ids[:n]]
    out["score_gap"] = min(score_gaps, default=math.inf)
    return out
