"""Oracle: Song Alchemy's candidate list and sampling (tasks/song_alchemy.py:420-486, :916-930, :959-1049) in
float64.  TEST INFRASTRUCTURE ONLY.

Restates, over an in-memory library (the index's stored rows, item "item<i>" at row i) and a metadata table:
  1. the by-vector chain of find_nearest_neighbors_by_vector (voyager_manager.py:1589-1657) on the add centroid's
     k-NN list (exact float64 distance, ties by lower row), cut at [:n] -- or, for the single-song temperature-0
     branch, the given neighbour list as it is;
  2. the add and subtract songs taken out;
  3. the subtract filter: d(sub, v) >= threshold keeps v;
  4. the distance of every kept candidate to the add centroid;
and the temperature sampling over those distances.  The two centroid distances use song_alchemy's own float64
formulas, so they agree bit for bit with the reference's; the chain's filter distances are float64 where the
reference's are float32.

Besides the answer it reports the gaps that decided it: `filter_gap` (closest any filter distance came to its
threshold), `sub_gap` (closest a subtract distance came to its threshold), `knn_gap` (closest two neighbours came that
the k-NN prefix keeps apart) and, from sample(), `sample_gap` (closest a draw came to a cumulative boundary, or two
sorted distances at temperature 0).
"""
from __future__ import annotations

import math
import random

import numpy as np

from audiomuse_ai_b200 import song_path as sp
from oracle import knn as oknn
from oracle import song_path as osp


def centroid_distance(c, v, metric):
    """song_alchemy.py:469-479 / :923-929: 'angular' arccos(clip(c / (|c| or 1) . v / (|v| or 1))) / pi, else
    ||c - v||, in float64."""
    c, v = np.asarray(c, dtype=float), np.asarray(v, dtype=float)
    if metric == "angular":
        a = c / (np.linalg.norm(c) or 1.0)
        b = v / (np.linalg.norm(v) or 1.0)
        return float(np.arccos(np.clip(np.dot(a, b), -1.0, 1.0)) / np.pi)
    return float(np.linalg.norm(c - v))


def knn_list(rows, space, vec, k):
    """The k nearest rows to `vec` (float32, as the index takes it), exact float64, ties by lower row, with the
    smallest gap between distances the prefix keeps apart."""
    q = np.asarray(vec, np.float32)
    dist = oknn.exact_scores_f64(rows, q[None, :], oknn.COSINE if space == "cosine" else oknn.EUCLIDEAN)[0]
    order = np.lexsort((np.arange(len(rows)), dist))
    ds = dist[order]
    inner = np.diff(ds[:k])
    if k < len(rows):
        inner = np.append(inner, ds[k] - ds[k - 1])
    inner = inner[inner > 0]
    return [f"item{r}" for r in order[:k]], float(inner.min()) if len(inner) else np.inf


def keys(table, items):
    """item -> (its (author, title) signature, its raw author or None when falsy); no entry: no details."""
    return {i: (sp.signature(table[i]), table[i].get("author") or None) for i in items if i in table}


def chain(rows, keyed, cfg, items, n):
    """find_nearest_neighbors_by_vector after its query: the distance filter, the same-song dedupe and the raw-author
    cap, cut at [:n].  keyed: keys().  cfg: VOYAGER_METRIC, THRESHOLD_COSINE, THRESHOLD_EUCLIDEAN, LOOKBACK, BATCH,
    MAX_SONGS_PER_ARTIST, ELIMINATE_DUPLICATES.  Returns (the surviving items, filter_gap)."""
    x64 = np.asarray(rows, np.float32).astype(np.float64)
    vmet = "cosine" if cfg["VOYAGER_METRIC"] == "angular" else "euclidean"
    thr = cfg["THRESHOLD_COSINE"] if vmet == "cosine" else cfg["THRESHOLD_EUCLIDEAN"]
    lookback, batch, cap = cfg["LOOKBACK"], cfg["BATCH"], cfg["MAX_SONGS_PER_ARTIST"]
    gap = np.inf
    if lookback > 0:
        kept, batched, base = [], len(items) > batch, 0
        for i, it in enumerate(items):
            if batched and i % batch == 0:
                base = len(kept)
            close = False
            for o in kept[max(0, (base if batched else len(kept)) - lookback):]:
                dd = osp.direct(x64[int(it[4:])], x64[int(o[4:])], vmet)
                if np.isfinite(dd):
                    gap = min(gap, abs(dd - thr))
                close = close or dd < thr
            if not close:
                kept.append(it)
        items = kept
    seen, unique = set(), []
    for it in items:
        if it not in keyed or keyed[it][0] in seen:
            continue
        seen.add(keyed[it][0])
        unique.append(it)
    if cfg["ELIMINATE_DUPLICATES"] and cap is not None and cap > 0:
        counts, capped = {}, []
        for it in unique:
            a = keyed[it][1]
            if a is not None and counts.get(a, 0) < cap:
                capped.append(it)
                counts[a] = counts.get(a, 0) + 1
        unique = capped
    return unique[:n], gap


def candidates(rows, keyed, cfg, path_metric, add_c, sub_c, sub_threshold, listed, excluded, n, skip_chain):
    """Steps 1-4 over the k-NN list (or neighbour list) `listed`, keyed by keys(): returns a dict with the chain's survivors
    (`chain`), the kept candidates and the filtered-out ones in order, `distances` (kept item -> d(add)),
    `dsub` (item -> d(sub)), filter_gap and sub_gap."""
    x64 = np.asarray(rows, np.float32).astype(np.float64)
    survivors, filter_gap = (list(listed), np.inf) if skip_chain else chain(rows, keyed, cfg, listed, n)
    kept, filtered, dsub, sub_gap = [], [], {}, np.inf
    for it in survivors:
        if it in excluded:
            continue
        v = x64[int(it[4:])]
        if sub_c is not None:
            dsub[it] = centroid_distance(sub_c, v, path_metric)
            sub_gap = min(sub_gap, abs(dsub[it] - sub_threshold))
            if not dsub[it] >= sub_threshold:
                filtered.append(it)
                continue
        kept.append(it)
    kept = kept[:n]
    distances = {it: centroid_distance(add_c, x64[int(it[4:])], path_metric) for it in kept}
    return {"chain": survivors, "kept": kept, "filtered_out": filtered, "distances": distances, "dsub": dsub,
            "filter_gap": filter_gap, "sub_gap": sub_gap}


def sample(ids, distances, temperature, n, seed):
    """song_alchemy.py:959-1049 from random.seed(seed): (the chosen ids in order, sample_gap)."""
    if not ids:
        return [], np.inf
    if temperature == 0.0:
        order = sorted(ids, key=lambda i: distances[i])
        ds = [distances[i] for i in order[:n + 1]]
        gaps = [b - a for a, b in zip(ds, ds[1:]) if b > a]
        return order[:n], min(gaps, default=np.inf)
    rng = random.Random(seed)
    logits = [-float(distances[i]) / temperature for i in ids]
    w = [math.exp(t - max(logits)) for t in logits]
    probs = [e / sum(w) for e in w]
    avail, chosen, gap = list(ids), [], np.inf
    for _ in range(min(n, len(avail))):
        s = sum(probs)
        r = rng.random() * s
        acc, k = 0.0, 0
        for j, p in enumerate(probs):
            lo = acc
            acc += p
            if r <= acc:
                k = j
                gap = min(gap, r - lo, acc - r)
                break
        chosen.append(avail.pop(k))
        probs.pop(k)
    return chosen, gap
