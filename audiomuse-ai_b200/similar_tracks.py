"""The plain similar-tracks requests of tasks/voyager_manager.py on the device index.

find_nearest_neighbors_by_id without the radius walk (:1493-1545) and find_nearest_neighbors_by_vector (:1547-1657)
each make one k-NN query, then run their filters in Python: the distance filter, a name dedupe (O(k^2) for the
by-vector one), the mood filter (by id) and the artist cap, with several database reads along the way.  Here one
get_score_data_by_ids read supplies titles, authors and other_features for every stage, and one am_knn_similar call
runs the stages on the device in k-NN order and stops after n songs.  get_max_distance_for_id (:1660-1702) asked the
index for every row (query(k=len(index)), a full sort and a copy of N ids and distances to the host) to keep one
maximum; am_knn_farthest finds that row in one pass.

make_find_nearest_neighbors_by_id(vm), make_find_nearest_neighbors_by_vector(vm) and make_get_max_distance_for_id(vm)
return the drop-ins; they read every configuration value and helper on the reference's voyager_manager (vm) at call
time, as the reference reads its own module globals.  The k-NN queries keep the reference's error handling (a
RecallError or any other failure of the query gives [] or None); a failing am_knn_similar / am_knn_farthest raises
B200Error.
"""
from __future__ import annotations

import logging
import sys

import numpy as np

from . import _lib
from .by_vector import Keys, candidate_keys, chain_config, query_size, signature

logger = logging.getLogger(__name__)

MOOD_FEATURES = ("danceable", "aggressive", "happy", "party", "relaxed", "sad")   # voyager_manager.py:775


def parse_mood_features(other_features):
    """_parse_mood_features (voyager_manager.py:824-838): "key:value" pairs split on ',' (pairs without ':' are
    skipped), keys and values stripped, values through float(); any failure gives {}."""
    try:
        features = {}
        for pair in other_features.split(","):
            if ":" in pair:
                key, value = pair.split(":", 1)
                features[key.strip()] = float(value.strip())
        return features
    except Exception:
        return {}


def mood_row(features):
    """The six features in MOOD_FEATURES order, 0.0 where missing (:790)."""
    return [features.get(f, 0.0) for f in MOOD_FEATURES]


def config(vm, eliminate_duplicates):
    """am_similar_cfg from voyager_manager's configuration as it holds it now."""
    ch = chain_config(vm, eliminate_duplicates)
    return _lib.SimilarCfg(
        metric=ch.pop("voyager_metric"), cap=ch.pop("voyager_cap"), **ch,
        mood_sum=1 if sys.version_info >= (3, 12) else 0,   # sum() of floats is compensated from CPython 3.12 on
        mood_threshold=float(vm.MOOD_SIMILARITY_THRESHOLD))


def by_id_query_size(n, eliminate_duplicates, radius_similarity, mood_similarity, size):
    """voyager_manager.py:1418-1440: the neighbours find_nearest_neighbors_by_id asks the index for.  The mood term
    reads the caller's mood_similarity, not the configured default, as the reference does."""
    if radius_similarity or eliminate_duplicates:
        q = n + max(20, int(n * 3)) + 1
    else:
        q = n + max(3, int(n * 0.20)) + 1
    if mood_similarity:
        q = n + max(20, int(n * (8 if eliminate_duplicates else 4))) + 1
    return min(q, size)


def _query(vm, vector, k):
    """(ids, distances) of the index query, or None where the reference returns early (RecallError or any other
    failure of the query)."""
    try:
        return vm.voyager_index.query(vector, k=k)
    except vm.voyager.RecallError as e:
        logger.warning(f"Voyager RecallError: {e}. Returning empty list.")
    except Exception as e:
        logger.error(f"An unexpected error occurred during Voyager query: {e}", exc_info=True)
    return None


def _run(vm, items, distances, n, eliminate_duplicates, target=None, target_details=None, mood=False):
    """One am_knn_similar call over the request's list (item ids in k-NN order); returns the reference's dicts."""
    from app_helper import get_score_data_by_ids

    if not items or n <= 0:
        return []
    details = {d["item_id"]: d for d in get_score_data_by_ids(items)}
    sig, raw = Keys(), Keys()
    target_sig = sig(signature(target_details)) if target_details is not None else -1
    cand_sig, cand_raw = candidate_keys(items, details, sig, raw)
    table = ok = target_mood = None
    if mood:
        t = target_details.get("other_features")
        tf = parse_mood_features(t) if t else {}
        if tf:   # no parsable target features: the stage does not run (:731-738)
            target_mood = mood_row(tf)
            parsed = [parse_mood_features(details[i]["other_features"])
                      if i in details and details[i].get("other_features") else {} for i in items]
            table = [mood_row(f) for f in parsed]
            ok = [1 if f else 0 for f in parsed]
        else:
            logger.warning(f"No mood features found for target song {target}. Skipping mood filtering.")
    pos, md = vm.voyager_index.similar(
        config(vm, eliminate_duplicates), None if target is None else vm.reverse_id_map[target], target_sig,
        [vm.reverse_id_map.get(i, -1) for i in items], cand_sig, cand_raw, len(sig), n, mood=table, mood_ok=ok,
        target_mood=target_mood)
    out = [{"item_id": items[p], "distance": distances[p]} for p in pos]
    if md is not None:
        for r, d in zip(out, md):
            r["mood_distance"] = float(d)
    return out


def make_find_nearest_neighbors_by_id(vm):
    """find_nearest_neighbors_by_id(target_item_id, n, eliminate_duplicates, mood_similarity, radius_similarity) on
    the device: the same list as voyager_manager.py:1372-1545.  radius_similarity hands the candidates to
    vm._radius_walk_get_candidates and vm._execute_radius_walk, looked up at call time."""

    def find_nearest_neighbors_by_id(target_item_id: str, n: int = 10, eliminate_duplicates: bool | None = None,
                                     mood_similarity: bool | None = None, radius_similarity: bool | None = None):
        if vm.voyager_index is None or vm.id_map is None or vm.reverse_id_map is None:
            raise RuntimeError("Voyager index is not loaded in memory. It may be missing, empty, or the server failed "
                               "to load it on startup.")
        from app_helper import get_score_data_by_ids

        target_list = get_score_data_by_ids([target_item_id])
        if not target_list:
            logger.error(f"Could not retrieve details for the target song {target_item_id}. Aborting neighbor search.")
            return []
        target_details = target_list[0]
        target_vid = vm.reverse_id_map.get(target_item_id)
        if target_vid is None:
            logger.warning(f"Target item_id '{target_item_id}' not found in the loaded Voyager index map.")
            return []
        try:
            query_vector = vm.voyager_index.get_vector(target_vid)
        except Exception as e:
            logger.error(f"Could not retrieve vector for Voyager ID {target_vid} (item_id: {target_item_id}): {e}")
            return []
        if radius_similarity is None:
            radius_similarity = vm.SIMILARITY_RADIUS_DEFAULT
        if eliminate_duplicates is None:
            eliminate_duplicates = vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT
        k = by_id_query_size(n, eliminate_duplicates, radius_similarity, mood_similarity, len(vm.voyager_index))
        if k <= 1:
            ids, dists = [], []
        else:
            res = _query(vm, query_vector, k)
            if res is None:
                return []
            ids, dists = res
        items, distances = [], []
        for vid, dist in zip(ids, dists):
            item_id = vm.id_map.get(vid)
            if item_id and item_id != target_item_id:
                items.append(item_id)
                distances.append(float(dist))
        if radius_similarity:
            from app_helper import get_db

            initial = [{"item_id": i, "distance": d} for i, d in zip(items, distances)]
            candidates = vm._radius_walk_get_candidates(
                target_item_id=target_item_id, anchor_vector=query_vector, initial_results=initial, db_conn=get_db(),
                original_song_details=target_details, eliminate_duplicates=eliminate_duplicates,
                mood_similarity=mood_similarity)
            return vm._execute_radius_walk(target_item_id=target_item_id, n=n, candidate_data=candidates,
                                           original_song_details=target_details,
                                           eliminate_duplicates=eliminate_duplicates)
        mood = vm.MOOD_SIMILARITY_ENABLE if mood_similarity is None else mood_similarity
        return _run(vm, items, distances, n, eliminate_duplicates, target=target_item_id,
                    target_details=target_details, mood=bool(mood))

    return find_nearest_neighbors_by_id


def make_find_nearest_neighbors_by_vector(vm):
    """find_nearest_neighbors_by_vector(query_vector, n, eliminate_duplicates) on the device: the same list as
    voyager_manager.py:1547-1657."""

    def find_nearest_neighbors_by_vector(query_vector: np.ndarray, n: int = 100, eliminate_duplicates: bool | None = None):
        if vm.voyager_index is None or vm.id_map is None:
            raise RuntimeError("Voyager index is not loaded in memory.")
        if eliminate_duplicates is None:
            eliminate_duplicates = vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT
        k = query_size(n, eliminate_duplicates, len(vm.voyager_index))
        if k <= 0:
            ids, dists = [], []
        else:
            res = _query(vm, query_vector, k)
            if res is None:
                return []
            ids, dists = res
        items, distances = [], []
        for vid, dist in zip(ids, dists):
            item_id = vm.id_map.get(vid)
            if item_id is not None:
                items.append(item_id)
                distances.append(float(dist))
        return _run(vm, items, distances, n, eliminate_duplicates)

    return find_nearest_neighbors_by_vector


def make_get_max_distance_for_id(vm):
    """get_max_distance_for_id(target_item_id) on the device: the same {max_distance, farthest_item_id} as
    voyager_manager.py:1660-1702, None for an item that is not in the index."""

    def get_max_distance_for_id(target_item_id: str):
        if vm.voyager_index is None or vm.id_map is None or vm.reverse_id_map is None:
            raise RuntimeError("Voyager index is not loaded in memory. It may be missing, empty, or the server failed "
                               "to load it on startup.")
        target_vid = vm.reverse_id_map.get(target_item_id)
        if target_vid is None:
            return None
        try:
            dist, far = vm.voyager_index.farthest(target_vid)
        except KeyError as e:
            logger.error(f"Could not retrieve vector for Voyager ID {target_vid} (item_id: {target_item_id}): {e}")
            return None
        if far is None:
            return {"max_distance": 0.0, "farthest_item_id": None}
        return {"max_distance": float(dist), "farthest_item_id": vm.id_map.get(far)}

    return get_max_distance_for_id
