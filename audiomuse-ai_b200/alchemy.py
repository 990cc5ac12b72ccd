"""The Song Alchemy request (tasks/song_alchemy.py:371-1115, song_alchemy) on the device index.

The reference asks find_nearest_neighbors_by_vector for 3 n neighbours of the add centroid (its by-vector chain:
distance filter, a quadratic same-song dedupe, the raw-author cap), then fetches one vector per candidate three times
over: for the subtract filter, for the local projection and for the displayed distances.  Here the add centroid's
k-NN list comes from one query, the list's details from one get_score_data_by_ids, and one am_knn_alchemy call runs the
chain, takes out the add and subtract songs, applies the subtract filter and measures both distances in float64,
gathering the survivors' rows for the projection when the precomputed map does not cover them all.

Everything else is the reference's: the centroids (_compute_centroid_from_items), the add and subtract points, the
precomputed map and artist-component projections, _project_with_discriminant / _project_to_2d for the points the map
lacks, and the temperature sampling with the module-level `random`, so equal distances and an equal generator state
give the same draws.  make_song_alchemy(sa, vm) looks every helper up on the reference's song_alchemy (sa) and
voyager_manager (vm) modules, and on app_helper / app_helper_artist, at call time.
"""
from __future__ import annotations

import importlib
import logging
import math
import random
from collections import namedtuple

import numpy as np

from . import _lib
from .by_vector import Keys, candidate_keys, chain_config, query_size

logger = logging.getLogger(__name__)

# the projection-id prefixes of each side's songs, anchors, moods and artist components
_Side = namedtuple("_Side", "song anchor mood comp")
_SIDES = (_Side("__add_id__", "__add_anchor__", "__add_mood__", "__add_artist_comp__"),
          _Side("__sub_id__", "__sub_anchor__", "__sub_mood__", "__sub_artist_comp__"))


def config(sa, vm, n, subtract_distance, skip_chain):
    """am_alchemy_cfg and the subtract threshold from the two modules' configuration as they hold it now."""
    p_ang = sa.config.PATH_DISTANCE_METRIC == "angular"
    if subtract_distance is None:
        subtract_distance = (sa.config.ALCHEMY_SUBTRACT_DISTANCE_ANGULAR if p_ang
                             else sa.config.ALCHEMY_SUBTRACT_DISTANCE_EUCLIDEAN)
    return _lib.AlchemyCfg(
        **chain_config(vm, bool(vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT)), path_metric=0 if p_ang else 1, n=int(n),
        skip_chain=int(skip_chain), subtract_threshold=float(subtract_distance))


def sample(ids, distances, temperature, n):
    """song_alchemy.py:959-1049: the best n by distance (stable) at temperature 0, else n weighted draws without
    replacement from softmax(-distance / temperature), with `random` as the reference draws them."""
    def best():
        return sorted(ids, key=lambda x: distances.get(x, float("inf")))[:n]

    if not ids:
        return []
    try:
        if float(temperature) == 0.0:
            return best()
        logits = [-float(distances[i]) / temperature for i in ids]
        top = max(logits)
        w = [math.exp(t - top) for t in logits]
        total = sum(w)
        avail, probs = list(ids), ([1.0 / len(w)] * len(w) if total <= 0 else [e / total for e in w])
        chosen = []
        for _ in range(min(n, len(avail))):
            s = sum(probs)
            if s <= 0:
                k = random.randrange(len(avail))
            else:
                r, acc, k = random.random() * s, 0.0, 0
                for j, p in enumerate(probs):
                    acc += p
                    if r <= acc:
                        k = j
                        break
            chosen.append(avail.pop(k))
            probs.pop(k)
        return chosen
    except Exception as e:
        logger.warning(f"Sampling failed, falling back to deterministic selection: {e}")
        return best()


def _anchor_vector(anchor_id):
    anchor = importlib.import_module("app_helper").get_alchemy_anchor_by_id(anchor_id)
    if anchor and anchor.get("centroid") and isinstance(anchor["centroid"], list):
        return anchor, np.array(anchor["centroid"], dtype=float)
    return anchor, None


def _points(sa, items, side):
    """The side's own points, song_alchemy.py:497-619: (projection ids, their vectors, the metadata list), songs
    first, then anchors, moods and the artists' GMM components (metadata only)."""
    pids, vecs, meta = [], [], []
    songs = [it for it in items if it.get("type") == "song"]
    if songs:
        details = {d["item_id"]: d for d in sa.get_score_data_by_ids([it["id"] for it in songs])}
        for it in songs:
            v = sa.get_vector_by_id(it["id"])
            if v is not None:
                d = details.get(it["id"], {})
                pids.append(side.song + it["id"])
                vecs.append(np.array(v, dtype=float))
                meta.append({"item_id": it["id"], "title": d.get("title"), "author": d.get("author"), "type": "song"})
    for it in items:
        if it.get("type") == "anchor":
            anchor, v = _anchor_vector(it["id"])
            if v is not None:
                pids.append(side.anchor + it["id"])
                vecs.append(v)
                meta.append({"item_id": it["id"], "title": anchor.get("name", "Anchor"), "author": "", "type": "anchor"})
    for it in items:
        if it.get("type") == "mood":
            v = sa._get_mood_centroid_vector(it["id"])
            if v is not None:
                pids.append(side.mood + it["id"])
                vecs.append(v)
                meta.append({"item_id": it["id"], "title": sa._get_mood_label(it["id"]), "author": "", "type": "mood"})
    for it in items:
        if it.get("type") == "artist":
            _, weights = sa._get_artist_gmm_vectors_and_weights(it["id"])
            for ci, w in enumerate(weights):
                name = importlib.import_module("app_helper_artist").get_artist_name_by_id(it["id"]) or it["id"]
                meta.append({"item_id": f"{it['id']}_comp{ci}", "title": f"Component {ci + 1} (w={w:.2f})",
                             "author": name, "is_artist_component": True, "weight": w})
    return pids, vecs, meta


def _map_coords(sa):
    """The precomputed main map (item id -> coordinate) and artist-component projections, song_alchemy.py:646-680."""
    try:
        id_map, proj = sa.load_map_projection("main_map")
    except Exception:
        id_map, proj = None, None
    to_coord = {}
    if id_map is not None and proj is not None:
        try:
            to_coord = {str(i): (float(c[0]), float(c[1])) for i, c in zip(id_map, proj.tolist())}
        except Exception:
            to_coord = {}
    comp = {}
    try:
        cache = importlib.import_module("app_helper").ARTIST_PROJECTION_CACHE
        if cache:
            cmap, cproj = cache.get("component_map", []), cache.get("projection")
            if cproj is not None and len(cmap) > 0:
                for k, info in enumerate(cmap[:len(cproj)]):
                    comp[f"{info['artist_id']}_{info['component_idx']}"] = (float(cproj[k][0]), float(cproj[k][1]))
    except Exception as e:
        logger.warning(f"Failed to load artist projection cache: {e}")
    return to_coord, comp


def _member_centroid(sa, items, mood_prefix, to_coord, comp, proj_map):
    """song_alchemy.py:749-797: the weighted mean of the side's members' map coordinates, or None."""
    coords, weights = [], []
    for it in items:
        t = it.get("type")
        c = (to_coord.get(str(it["id"])) if t in ("song", "anchor")
             else proj_map.get(mood_prefix + it["id"]) if t == "mood" else None)
        if c is not None:
            coords.append(np.array(c, dtype=float))
            weights.append(1.0)
    for it in items:
        if it.get("type") == "artist":
            _, ws = sa._get_artist_gmm_vectors_and_weights(it["id"])
            for ci, w in enumerate(ws):
                c = comp.get(f"{it['id']}_{ci}")
                if c is not None:
                    coords.append(np.array(c, dtype=float))
                    weights.append(w)
    if not coords:
        return None
    w = np.array(weights)
    m = np.sum(np.vstack(coords) * (w / np.sum(w))[:, np.newaxis], axis=0)
    return float(m[0]), float(m[1])


def _project(sa, proj_ids, vectors, meta, to_coord, comp):
    """song_alchemy.py:643-897: every projection id's 2-D point from the precomputed map where it has one; the rest
    are projected locally together (discriminant, else PCA).  `vectors` maps each projection id to its vector.
    Returns (proj_map, the projection used)."""
    proj_map, missing = {}, []
    for pid in proj_ids:
        if pid in ("__add_centroid__", "__subtract_centroid__"):
            continue
        key = pid
        for side in _SIDES:
            if pid.startswith(side.song):
                key = pid[len(side.song):]
        c = to_coord.get(str(key))
        if c is not None:
            proj_map[pid] = c
        else:
            missing.append(pid)
    for side, side_meta in zip(_SIDES, meta):
        for m in side_meta:
            parts = m["item_id"].split("_comp") if m.get("is_artist_component") else []
            if len(parts) == 2:
                c = comp.get(f"{parts[0]}_{int(parts[1])}")
                if c is not None:
                    proj_map[f"{side.comp}{parts[0]}_{int(parts[1])}"] = c
    # the ids still missing, with their vectors, go after the first list (the reference extends the same list, and
    # pairs its entries with the local projections in that order)
    local_vecs = []
    for pid in proj_ids:
        if pid in proj_map or pid in ("__add_centroid__", "__subtract_centroid__") or vectors.get(pid) is None:
            continue
        missing.append(pid)
        local_vecs.append(np.array(vectors[pid], dtype=float))
    used = "none"
    if local_vecs:
        try:
            local = None
            if len(local_vecs) >= 4:
                try:
                    add_v, sub_v = [], []
                    for pid in missing:
                        v = local_vecs[missing.index(pid)]
                        if pid.startswith(("__add_id__", "__add_artist_comp__")):
                            add_v.append(v)
                        elif pid.startswith(("__sub_id__", "__sub_artist_comp__")):
                            sub_v.append(v)
                    if add_v and sub_v:
                        local = sa._project_with_discriminant(add_v, sub_v, local_vecs)
                        used = "discriminant"
                except Exception:
                    local = None
            if local is None:
                try:
                    local = sa._project_to_2d(local_vecs)
                    used = "pca"
                except Exception:
                    local = [(0.0, 0.0) for _ in local_vecs]
            for pid, c in zip(missing, local):
                proj_map[pid] = (float(c[0]), float(c[1]))
        except Exception as e:
            logger.warning(f"Failed to compute local projections for missing ids: {e}")
    for pid in proj_ids:
        proj_map.setdefault(pid, (0.0, 0.0))
    return proj_map, used


def _with_album(d):
    for k in ("album", "album_artist"):
        if k not in d or not d[k]:
            d[k] = "Unknown"
    return d


def make_song_alchemy(sa, vm):
    """song_alchemy(add_items, subtract_items, add_ids, subtract_ids, n_results, subtract_distance, temperature) on
    the device: the same return dict as song_alchemy.py:371-1115, the same ValueError for an empty ADD set and the
    same empty results for a missing centroid or no neighbours."""

    def song_alchemy(add_items=None, subtract_items=None, add_ids=None, subtract_ids=None, n_results: int = None,
                     subtract_distance: float = None, temperature: float = None) -> dict:
        cfg_mod = sa.config
        n_results = min(cfg_mod.ALCHEMY_DEFAULT_N_RESULTS if n_results is None else n_results,
                        cfg_mod.ALCHEMY_MAX_N_RESULTS)
        if add_items is None and add_ids is not None:
            add_items = [{"type": "song", "id": i} for i in add_ids]
        if subtract_items is None and subtract_ids is not None:
            subtract_items = [{"type": "song", "id": i} for i in subtract_ids]
        if not add_items:
            raise ValueError("At least one item must be in the ADD set")
        empty = {"results": [], "filtered_out": [], "centroid_2d": None}
        add_c = sa._compute_centroid_from_items(add_items)
        if add_c is None:
            return empty
        sub_c = sa._compute_centroid_from_items(subtract_items) if subtract_items else None
        try:
            temperature = float(cfg_mod.ALCHEMY_TEMPERATURE if temperature is None else temperature)
        except Exception:
            logger.warning(f"Invalid temperature value passed to song_alchemy: {temperature!r}; falling back to "
                           "config default")
            try:
                temperature = float(cfg_mod.ALCHEMY_TEMPERATURE)
            except Exception:
                temperature = 1.0

        # the neighbour list: the reference's own by-id query for one song at temperature 0 (:423-427), else the add
        # centroid's k-NN list for the chain on the device
        listed = None
        if temperature == 0.0 and len(add_items) == 1 and add_items[0].get("type") == "song":
            try:
                listed = [nb["item_id"] for nb in sa.find_nearest_neighbors_by_id(add_items[0]["id"], n=n_results)
                          or []]
            except Exception:
                listed = None
        if listed is None:
            if vm.voyager_index is None or vm.id_map is None:
                raise RuntimeError("Voyager index is not loaded in memory.")
            k = query_size(n_results * 3, bool(vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT), len(vm.voyager_index))
            ids = vm.voyager_index.query(np.asarray(add_c, dtype=np.float32), k=k)[0] if k > 0 else []
            items = [vm.id_map.get(int(i)) for i in ids]
            items = [i for i in items if i is not None]
            skip_chain = False
        else:
            if not listed:
                return empty
            items, skip_chain = listed, True
        details = {d["item_id"]: d for d in sa.get_score_data_by_ids(items)} if items else {}
        sig, raw = Keys(), Keys()
        cand_sig, cand_raw = candidate_keys(items, details, sig, raw)
        own = [it["id"] for it in add_items + (subtract_items or []) if it.get("type") == "song" and it.get("id")]
        excl = list(dict.fromkeys(vm.reverse_id_map[i] for i in own if i in vm.reverse_id_map))
        to_coord, comp = _map_coords(sa)
        need_rows = any(str(i) not in to_coord for i in items)
        cfg = config(sa, vm, max(1, n_results * 3), subtract_distance, skip_chain)
        pos, status, _, dadd, rows = vm.voyager_index.alchemy(
            cfg, add_c, sub_c, [vm.reverse_id_map.get(i, -1) for i in items], cand_sig, cand_raw, len(sig), excl,
            rows=need_rows)
        if not skip_chain and len(pos) == 0:
            return empty
        cand = [items[p] for p, s in zip(pos, status) if s == 1][:max(n_results * 3, n_results)]
        filtered_out = [items[p] for p, s in zip(pos, status) if s == 2]
        distances = {items[p]: float(d) for p, s, d in zip(pos, status, dadd) if s == 1}
        row_of = {} if rows is None else {items[p]: r for p, s, r in zip(pos, status, rows) if s}

        # projection ids and vectors in the reference's order: each side's points, the centroids, the candidates
        # and the filtered-out ones
        proj_ids, meta, vectors = [], [], {}
        for side, side_items in zip(_SIDES, (add_items, subtract_items or [])):
            pids, vecs, side_meta = _points(sa, side_items, side)
            proj_ids += pids
            meta.append(side_meta)
            for p, v in zip(pids, vecs):
                vectors.setdefault(p, v)
        proj_ids.append("__add_centroid__")
        if sub_c is not None:
            proj_ids.append("__subtract_centroid__")
        proj_ids += cand + filtered_out
        vectors.update(row_of)
        proj_map, used = _project(sa, proj_ids, vectors, meta, to_coord, comp)
        try:
            members = [_member_centroid(sa, its, prefix, to_coord, comp, proj_map) if its else None
                       for its, prefix in ((add_items, "__add_mood__"), (subtract_items, "__sub_mood__"))]
            for key, c in zip(("__add_centroid__", "__subtract_centroid__"), members):
                if c is not None:
                    proj_map[key] = c
        except Exception as e:
            logger.warning(f"Failed to compute centroid from member coords: {e}")

        for i in cand:
            if i in details:
                _with_album(details[i])
        scored = [i for i in cand if i in details and i in distances]
        results = []
        for i in sample(scored, distances, temperature, n_results):
            d = details.get(i, {})
            d["distance"] = distances.get(i)
            d["embedding_2d"] = proj_map.get(i)
            results.append(_with_album(d))
        filtered = []
        for i in filtered_out:
            if i in details:
                d = details[i]
                d["embedding_2d"] = proj_map.get(i)
                filtered.append(_with_album(d))

        points = []
        for side, side_meta in zip(_SIDES, meta):
            pts = []
            for m in side_meta:
                if m.get("is_artist_component"):
                    pid = f"{side.comp}{m['item_id'].rsplit('_comp', 1)[0]}_{m['item_id'].split('_comp')[1]}"
                else:
                    pid = {"anchor": side.anchor, "mood": side.mood}.get(m.get("type"), side.song) + m["item_id"]
                pts.append({**m, "embedding_2d": proj_map.get(pid)})
            points.append(pts)
        centroid_2d = proj_map.get("__add_centroid__")
        return {"results": results, "filtered_out": filtered, "centroid_2d": centroid_2d,
                "add_centroid_2d": centroid_2d, "subtract_centroid_2d": proj_map.get("__subtract_centroid__"),
                "add_centroid_vector": add_c.tolist(),
                "subtract_centroid_vector": sub_c.tolist() if sub_c is not None else None,
                "add_points": points[0], "sub_points": points[1], "projection": used}

    return song_alchemy
