"""The Song Path request (tasks/path_manager.py:320-557, find_path_between_songs) on the device index.

The reference runs one centroid job at a time: per job a k-NN query, the by-vector chain of
find_nearest_neighbors_by_vector (voyager_manager.py:1547-1657: distance filter, same-song dedupe, raw-author cap),
two database reads, one get_vector per candidate and Python distance loops.  Here the jobs are planned on the host as
the reference plans them, all their centroids go to the index in one batched query (each job reads a prefix of the
top-k: the index orders by exact distance, ties by lower id, so a prefix of the top-K is the top-k), the candidates'
details come from one get_score_data_by_ids, and one am_knn_song_path call walks every job.  Only a failed job under
path_fix_size costs another round: its merged job is queried alone and the walk resumes at it with the carried state.

make_song_path(vm, pm) returns the drop-in; it looks everything up on the reference's voyager_manager (vm) and
path_manager (pm) modules at call time, as the reference reads its own module globals.
"""
from __future__ import annotations

import logging
from itertools import accumulate

import numpy as np

from . import _lib
from .by_vector import Keys, candidate_keys, chain_config, normalize, query_size, signature

logger = logging.getLogger(__name__)

K_BASE, K_MAX = 10, 1000   # path_manager.py:379-380


def interpolate_centroids(v1, v2, num, metric="euclidean"):
    """path_manager.py:55-103 in float64: SLERP with a linearly interpolated magnitude for 'angular' (straight lines
    for a zero vector or (anti)parallel ends), np.linspace otherwise."""
    a = np.array(v1, dtype=float)
    b = np.array(v2, dtype=float)
    if metric != "angular":
        return np.linspace(a, b, num=num)
    na, nb = np.linalg.norm(a), np.linalg.norm(b)
    if na == 0 or nb == 0:
        return np.linspace(a, b, num=num)
    ua, ub = a / na, b / nb
    theta = np.arccos(np.clip(np.dot(ua, ub), -1.0, 1.0))
    if np.isclose(theta, 0) or np.isnan(theta):
        return np.linspace(a, b, num=num)
    sin_theta = np.sin(theta)
    if np.isclose(sin_theta, 0):
        return np.linspace(a, b, num=num)
    rows = []
    for t in np.linspace(0, 1, num):
        wa = np.sin((1 - t) * theta) / sin_theta
        wb = np.sin(t * theta) / sin_theta
        rows.append((wa * ua + wb * ub) * ((1 - t) * na + t * nb))
    return np.array(rows)


def initial_job_count(num_intermediate, start_neighbours, end_neighbours):
    """path_manager.py:403-413: half the shared neighbourhood of the two ends (or of their union), at least 1."""
    s, e = set(start_neighbours), set(end_neighbours)
    representative = len(s & e) or len(s | e)
    if representative <= 0:
        return num_intermediate
    return int(max(1, min(num_intermediate, representative // 2)))


def plan_jobs(intermediate, initial_count, path_fix_size):
    """The jobs before any merge (path_manager.py:423-464): one per centroid looking for one song (always so without
    path_fix_size), or `initial_count` buckets of consecutive centroids, each at the buckets' mean with a scaled k."""
    m = len(intermediate)
    if not path_fix_size or initial_count >= m:
        return [{"vector": intermediate[i], "k": K_BASE, "indices": [i], "need": 1} for i in range(m)]
    step = float(m) / float(initial_count)
    k = min(K_MAX, max(K_BASE, int(K_BASE * (m / float(initial_count)))))
    jobs = []
    for j in range(initial_count):
        lo = int(round(j * step))
        hi = max(lo, int(round((j + 1) * step)) - 1)
        lo, hi = max(0, min(lo, m - 1)), max(0, min(hi, m - 1))
        idx = list(range(lo, hi + 1))
        jobs.append({"vector": np.mean([intermediate[i] for i in idx], axis=0), "k": k, "indices": idx,
                     "need": len(idx)})
    return jobs


def merge_jobs(jobs, i, intermediate, metric):
    """path_manager.py:501-527: job i failed; it absorbs job i + 1 and aims at the midpoint of its first and the
    other's last original centroid, with their k summed (capped) and all their songs still to find."""
    a, b = jobs[i], jobs.pop(i + 1)
    a["vector"] = interpolate_centroids(intermediate[a["indices"][0]], intermediate[b["indices"][-1]], 3, metric)[1]
    a["k"] = min(a["k"] + b["k"], K_MAX)
    a["need"] = a["need"] + b["need"]
    a["indices"] = a["indices"] + b["indices"]


def config(vm, pm, stop_on_failure):
    """am_song_path_cfg from the two modules' configuration as they hold it now."""
    pcap = pm.MAX_SONGS_PER_ARTIST
    p_ang = pm.PATH_DISTANCE_METRIC == "angular"
    return _lib.SongPathCfg(
        **chain_config(vm, bool(vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT)), path_metric=0 if p_ang else 1,
        path_lookback=int(pm.DUPLICATE_DISTANCE_CHECK_LOOKBACK),
        path_cap=int(pcap) if pcap is not None and pcap > 0 else 0, stop_on_failure=int(bool(stop_on_failure)),
        path_threshold=float(pm.DUPLICATE_DISTANCE_THRESHOLD_COSINE if p_ang else pm.DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN))


class _Request:
    """One request's candidates, their keys and the walk's carried state."""

    def __init__(self, vm, start_details, end_details, start_id, end_id):
        self.vm = vm
        self.details = {}
        self.sig, self.author, self.raw = Keys(), Keys(), Keys()
        self.used_ids = [vm.reverse_id_map[start_id], vm.reverse_id_map[end_id]]
        for d in (start_details, end_details):
            self.sig(signature(d))
        self.used_sig = np.ones(len(self.sig), dtype=np.uint8)
        self.author_count = np.zeros(0, dtype=np.int32)
        for d in (start_details, end_details):
            a = normalize(d.get("author"))
            if a:
                self._count(a)
        self.path_ids = [vm.reverse_id_map[start_id]]
        self.end_row = vm.reverse_id_map[end_id]

    def _count(self, author):
        k = self.author(author)
        if k >= len(self.author_count):
            self.author_count = np.concatenate([self.author_count, np.zeros(k + 1 - len(self.author_count), np.int32)])
        self.author_count[k] += 1

    def candidates(self, jobs):
        """Queries the jobs' centroids in one batch and attaches each job's k-NN prefix (item ids) to it; returns the
        item ids whose details are not known yet."""
        vm = self.vm
        ed = bool(vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT)
        size = len(vm.voyager_index)
        sizes = [query_size(j["k"], ed, size) for j in jobs]
        k = max(sizes, default=0)
        ids = np.zeros((len(jobs), 0), dtype=np.int64)
        if k > 0:
            q = np.stack([np.asarray(j["vector"], dtype=np.float32) for j in jobs])
            ids = np.asarray(vm.voyager_index.query(q, k=k)[0], dtype=np.int64).reshape(len(jobs), k)
        new = []
        for j, s, row in zip(jobs, sizes, ids):
            items = [vm.id_map.get(int(v)) for v in row[:s]]
            j["items"] = [i for i in items if i is not None]
            new += [i for i in j["items"] if i not in self.details]
        return list(dict.fromkeys(new))

    def add_details(self, rows):
        for d in rows:
            self.details[d["item_id"]] = d

    def walk(self, jobs, cfg):
        """One am_knn_song_path call over `jobs`; returns (songs found per job, item ids taken, failed job or None,
        distances along the path to the end song)."""
        vm = self.vm
        items = [it for j in jobs for it in j["items"]]
        off = list(accumulate((len(j["items"]) for j in jobs), initial=0))
        sig, raw = candidate_keys(items, self.details, self.sig, self.raw)
        author = [self.author(normalize(self.details[i].get("author")) if i in self.details else "") for i in items]
        self.used_sig = np.concatenate([self.used_sig, np.zeros(len(self.sig) - len(self.used_sig), np.uint8)])
        self.author_count = np.concatenate([self.author_count,
                                            np.zeros(len(self.author) - len(self.author_count), np.int32)])
        found, pos, failed, self.used_ids, self.path_ids, dist = vm.voyager_index.song_path(
            cfg, off, [j["k"] for j in jobs], [j["need"] for j in jobs], [vm.reverse_id_map.get(i, -1) for i in items],
            sig, author, raw, self.used_ids, self.used_sig, self.author_count, self.path_ids, self.end_row)
        return found, [items[p] for p in pos], failed, dist


def make_song_path(vm, pm):
    """find_path_between_songs(start_item_id, end_item_id, Lreq, path_fix_size) on the device: same (path details,
    total distance) as path_manager.py:320-557.  Lreq < 2, missing ends and the initial-count heuristic's two
    find_nearest_neighbors_by_id calls stay on the host exactly as the reference has them."""

    def find_path_between_songs(start_item_id, end_item_id, Lreq=None, path_fix_size=None):
        import app_helper

        Lreq = pm.PATH_DEFAULT_LENGTH if Lreq is None else Lreq
        path_fix_size = pm.PATH_FIX_SIZE if path_fix_size is None else path_fix_size
        if Lreq < 2:   # path_manager.py:332-345
            if start_item_id == end_item_id:
                return pm._create_path_from_ids([start_item_id]), 0.0
            details = pm._create_path_from_ids([start_item_id, end_item_id])
            v1, v2 = pm.get_vector_by_id(start_item_id), pm.get_vector_by_id(end_item_id)
            return details, (pm.get_distance(v1, v2) if v1 is not None and v2 is not None else 0.0)

        start_vec, end_vec = pm.get_vector_by_id(start_item_id), pm.get_vector_by_id(end_item_id)
        start_list = app_helper.get_score_data_by_ids([start_item_id])
        end_list = app_helper.get_score_data_by_ids([end_item_id])
        if start_vec is None or end_vec is None or not start_list or not end_list:
            logger.error("Could not retrieve vectors or details for start or end song.")
            return None, 0.0
        req = _Request(vm, start_list[0], end_list[0], start_item_id, end_item_id)
        found_items = []
        metric = pm.PATH_DISTANCE_METRIC
        num_intermediate = Lreq - 2
        jobs = []
        if num_intermediate > 0:
            intermediate = interpolate_centroids(start_vec, end_vec, Lreq, metric)[1:-1]
            try:
                sample_n = max(10, int(pm.PATH_CANDIDATES_PER_STEP))
            except Exception:
                sample_n = 50
            try:
                start_nb = [n["item_id"] for n in (pm.find_nearest_neighbors_by_id(start_item_id, n=sample_n) or [])]
                end_nb = [n["item_id"] for n in (pm.find_nearest_neighbors_by_id(end_item_id, n=sample_n) or [])]
            except Exception as e:
                logger.debug(f"Heuristic neighbor sampling failed: {e}")
                start_nb, end_nb = [], []
            jobs = plan_jobs(intermediate, initial_job_count(num_intermediate, start_nb, end_nb), path_fix_size)
        cfg = config(vm, pm, path_fix_size)
        i = 0
        pending = jobs
        while True:
            new = req.candidates(pending) if pending else []
            if new:
                req.add_details(app_helper.get_score_data_by_ids(new))
            _, taken, failed, dist = req.walk(jobs[i:], cfg)
            found_items += taken
            if failed is None or not path_fix_size:
                break
            i += failed
            if i + 1 >= len(jobs):
                logger.error(f"CRITICAL: Last centroid job failed (k={jobs[i]['k']}) and cannot merge. Path will be short.")
                break
            merge_jobs(jobs, i, intermediate, metric)
            pending = [jobs[i]]

        path_ids = [start_item_id] + found_items + [end_item_id]
        final = pm._create_path_from_ids(path_ids)
        final_ids = [d["item_id"] for d in final]
        if final_ids == path_ids:
            total = float(sum(dist))
        elif final_ids == path_ids[:-1]:   # start == end: the end song is the start song again
            total = float(sum(dist[:-1]))
        else:   # songs without details dropped: distances along what is left, as the reference measures them
            vecs = [pm.get_vector_by_id(s) for s in final_ids]
            total = 0.0
            for v1, v2 in zip(vecs, vecs[1:]):
                if v1 is not None and v2 is not None:
                    total += pm.get_distance(v1, v2)
        if len(final) != Lreq:
            logger.warning(f"Final path length is {len(final)}, but {Lreq} was requested.")
        return final, total

    return find_path_between_songs
