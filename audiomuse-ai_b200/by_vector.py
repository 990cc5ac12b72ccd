"""The host side of the by-vector chain (find_nearest_neighbors_by_vector, voyager_manager.py:1547-1657) that the song
path, Song Alchemy and the plain similar-tracks requests run on the device: the k-NN query size, the chain's
configuration and the dense signature and raw-author keys of its candidates."""
from __future__ import annotations


def query_size(n, eliminate_duplicates, size):
    """voyager_manager.py:1561-1573: the neighbours find_nearest_neighbors_by_vector asks the index for."""
    q = n + int(n * 4) if eliminate_duplicates else n + int(n * 0.2)
    return max(0, min(q, size))


def chain_config(vm, eliminate_duplicates):
    """The chain's fields of am_song_path_cfg / am_alchemy_cfg (am_similar_cfg names the metric and the cap without
    "voyager_") from voyager_manager (vm) as it holds it now: the VOYAGER_METRIC (0 angular, 1 euclidean), the distance
    filter's lookback, batch and the threshold of the metric, and the raw-author cap (0: none), only under
    eliminate_duplicates."""
    ang = vm.VOYAGER_METRIC == "angular"
    cap = vm.MAX_SONGS_PER_ARTIST
    return dict(
        voyager_metric=0 if ang else 1, filter_lookback=int(vm.DUPLICATE_DISTANCE_CHECK_LOOKBACK),
        filter_batch=int(vm.BATCH_SIZE_VECTOR_OPS),
        voyager_cap=int(cap) if eliminate_duplicates and cap is not None and cap > 0 else 0,
        filter_threshold=float(vm.DUPLICATE_DISTANCE_THRESHOLD_COSINE if ang else vm.DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN))


def normalize(text):
    """_normalize_string / _normalize_signature's field normalisation."""
    return (text or "").strip().lower()


def signature(details):
    return normalize(details.get("author")), normalize(details.get("title"))


class Keys:
    """Dense int keys, assigned in order of first appearance."""

    def __init__(self):
        self.ids = {}

    def __call__(self, value):
        return self.ids.setdefault(value, len(self.ids))

    def __len__(self):
        return len(self.ids)


def candidate_keys(items, details, sig, raw):
    """The signature and raw-author keys of `items` (item id -> details in `details`) from the Keys sig and raw: -1 for
    an item without details, and for a falsy author."""
    cand_sig = [sig(signature(details[i])) if i in details else -1 for i in items]
    cand_raw = [raw(details[i]["author"]) if i in details and details[i].get("author") else -1 for i in items]
    return cand_sig, cand_raw
