"""Drop-in for the ``voyager`` module surface the reference uses (voyager==2.1.0, Spotify HNSW):

    voyager.Index(space, num_dimensions, M=, ef_construction=)   voyager_manager.py:341-346,
    index.add_items(vectors, ids=)                                clap_text_search.py:242,263
    index.query(vector, k) -> (ids, distances)                    voyager_manager.py:1447,1580,1681
    index.get_vector(id), len(index), index.num_elements, index.ef
    index.save(path | file), Index.load(file)                     voyager_manager.py:183,375-384
    voyager.Space.{Cosine, Euclidean, InnerProduct}, voyager.RecallError

Instead of an HNSW graph the index is the flat [N, d] matrix in HBM and ``query`` is the exact
brute-force top-k of libaudiomuse_b200 (am_knn_*): same return convention (ascending distance,
distance = 1 - cos for Cosine), exact instead of approximate, and ``query`` also accepts a
[nq, d] batch (voyager does too).  M / ef_construction / ef are accepted and ignored.

Monkey-patch point in the reference: ``sys.modules['voyager'] = audiomuse_ai_b200.voyager_compat``
before importing tasks.voyager_manager / tasks.clap_text_search (INTEGRATION.md).
"""
from __future__ import annotations

import ctypes as C
import enum
import io
import struct
import threading
from typing import Optional

import numpy as np

from . import _lib


class Space(enum.IntEnum):
    Euclidean = 0
    InnerProduct = 1
    Cosine = 2


class StorageDataType(enum.IntEnum):
    Float8 = 16
    Float32 = 32
    E4M3 = 48


class RecallError(RuntimeError):
    """Raised when fewer than k neighbours can be returned (voyager.RecallError)."""


_METRIC = {Space.Cosine: 0, Space.Euclidean: 1, Space.InnerProduct: 2}
_MAGIC = b"AMIX"


class Index:
    def __init__(self, space: Space = Space.Cosine, num_dimensions: int = 0, M: int = 12,
                 ef_construction: int = 200, random_seed: int = 1, max_elements: int = 1,
                 storage_data_type: StorageDataType = StorageDataType.Float32):
        if num_dimensions <= 0:
            raise ValueError("num_dimensions must be positive")
        self.space = Space(space)
        self.num_dimensions = int(num_dimensions)
        self.M = M
        self.ef_construction = ef_construction
        self.ef = 10
        self._rows = np.zeros((0, self.num_dimensions), dtype=np.float32)
        self._ids = np.zeros((0,), dtype=np.int64)
        self._identity_ids = True
        self._id_to_row = {}
        self._handle: Optional[C.c_void_p] = None
        self._dirty = False
        self._mu = threading.RLock()

    # ------------------------------------------------------------------ building
    def add_items(self, vectors, ids=None, num_threads: int = -1):
        """Appends rows; an id that is already present has its vector REPLACED in place (voyager / hnswlib update
        the stored vector of an existing label; appending a second row would return the id twice from query)."""
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        if v.ndim == 1:
            v = v[np.newaxis, :]
        if v.ndim != 2 or v.shape[1] != self.num_dimensions:
            raise ValueError(f"expected vectors of dimension {self.num_dimensions}, got {v.shape}")
        with self._mu:
            self._materialise_rows()
            start = len(self._ids)
            if ids is None:
                nxt = start if self._identity_ids else (int(self._ids.max()) + 1 if start else 0)
                new_ids = np.arange(nxt, nxt + len(v), dtype=np.int64)
            else:
                new_ids = np.asarray(list(ids), dtype=np.int64)
            if len(new_ids) != len(v):
                raise ValueError("ids and vectors differ in length")
            fresh = np.ones(len(v), dtype=bool)
            if start and ids is not None:
                for a, row in enumerate(self._rows_of(new_ids, strict=False)):
                    if row >= 0:
                        self._rows[row] = v[a]
                        fresh[a] = False
            if len(new_ids) > 1 and ids is not None:  # duplicates inside this call: the last one wins
                last = {}
                for a, i in enumerate(new_ids):
                    if fresh[a]:
                        if int(i) in last:
                            fresh[last[int(i)]] = False
                        last[int(i)] = a
            if fresh.any():
                base = len(self._ids)
                self._rows = np.concatenate([self._rows, v[fresh]], axis=0)
                self._ids = np.concatenate([self._ids, new_ids[fresh]])
                self._identity_ids = bool(self._identity_ids and np.array_equal(new_ids[fresh], np.arange(base, base + int(fresh.sum()))))
                if not self._identity_ids:
                    self._id_to_row = {int(i): r for r, i in enumerate(self._ids)}
            self._dirty = True
        return [int(i) for i in new_ids]

    def add_item(self, vector, id=None):
        return self.add_items(np.asarray(vector, dtype=np.float32)[np.newaxis, :],
                              None if id is None else [id])[0]

    @classmethod
    def from_device(cls, rows_dev, space: Space = Space.Cosine) -> "Index":
        """Index over rows already in HBM (a torch.cuda f32[N, d] tensor, e.g. the all-gathered embedding matrix):
        am_knn_build_dev takes a device-to-device copy (cosine rows are stored unit-normalised, so the index owns its
        rows; 0.06 ms per 100 k x 512) -- no host round trip.  Ids are 0..N-1."""
        import torch

        rows_dev = rows_dev.contiguous()
        n, d = rows_dev.shape
        idx = cls(space, int(d))
        lib = _lib.load()
        h = C.c_void_p()
        _lib.check(lib.am_knn_build_dev(C.c_void_p(rows_dev.data_ptr()), int(n), int(d), _METRIC[idx.space],
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(h)))
        torch.cuda.current_stream().synchronize()
        idx._handle = h
        idx._rows = None                       # fetched from the device only if someone asks (save / add_items)
        idx._ids = np.arange(n, dtype=np.int64)
        idx._dirty = False
        return idx

    def _materialise_rows(self):
        if self._rows is None:
            n = len(self._ids)
            rows = np.empty((n, self.num_dimensions), dtype=np.float32)
            if n:
                all_rows = np.arange(n, dtype=np.int64)
                _lib.check(_lib.load().am_knn_get_vectors(self._handle, _lib.ptr(all_rows), n, _lib.ptr(rows)))
            self._rows = rows

    def _ensure_built(self):
        with self._mu:
            if self._handle is not None and not self._dirty:
                return self._handle
            lib = _lib.load()
            self._free()
            h = C.c_void_p()
            rows = np.ascontiguousarray(self._rows, dtype=np.float32)
            _lib.check(lib.am_knn_build(_lib.ptr(rows), rows.shape[0], self.num_dimensions,
                                        _METRIC[self.space], C.byref(h)))
            self._handle = h
            self._dirty = False
            return h

    def _free(self):
        if self._handle is not None:
            _lib.load().am_knn_free(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass

    # ------------------------------------------------------------------ inspection
    def __len__(self):
        return int(len(self._ids))

    @property
    def num_elements(self):
        return len(self)

    @property
    def ids(self):
        return [int(i) for i in self._ids]

    def __contains__(self, id):
        return self._rows_of([id], strict=False)[0] >= 0

    def _rows_of(self, ids, strict: bool) -> np.ndarray:
        """i64 rows of `ids` (any shape): a range test for identity ids, else one pass over the id dict.  An id that is
        not in the index raises KeyError when `strict`, and becomes -1 otherwise."""
        a = np.asarray(ids, dtype=np.int64)
        if self._identity_ids:
            rows = np.where((a >= 0) & (a < len(self._ids)), a, -1)
        else:
            get = self._id_to_row.get
            rows = np.fromiter((get(int(i), -1) for i in a.ravel()), dtype=np.int64, count=a.size).reshape(a.shape)
        if strict and (rows < 0).any():
            raise KeyError(f"id {int(a.ravel()[np.argmax(rows.ravel() < 0)])} not in index")
        return rows

    def _row_of(self, id) -> int:
        return int(self._rows_of([id], strict=True)[0])

    def _candidates(self, cand_ids, *keys):
        """(i64 rows of the candidate ids, -1 for an id not in the index, then each key array as i32), all 1-D and of one
        length."""
        rows = self._rows_of(cand_ids, strict=False)
        keys = [np.ascontiguousarray(k, dtype=np.int32) for k in keys]
        if rows.ndim != 1 or any(k.shape != rows.shape for k in keys):
            raise ValueError("candidate arrays differ in length")
        return (rows, *keys)

    def get_vector(self, id) -> np.ndarray:
        """The STORED vector: unit-normalised for Space.Cosine, like voyager.  One row gathered on the device and
        copied back (no host mirror of the library)."""
        return self.get_vectors([id])[0]

    def get_vectors(self, ids) -> np.ndarray:
        """Stored vectors of several ids: one device gather + one copy (no host mirror of the library)."""
        rows = self._rows_of(ids, strict=True)
        out = np.empty((len(rows), self.num_dimensions), dtype=np.float32)
        if len(rows):
            h = self._ensure_built()
            _lib.check(_lib.load().am_knn_get_vectors(h, _lib.ptr(rows), len(rows), _lib.ptr(out)))
        return out

    # ------------------------------------------------------------------ query
    def query(self, vectors, k: int = 1, num_threads: int = -1, query_ef: int = -1, mode: int = 0):
        q = np.ascontiguousarray(vectors, dtype=np.float32)
        single = q.ndim == 1
        if single:
            q = q[np.newaxis, :]
        if q.ndim != 2 or q.shape[1] != self.num_dimensions:
            raise ValueError(f"query must have dimension {self.num_dimensions}, got {q.shape}")
        k = int(k)
        if k > len(self):
            raise RecallError(f"Fewer than expected results were retrieved; only found {len(self)} of {k} "
                              "requested neighbors.")
        nq = q.shape[0]
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float32)
        if k > 0 and nq > 0:
            h = self._ensure_built()
            st = _lib.load().am_knn_query(h, _lib.ptr(q), nq, k, int(mode), _lib.ptr(ids), _lib.ptr(dist))
            if st == _lib.AM_ERR_RECALL:
                raise RecallError(_lib.last_error())
            _lib.check(st)
            if not self._identity_ids:
                ids = self._ids[ids]
        ids = ids.astype(np.uint64)
        return (ids[0], dist[0]) if single else (ids, dist)

    # ------------------------------------------------------------------ duplicate filter (SURVEY 8(f) row 2)
    def filter_by_distance(self, ids, threshold: float, lookback: int = 1, batch: int = 50):
        """Device version of voyager_manager._filter_by_distance (voyager_manager.py:526-617) on the vectors
        already in HBM: `ids` is one result list (closest first) or an array [n_lists, n] of them; returns a
        boolean keep mask of the same shape.  Ids that are not in the index are dropped, like the reference
        drops items whose vector is missing.  threshold / lookback: config.DUPLICATE_DISTANCE_* (config.py:550-552);
        batch: BATCH_SIZE_VECTOR_OPS (voyager_manager.py:63)."""
        arr = np.asarray(ids)
        single = arr.ndim == 1
        lists = arr[np.newaxis, :] if single else arr
        rows = self._rows_of(lists, strict=False)
        keep = np.zeros(lists.shape, dtype=np.uint8)
        if lists.size:
            h = self._ensure_built()
            _lib.check(_lib.load().am_knn_filter_by_distance(h, _lib.ptr(rows), int(lists.shape[0]), int(lists.shape[1]),
                                                             float(threshold), int(lookback), int(batch), _lib.ptr(keep)))
        keep = keep.astype(bool)
        return keep[0] if single else keep

    # ------------------------------------------------------------------ radius walk (voyager_manager.py:941-1367)
    def radius_walk(self, anchor, ids, artists, n: int, eliminate_duplicates: bool, max_songs_per_artist,
                    metric: str):
        """The reference's _execute_radius_walk over the stored vectors of `ids` (the candidates in the order the
        candidate filters leave them; ids not in the index are dropped, as a missing vector is), in one device call.
        artists: one int per candidate, a dense id per distinct truthy author and -1 for a falsy one.
        max_songs_per_artist: config.MAX_SONGS_PER_ARTIST (None or <= 0 disables the artist rules); metric:
        config.VOYAGER_METRIC ('angular' -> 1 - cos, anything else -> euclidean, as get_direct_distance reads it).
        Returns (positions in `ids` in walk order, their float64 anchor distances)."""
        a = np.ascontiguousarray(anchor, dtype=np.float32).reshape(-1)
        if a.shape[0] != self.num_dimensions:
            raise ValueError(f"anchor must have dimension {self.num_dimensions}, got {a.shape}")
        rows = self._rows_of(ids, strict=False)
        art = np.ascontiguousarray(artists, dtype=np.int32)
        if art.shape != rows.shape:
            raise ValueError("ids and artists differ in length")
        n = max(0, int(n))
        cap = 0 if max_songs_per_artist is None else int(max_songs_per_artist)
        pos = np.empty(max(n, 1), dtype=np.int32)
        dist = np.empty(max(n, 1), dtype=np.float64)
        count = C.c_int32(0)
        if len(rows) and n:
            h = self._ensure_built()
            _lib.check(_lib.load().am_knn_radius_walk(h, _lib.ptr(a), _lib.ptr(rows), _lib.ptr(art), len(rows), n,
                                                      int(bool(eliminate_duplicates)), cap,
                                                      0 if metric == "angular" else 1, _lib.ptr(pos), _lib.ptr(dist),
                                                      C.byref(count)))
        return pos[:count.value].copy(), dist[:count.value].copy()

    # ------------------------------------------------------------------ song path (path_manager.py:180-317)
    def song_path(self, cfg, job_off, job_n, job_need, cand_ids, cand_sig, cand_author, cand_author_raw, used_ids,
                  used_sig, author_count, path_ids, end_id):
        """The song path's centroid jobs over their k-NN prefixes in one device call (am_knn_song_path).
        cfg: an _lib.SongPathCfg.  job_off i32[n_jobs + 1] delimits each job's candidates in cand_ids (index ids in
        k-NN order; ids not in the index have no vector); cand_sig / cand_author / cand_author_raw are the dense keys
        the header describes.  used_sig (u8) and author_count (i32) are updated in place.  Returns (found i32[n_jobs],
        accepted candidate positions in path order, the failed job or None, used ids, path ids, f64 distances between
        consecutive path songs and the end song)."""
        n_jobs = len(job_n)
        off = np.ascontiguousarray(job_off, dtype=np.int32)
        jn = np.ascontiguousarray(job_n, dtype=np.int32)
        need = np.ascontiguousarray(job_need, dtype=np.int32)
        if off.shape != (n_jobs + 1,) or need.shape != (n_jobs,):
            raise ValueError("job_off / job_need do not match job_n")
        rows, sig, author, raw = self._candidates(cand_ids, cand_sig, cand_author, cand_author_raw)
        if n_jobs and off[-1] != len(rows):
            raise ValueError("candidate arrays differ in length")
        if used_sig.dtype != np.uint8 or author_count.dtype != np.int32:
            raise ValueError("used_sig must be uint8 and author_count int32")
        total = int(need.sum())
        used = np.empty(len(used_ids) + total, dtype=np.int64)
        used[:len(used_ids)] = self._rows_of(used_ids, strict=True)
        path = np.empty(len(path_ids) + total, dtype=np.int64)
        path[:len(path_ids)] = self._rows_of(path_ids, strict=True)
        n_used, n_path, failed = C.c_int32(len(used_ids)), C.c_int32(len(path_ids)), C.c_int32(-1)
        found = np.zeros(max(n_jobs, 1), dtype=np.int32)
        pos = np.empty(max(total, 1), dtype=np.int32)
        dist = np.empty(len(path), dtype=np.float64)
        h = self._ensure_built()
        _lib.check(_lib.load().am_knn_song_path(
            h, C.byref(cfg), n_jobs, _lib.ptr(off), _lib.ptr(jn), _lib.ptr(need), _lib.ptr(rows), _lib.ptr(sig),
            _lib.ptr(author), _lib.ptr(raw), len(used_sig), len(author_count), _lib.ptr(used), C.byref(n_used),
            _lib.ptr(used_sig), _lib.ptr(author_count), _lib.ptr(path), C.byref(n_path), self._row_of(end_id),
            _lib.ptr(found), _lib.ptr(pos), C.byref(failed), _lib.ptr(dist)))
        found = found[:n_jobs].copy()
        return (found, pos[:int(found.sum())].copy(), None if failed.value < 0 else failed.value,
                self._ids[used[:n_used.value]].tolist(), self._ids[path[:n_path.value]].tolist(),
                dist[:n_path.value].copy())

    # ------------------------------------------------------------------ Song Alchemy (tasks/song_alchemy.py:420-930)
    def alchemy(self, cfg, add_centroid, sub_centroid, cand_ids, cand_sig, cand_author_raw, n_sig, excl_ids,
                rows: bool = False):
        """Song Alchemy's candidate list in one device call (am_knn_alchemy).  cfg: an _lib.AlchemyCfg.  cand_ids are
        index ids in k-NN order (ids not in the index have no vector), cand_sig / cand_author_raw the dense keys the
        header describes, n_sig the number of signature keys; excl_ids the add and subtract songs' ids in the index.
        The centroids stay float64.  Returns (positions in cand_ids of the chain's survivors, their status: 1 kept,
        2 filtered out, 0 taken out; f64 distances to the subtract and add centroids, and their f32 stored rows when
        `rows`, else None)."""
        add = np.ascontiguousarray(add_centroid, dtype=np.float64).reshape(-1)
        sub = None if sub_centroid is None else np.ascontiguousarray(sub_centroid, dtype=np.float64).reshape(-1)
        if add.shape[0] != self.num_dimensions or (sub is not None and sub.shape[0] != self.num_dimensions):
            raise ValueError(f"centroids must have dimension {self.num_dimensions}")
        cand, sig, raw = self._candidates(cand_ids, cand_sig, cand_author_raw)
        if not 1 <= cfg.n <= _lib.ALCHEMY_MAX_N or len(cand) > _lib.ALCHEMY_MAX_CANDIDATES or (
                cfg.skip_chain and len(cand) > cfg.n):
            raise ValueError(f"{len(cand)} candidates for n = {cfg.n}: n must be in [1, {_lib.ALCHEMY_MAX_N}], the "
                             f"candidates at most {_lib.ALCHEMY_MAX_CANDIDATES}, and at most n without the chain")
        excl = self._rows_of(excl_ids, strict=True)
        n_out = max(1, min(len(cand), int(cfg.n)))
        count = C.c_int32(0)
        pos = np.empty(n_out, dtype=np.int32)
        status = np.empty(n_out, dtype=np.uint8)
        dsub = np.empty(n_out, dtype=np.float64)
        dadd = np.empty(n_out, dtype=np.float64)
        out_rows = np.empty((n_out, self.num_dimensions), dtype=np.float32) if rows else None
        h = self._ensure_built()
        _lib.check(_lib.load().am_knn_alchemy(
            h, C.byref(cfg), _lib.ptr(add), None if sub is None else _lib.ptr(sub), len(cand), _lib.ptr(cand),
            _lib.ptr(sig), _lib.ptr(raw), int(n_sig), len(excl), _lib.ptr(excl), C.byref(count), _lib.ptr(pos),
            _lib.ptr(status), _lib.ptr(dsub), _lib.ptr(dadd), None if out_rows is None else _lib.ptr(out_rows)))
        k = count.value
        return (pos[:k].copy(), status[:k].copy(), dsub[:k].copy(), dadd[:k].copy(),
                None if out_rows is None else out_rows[:k].copy())

    # ------------------------------------------------------------------ similar tracks (voyager_manager.py:1493-1702)
    def similar(self, cfg, target_id, target_sig, cand_ids, cand_sig, cand_author_raw, n_sig, n: int, mood=None,
                mood_ok=None, target_mood=None):
        """A plain similar-tracks request after its k-NN query in one device call (am_knn_similar).  cfg: an
        _lib.SimilarCfg.  target_id: the by-id request's target (index id), or None for a by-vector request;
        target_sig its signature key (-1: none).  cand_ids are index ids in k-NN order (ids not in the index have no
        vector), cand_sig / cand_author_raw the dense keys the header describes, n_sig the number of signature keys.
        mood f64[n_cand, 6] / mood_ok / target_mood f64[6] run the mood stage, mood=None skips it.  Returns (positions in
        cand_ids of the survivors, in order; their f64 mood distances, or None without the mood stage)."""
        cand, sig, raw = self._candidates(cand_ids, cand_sig, cand_author_raw)
        target = -1 if target_id is None else self._row_of(target_id)
        if mood is not None:
            mood = np.ascontiguousarray(mood, dtype=np.float64).reshape(len(cand), 6)
            mood_ok = np.ascontiguousarray(mood_ok, dtype=np.uint8)
            target_mood = np.ascontiguousarray(target_mood, dtype=np.float64).reshape(6)
            if mood_ok.shape != cand.shape:
                raise ValueError("mood_ok and the candidates differ in length")
        n_out = max(1, min(len(cand), int(n)))
        count = C.c_int32(0)
        pos = np.empty(n_out, dtype=np.int32)
        md = np.empty(n_out, dtype=np.float64)
        h = self._ensure_built()
        _lib.check(_lib.load().am_knn_similar(
            h, C.byref(cfg), target, int(target_sig), len(cand), _lib.ptr(cand), _lib.ptr(sig), _lib.ptr(raw), int(n_sig),
            None if mood is None else _lib.ptr(mood), None if mood is None else _lib.ptr(mood_ok),
            None if mood is None else _lib.ptr(target_mood), int(n), C.byref(count), _lib.ptr(pos), _lib.ptr(md)))
        k = count.value
        return pos[:k].copy(), (None if mood is None else md[:k].copy())

    def farthest(self, id):
        """get_max_distance_for_id's answer for the stored vector of `id` in one pass (am_knn_farthest): (the largest
        float32 distance query(k=len) would return to another id, that id), or (0.0, None) when there is none."""
        row = self._row_of(id)
        q = self.get_vector(id)
        out_row, out_dist = C.c_int64(-1), C.c_float(0.0)
        h = self._ensure_built()
        _lib.check(_lib.load().am_knn_farthest(h, _lib.ptr(q), row, C.byref(out_row), C.byref(out_dist)))
        if out_row.value < 0:
            return 0.0, None
        return float(out_dist.value), int(self._ids[out_row.value])

    # ------------------------------------------------------------------ persistence
    def as_bytes(self) -> bytes:
        with self._mu:
            self._materialise_rows()
            head = _MAGIC + struct.pack("<IIIQ", 1, int(self.space), self.num_dimensions, len(self._ids))
            return head + self._ids.astype("<i8").tobytes() + self._rows.astype("<f4").tobytes()

    def save(self, output_path_or_file):
        data = self.as_bytes()
        if hasattr(output_path_or_file, "write"):
            output_path_or_file.write(data)
        else:
            with open(output_path_or_file, "wb") as f:
                f.write(data)

    @classmethod
    def load(cls, file_or_path, space: Optional[Space] = None, num_dimensions: Optional[int] = None,
             storage_data_type=None) -> "Index":
        if hasattr(file_or_path, "read"):
            data = file_or_path.read()
        else:
            with open(file_or_path, "rb") as f:
                data = f.read()
        if data[:4] != _MAGIC:
            raise RuntimeError("not an audiomuse-b200 flat index (a voyager HNSW blob cannot be read here: "
                               "rebuild from the embedding table, voyager_manager.build_and_store_voyager_index)")
        ver, sp, d, n = struct.unpack_from("<IIIQ", data, 4)
        if ver != 1:
            raise RuntimeError(f"unsupported flat-index version {ver}")
        off = 4 + struct.calcsize("<IIIQ")
        ids = np.frombuffer(data, dtype="<i8", count=n, offset=off)
        rows = np.frombuffer(data, dtype="<f4", count=n * d, offset=off + 8 * n).reshape(n, d)
        idx = cls(Space(sp), d)
        idx.add_items(rows, ids=ids)
        return idx


def loads(data: bytes) -> Index:
    return Index.load(io.BytesIO(data))
