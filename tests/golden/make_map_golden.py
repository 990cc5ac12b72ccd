#!/usr/bin/env python
"""Golden record of the library map projection as the reference builds it.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_map_golden.py
    # writes tests/golden/map_golden.npz

Runs app_helper.build_and_store_map_projection('main_map') (app_helper.py:1314-1372), UNMODIFIED and on the CPU,
over a fake database, with flask / redis / rq / psycopg2 / app_auth as inert stand-ins and a stand-in `umap` module
whose UMAP records its constructor arguments and the matrix it is given and returns a fixed seeded array.  The real
tasks.song_alchemy._project_with_umap (:272-287) runs around it.  Recorded:
  - the track ids in database order and which of them have no embedding (NULL or empty: skipped by the reference);
  - the matrix handed to _project_with_umap and the UMAP constructor kwargs;
  - the array the stand-in returned, and what the reference made of it: the coordinates saved, the blob and id map
    written to map_projection_data and its embedding_dimension.
tests/test_umap_host.py and tests/test_gpu_umap.py replay the record.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402

N_TRACKS, DIM, SEED = 400, 200, 17
NULL_ROWS = (3, 50, 51, 299, 398)          # embedding NULL
EMPTY_ROWS = (120, 321)                    # embedding present but zero-length


def library(seed=SEED):
    """the fake library's score rows (item ids in database order) and 200-d float32 embeddings in 12 loose groups"""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((12, DIM)).astype(np.float32)
    emb = (c[rng.integers(0, 12, N_TRACKS)] + 0.5 * rng.standard_normal((N_TRACKS, DIM))).astype(np.float32)
    ids = [f"track-{int(v):06d}" for v in rng.permutation(10 ** 6)[:N_TRACKS]]
    return ids, emb


class _Any:
    """an attribute of a stand-in module: callable, subscriptable, usable as a base class"""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Any()

    def __getattr__(self, name):
        return _Any()

    @classmethod
    def from_url(cls, *a, **k):
        return cls()


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__getattr__ = lambda attr: _Any
    sys.modules[name] = m
    return m


class MapDB:
    """Answers get_all_tracks' join and save_map_projection's upsert."""

    def __init__(self, ids, emb):
        self.rows = []
        for i, item in enumerate(ids):
            e = None if i in NULL_ROWS else (b"" if i in EMPTY_ROWS else emb[i].tobytes())
            self.rows.append(rh.DictRow({"item_id": item, "title": f"Song {i}", "author": f"Artist {i % 40}",
                                         "tempo": 120.0, "key": "C", "scale": "major", "mood_vector": "rock:0.5",
                                         "energy": 0.1, "other_features": "", "year": 2000, "rating": None,
                                         "file_path": f"/music/{i}.flac", "embedding": e}))
        self.saved = []

    def cursor(self, cursor_factory=None, **kw):
        db = self

        class Cur:
            def execute(self, sql, params=None):
                s = " ".join(sql.split())
                if s.startswith("SELECT s.item_id") and "LEFT JOIN embedding" in s:
                    self._rows = list(db.rows)
                elif s.startswith("INSERT INTO map_projection_data"):
                    db.saved.append(params)
                else:
                    raise AssertionError(f"MapDB: unexpected SQL: {s[:120]}")

            def fetchall(self):
                return self._rows

            def close(self):
                pass

        return Cur()

    def commit(self):
        pass

    def rollback(self):
        pass


def main():
    assert rh.available(), "set AUDIOMUSE_REFERENCE to a checkout of the reference"
    if rh.REF not in sys.path:
        sys.path.insert(0, rh.REF)
    for k in [k for k in sys.modules if k == "tasks" or k.startswith("tasks.") or k in ("config", "app_helper")]:
        del sys.modules[k]
    calls = []
    fixed = np.random.default_rng(SEED + 1).uniform(-3.0, 7.0, (N_TRACKS - len(NULL_ROWS) - len(EMPTY_ROWS), 2))
    fixed = fixed.astype(np.float32)

    class UMAP:
        def __init__(self, **kwargs):
            calls.append({"kwargs": dict(kwargs)})

        def fit_transform(self, X):
            calls[-1]["X"] = np.array(X, copy=True)
            assert len(X) == len(fixed)
            return fixed.copy()

    _module("umap", UMAP=UMAP)
    _module("flask", g=types.SimpleNamespace())
    _module("redis", Redis=_Any)
    _module("rq", Queue=_Any)
    _module("rq.job", Job=_Any, JobStatus=_Any)
    _module("rq.exceptions", NoSuchJobError=Exception)
    _module("rq.command", send_stop_job_command=_Any())
    _module("app_auth")
    _module("psycopg2", OperationalError=Exception, Binary=rh.Binary, connect=_Any())
    _module("psycopg2.extras", DictCursor=object)
    sys.modules["psycopg2"].extras = sys.modules["psycopg2.extras"]
    tasks_pkg = types.ModuleType("tasks")
    tasks_pkg.__path__ = [os.path.join(rh.REF, "tasks")]
    sys.modules["tasks"] = tasks_pkg
    _module("tasks.voyager_manager")
    import config  # noqa: F401  (the reference's: pure env-var defaults)

    ids, emb = library()
    db = MapDB(ids, emb)
    ah = rh._load("app_helper", "app_helper.py")
    ah.get_db = lambda: db
    sa = rh._load("tasks.song_alchemy", "tasks/song_alchemy.py")
    assert ah.build_and_store_map_projection("main_map") is True
    assert len(calls) == 1, "the reference did not reach umap.UMAP"
    (name, blob, id_map_json, dim), = db.saved
    proj = np.frombuffer(blob.adapted, dtype=np.float32).reshape(-1, 2)
    kept = [i for i in range(N_TRACKS) if i not in NULL_ROWS and i not in EMPTY_ROWS]
    assert json.loads(id_map_json) == [ids[i] for i in kept]
    assert np.array_equal(calls[0]["X"], emb[kept])
    out = {"item_ids": np.array(ids), "null_rows": np.array(NULL_ROWS),
           "empty_rows": np.array(EMPTY_ROWS), "matrix": calls[0]["X"],
           "umap_kwarg_names": np.array(sorted(calls[0]["kwargs"])),
           "umap_kwarg_values": np.array([repr(calls[0]["kwargs"][k]) for k in sorted(calls[0]["kwargs"])]),
           "umap_output": fixed, "projection": proj, "blob": np.frombuffer(blob.adapted, dtype=np.uint8),
           "id_map_json": np.array(id_map_json), "index_name": np.array(name), "embedding_dimension": np.int64(dim),
           "cache_ids": np.array(ah.MAP_PROJECTION_CACHE["id_map"])}
    assert sa._project_with_umap.__module__ == "tasks.song_alchemy"
    print(calls[0]["kwargs"], out["matrix"].shape, out["matrix"].dtype, proj.shape, name, dim)
    path = os.path.join(HERE, "map_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
