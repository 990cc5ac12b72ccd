#!/usr/bin/env python
"""Golden record of the artist-similarity index as the reference builds it.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_artist_gmm_golden.py
    # writes tests/golden/artist_gmm_golden.npz

Runs tasks/artist_gmm_manager.build_and_store_artist_index (:406-721), UNMODIFIED and on the CPU with the installed
scikit-learn, over a fake database and a recording stand-in `voyager` module.  The seeded library (library() below)
has about 200 artists with Pareto-distributed track counts: 1-4-track artists, one artist with more than 2 000
tracks, duplicated tracks, one artist whose embeddings are all identical and NULL embeddings.  Recorded per artist:
  - the rows in the order the reference fetched them, as indices into library()'s embedding matrix (the matrix is
    rebuilt from its seed by the tests, and its SHA-256 is recorded to prove it);
  - the stored gmm_params: K, is_few_songs, the float32 weights / means / covariances of the fitted artists, and the
    SHA-256 of json.dumps of each artist's stored dict;
  - the artist_map_json and the vectors handed to add_items.
tests/test_artist_gmm_host.py and tests/test_gpu_artist_gmm.py replay the record.
"""
import hashlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402

N_ARTISTS, DIM, SEED = 200, 200, 23
BIG_ARTIST, CONST_ARTIST = 7, 11


def library(seed=SEED):
    """score rows (author, item_id, title), embeddings f32[N, DIM] and the item ids whose embedding is NULL"""
    rng = np.random.default_rng(seed)
    sizes = np.minimum((rng.pareto(1.2, N_ARTISTS) + 1.0) * 2.0, 300).astype(int)
    sizes[BIG_ARTIST] = 2100
    sizes[3], sizes[4], sizes[5] = 1, 2, 4
    rows, emb, null = [], [], set()
    for a, n in enumerate(sizes):
        groups = 1 + int(rng.integers(0, 5))
        c = rng.standard_normal((groups, DIM))
        X = c[rng.integers(0, groups, n)] + rng.uniform(0.3, 1.2) * rng.standard_normal((n, DIM))
        if a == CONST_ARTIST:
            X[:] = X[0]
        if n > 8 and a % 3 == 0:                     # duplicated tracks
            X[rng.integers(0, n, n // 4)] = X[rng.integers(0, n, n // 4)]
        for t in range(n):
            item = f"item-{a:03d}-{t:04d}"
            rows.append((f"Artist {a:03d}", item, f"Song {t:04d}"))
            emb.append(X[t].astype(np.float32))
            if n > 6 and rng.random() < 0.03:
                null.add(item)
    return rows, np.stack(emb), null


class ArtistDB:
    """Answers the SQL of build_and_store_artist_index."""

    def __init__(self, rows, emb, null):
        self.score = sorted(rows, key=lambda r: (r[0], r[2]))
        self.emb = {r[1]: (None if r[1] in null else emb[i].tobytes()) for i, r in enumerate(rows)}
        self.fetches, self.stored = [], []

    def cursor(self, *a, **k):
        db = self

        class Cur:
            def execute(self, sql, params=None):
                s = " ".join(sql.split())
                if s.startswith("SELECT gmm_params_json FROM artist_index_data"):
                    self._rows = []
                elif s.startswith("SELECT index_name, artist_map_json, gmm_params_json FROM artist_index_data"):
                    self._rows = []
                elif s.startswith("SELECT DISTINCT author, item_id, title FROM score"):
                    self._rows = list(db.score)
                elif s.startswith("SELECT item_id, embedding FROM embedding WHERE item_id = ANY"):
                    self._rows = [(i, db.emb[i]) for i in params[0] if db.emb.get(i) is not None]
                    db.fetches.append([i for i, _ in self._rows])
                elif s.startswith("DELETE FROM artist_index_data"):
                    self._rows = []
                elif s.startswith("INSERT INTO artist_index_data"):
                    db.stored.append(params)
                else:
                    raise AssertionError(f"ArtistDB: unexpected SQL: {s[:120]}")

            def fetchone(self):
                return self._rows[0] if self._rows else None

            def fetchall(self):
                return list(self._rows)

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
    for k in [k for k in sys.modules if k == "tasks" or k.startswith("tasks.") or k in ("config", "voyager")]:
        del sys.modules[k]
    added = []

    class Index:
        def __init__(self, space, num_dimensions, M=12, ef_construction=200):
            self.n = 0

        def add_items(self, vectors, ids=None):
            added.append((np.array(vectors, copy=True), np.array(ids, copy=True)))
            self.n += len(vectors)

        @property
        def num_elements(self):
            return self.n

        def save(self, path):
            with open(path, "wb") as f:
                f.write(b"recorded")

    vm = types.ModuleType("voyager")
    vm.Index = Index
    vm.Space = types.SimpleNamespace(Euclidean=0, Cosine=1)
    sys.modules["voyager"] = vm
    tasks_pkg = types.ModuleType("tasks")
    tasks_pkg.__path__ = [os.path.join(rh.REF, "tasks")]
    sys.modules["tasks"] = tasks_pkg
    import config  # noqa: F401  (the reference's: pure env-var defaults)

    rows, emb, null = library()
    index_of = {r[1]: i for i, r in enumerate(rows)}
    db = ArtistDB(rows, emb, null)
    agm = rh._load("tasks.artist_gmm_manager", "tasks/artist_gmm_manager.py")
    agm.build_and_store_artist_index(db)
    (name, blob, artist_map_json, gmm_params_json), = db.stored
    params = json.loads(gmm_params_json)
    artists = sorted({r[0] for r in rows})
    assert len(db.fetches) == len(artists)
    row_index, offsets = [], [0]
    K, few, w, m, c, sha, thash = [], [], [], [], [], [], []
    for a, fetched in zip(artists, db.fetches):
        row_index += [index_of[i] for i in fetched]
        offsets.append(len(row_index))
        p = params.get(a)
        K.append(-1 if p is None else p["n_components"])
        few.append(bool(p and p["is_few_songs"]))
        sha.append(hashlib.sha256(json.dumps(p).encode()).hexdigest() if p else "")
        thash.append(p["tracks_hash"] if p else "")
        if p and not p["is_few_songs"]:
            w.append(np.array(p["weights"], np.float32))
            m.append(np.array(p["means"], np.float32))
            c.append(np.array(p["covariances"], np.float32))
    vectors, ids = added[0]
    out = {"artists": np.array(artists), "row_index": np.array(row_index, np.int32),
           "row_offsets": np.array(offsets, np.int64), "n_components": np.array(K, np.int32),
           "is_few_songs": np.array(few), "weights": np.concatenate(w), "means": np.concatenate(m),
           "covariances": np.concatenate(c), "params_sha256": np.array(sha), "tracks_hash": np.array(thash),
           "artist_map_json": np.array(artist_map_json), "index_name": np.array(name),
           "add_items_vectors": vectors.astype(np.float32), "add_items_ids": ids.astype(np.int64),
           "library_sha256": np.array(hashlib.sha256(emb.tobytes()).hexdigest())}
    fitted = int((~out["is_few_songs"] & (out["n_components"] > 0)).sum())
    print(len(artists), "artists,", len(row_index), "rows fetched,", fitted, "fitted", len(null), "NULL")
    path = os.path.join(HERE, "artist_gmm_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
