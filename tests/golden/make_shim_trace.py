#!/usr/bin/env python
"""Golden record of the reference's index builder / loader and integration points running over the shims.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_shim_trace.py
    # writes tests/golden/shim_trace.json

Runs, UNMODIFIED, tasks.voyager_manager.build_and_store_voyager_index / load_voyager_index_for_querying (:145-460) and
the not-loaded error paths over a FakeDB, with `voyager` resolving to a recording wrapper of
audiomuse_ai_b200.voyager_compat, and applies integration.apply to the reference's clustering / CLAP / voyager modules.
Stored per scenario: every call the reference made into `voyager` (constructor arguments, digests of the arrays and
byte streams it passed, the bytes `save` wrote, what `load` raised, the `ef` it set), the index rows it wrote to the
database, and its final state.  tests/test_reference_shims.py replays the calls against voyager_compat.
"""
import hashlib
import io
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402
from tests.test_reference_shims import OLD_HNSW_BLOB, fill  # noqa: E402


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


class Recorder:
    """`voyager` as the reference imports it: voyager_compat with every call appended to self.calls."""

    def __init__(self, vc):
        self.vc, self.calls = vc, []
        rec = self
        mod = types.ModuleType("voyager")
        mod.__dict__.update({k: getattr(vc, k) for k in dir(vc) if not k.startswith("__")})

        class Index:
            def __new__(cls, space, num_dimensions, M=12, ef_construction=200, **kw):
                rec.calls.append({"op": "Index", "space": space.name, "num_dimensions": int(num_dimensions), "M": int(M),
                                  "ef_construction": int(ef_construction)})
                return rec.wrap(vc.Index(space, num_dimensions=num_dimensions, M=M, ef_construction=ef_construction, **kw))

            @staticmethod
            def load(stream, *a, **kw):
                if hasattr(stream, "read"):      # BytesIO (one row) or a temporary file (reassembled segments)
                    pos = stream.tell()
                    data = stream.read()
                    stream.seek(pos)
                else:
                    with open(stream, "rb") as f:
                        data = f.read()
                c = {"op": "load", "len": len(data), "sha256": sha(data), "raised": None}
                rec.calls.append(c)
                try:
                    return rec.wrap(vc.Index.load(io.BytesIO(data), *a, **kw))
                except Exception as e:
                    c["raised"] = type(e).__name__
                    raise

        mod.Index = Index
        self.module = mod

    def wrap(self, ix):
        rec = self

        class Proxy:
            def add_items(self, vectors, ids=None, **kw):
                v = np.ascontiguousarray(vectors, dtype=np.float32)
                i = np.ascontiguousarray(ids, dtype=np.int64)
                rec.calls.append({"op": "add_items", "shape": list(v.shape), "sha256": sha(v.tobytes()),
                                  "ids_sha256": sha(i.tobytes())})
                return ix.add_items(vectors, ids=ids, **kw)

            def save(self, path):
                ix.save(path)
                data = open(path, "rb").read()
                rec.calls.append({"op": "save", "len": len(data), "sha256": sha(data)})

            def __getattr__(self, n):
                v = getattr(ix, n)
                if n == "num_elements":
                    rec.calls.append({"op": "get", "name": n, "value": int(v)})
                return v

            def __setattr__(self, n, v):
                rec.calls.append({"op": "set", "name": n, "value": v})
                setattr(ix, n, v)

            def __len__(self):
                return len(ix)

        return Proxy()


def id_map_summary(m):
    """id_map_json of a row: entries, first / last item, whether a skipped row leaked in ("" when the row has none)"""
    if not m:
        return ""
    ids = json.loads(m)
    return {"entries": len(ids), "first": ids.get("0"), "last": ids.get(str(len(ids) - 1)),
            "has_skipped_rows": any(v in ("broken", "short") for v in ids.values())}


def rows_record(db):
    return {k: {"len": len(b), "sha256": sha(b), "id_map": id_map_summary(m), "dim": d}
            for k, (b, m, d) in db.index_rows.items()}


def state(vm):
    return {"index_loaded": vm.voyager_index is not None, "id_map_len": len(vm.id_map or {}),
            "ef": getattr(vm.voyager_index, "ef", None) if vm.voyager_index is not None else None}


def scenario(fn):
    from audiomuse_ai_b200 import voyager_compat as vc
    rec = Recorder(vc)
    db = rh.FakeDB()
    ref = rh.load_reference(rec.module, db)
    out = fn(ref, db, rec)
    out["config"] = {"EMBEDDING_DIMENSION": ref.config.EMBEDDING_DIMENSION, "INDEX_NAME": ref.config.INDEX_NAME,
                     "VOYAGER_QUERY_EF": ref.config.VOYAGER_QUERY_EF}
    return out


def single_row(ref, db, rec):
    vm = ref.vm
    fill(db, 500, ref.config.EMBEDDING_DIMENSION)
    vm.build_and_store_voyager_index(db)
    build = rec.calls[:]
    rows = rows_record(db)
    del rec.calls[:]
    vm.voyager_index = None
    vm.load_voyager_index_for_querying(force_reload=True)
    return {"build": build, "rows": rows, "commits": db.commits, "load": rec.calls[:], "state": state(vm)}


def segmented_rows(ref, db, rec):
    vm = ref.vm
    fill(db, 4000, ref.config.EMBEDDING_DIMENSION)
    vm.VOYAGER_MAX_PART_SIZE = 1 << 20
    vm.build_and_store_voyager_index(db)
    build = rec.calls[:]
    rows = rows_record(db)
    order = sorted(db.index_rows, key=lambda s: int(s.split("_")[-2]))
    del rec.calls[:]
    vm.voyager_index = None
    vm.load_voyager_index_for_querying(force_reload=True)
    load, st = rec.calls[:], state(vm)
    del rec.calls[:]
    del db.index_rows[order[1]]
    vm.load_voyager_index_for_querying(force_reload=True)
    return {"build": build, "rows": rows, "part_order": order, "load": load, "state": st,
            "load_missing_part": rec.calls[:], "state_missing_part": state(vm)}


def old_hnsw_blob(ref, db, rec):
    vm = ref.vm
    db.index_rows[ref.config.INDEX_NAME] = (OLD_HNSW_BLOB, json.dumps({"0": "item0"}), ref.config.EMBEDDING_DIMENSION)
    vm.load_voyager_index_for_querying(force_reload=True)
    return {"load": rec.calls[:], "state": state(vm)}


def not_loaded(ref, db, rec):
    vm = ref.vm
    vm.voyager_index = vm.id_map = vm.reverse_id_map = None
    raised = {}
    for name, arg in (("find_nearest_neighbors_by_vector", np.zeros(ref.config.EMBEDDING_DIMENSION, np.float32)),
                      ("find_nearest_neighbors_by_id", "item0"), ("get_max_distance_for_id", "item0")):
        try:
            getattr(vm, name)(arg)
            raised[name] = None
        except Exception as e:
            raised[name] = type(e).__name__
    return {"raised": raised, "calls": rec.calls[:]}


def integration_points(ref, db, rec):
    """Which module attributes the reference's callers look up (integration.apply replaces them) and the
    constructor arguments the reference's factories pass to the clustering classes after the patch."""
    import importlib.util
    from audiomuse_ai_b200 import clustering_gpu as b200_cg, integration
    spec = importlib.util.spec_from_file_location("tasks.clustering_gpu", os.path.join(rh.REF, "tasks", "clustering_gpu.py"))
    ref_cg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_cg)
    clap_src = open(os.path.join(rh.REF, "tasks", "clap_analyzer.py")).read()
    clustering_names = [n for n in ("GPUKMeans", "GPUDBSCAN", "GPUPCA", "check_gpu_available", "get_clustering_model",
                                    "get_pca_model") if hasattr(ref_cg, n)]
    seen = []

    def recording(cls):
        class Rec(cls):
            def __init__(self, *a, **kw):
                seen.append({"class": cls.__name__, "args": list(a), "kwargs": kw})
                super().__init__(*a, **kw)
        return Rec

    integration.apply(clustering=ref_cg, allow_sklearn_fallback=False)
    for n in ("GPUKMeans", "GPUDBSCAN", "GPUPCA"):
        setattr(ref_cg, n, recording(getattr(b200_cg, n)))
    made = {"kmeans": ref_cg.get_clustering_model("kmeans", {"n_clusters": 7}, use_gpu=True),
            "dbscan": ref_cg.get_clustering_model("dbscan", {"eps": 0.5, "min_samples": 4}, use_gpu=True),
            "pca": ref_cg.get_pca_model(12, use_gpu=True)}
    return {"clap_defs": [n for n in integration.CLAP_NAMES if f"def {n}(" in clap_src],
            "voyager_manager_has_filter_by_distance": callable(getattr(ref.vm, "_filter_by_distance", None)),
            "clustering_names": clustering_names, "constructed": seen,
            "factory_results": {k: type(v).__mro__[1].__name__ for k, v in made.items()}}


def main():
    assert rh.available(), "set AUDIOMUSE_REFERENCE to a checkout of the reference"
    out = {name: scenario(fn) for name, fn in (("single_row", single_row), ("segmented_rows", segmented_rows),
                                               ("old_hnsw_blob", old_hnsw_blob), ("not_loaded", not_loaded),
                                               ("integration", integration_points))}
    path = os.path.join(HERE, "shim_trace.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True, default=lambda o: o.item() if hasattr(o, "item") else str(o))
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
