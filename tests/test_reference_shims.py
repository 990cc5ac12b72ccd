"""The reference's OWN index builder / loader and integration points over the shims, by replay of a golden record
(tests/golden/make_shim_trace.py ran tasks/voyager_manager.py:145-460 and tasks/clustering_gpu.py unmodified, with
`voyager` resolving to a recording wrapper of audiomuse_ai_b200.voyager_compat, against a fake DB).

Recorded: every call the reference made into `voyager` (constructor arguments, digests of the rows and ids it added,
the bytes `save` wrote, the byte streams it handed to `Index.load` and what that raised, the `ef` it set), the index
rows it wrote to the database (flat AMIX blob in one row or <name>_<i>_<n> segments of <= VOYAGER_MAX_PART_SIZE bytes,
id_map_json in part 1 only) and its final state.  The tests regenerate the same seeded rows, replay the calls on
voyager_compat and check that the shim returns / raises / writes what it did for the reference.  Queries need the GPU:
tests/test_gpu_ref_trace.py covers them the same way."""
import hashlib
import io
import json
import os
import sys
import tempfile
import types

import numpy as np
import pytest

from tests import ref_harness as rh  # noqa: F401  (FakeDB, used by the golden generator too)

OLD_HNSW_BLOB = b"VOYA" + b"\x00" * 64     # an index written by the real voyager (HNSW) before the shim


def fill(db, n, d, seed=3):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    db.embeddings = [(f"item{i}", x[i].tobytes()) for i in range(n)]
    db.embeddings.insert(5, ("broken", None))                               # NULL blob: skipped by the builder (:351)
    db.embeddings.insert(9, ("short", np.zeros(d - 1, np.float32).tobytes()))   # wrong dimension: skipped (:357)
    return x


def _sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(scope="module")
def trace(golden_dir):
    with open(os.path.join(golden_dir, "shim_trace.json")) as f:
        return json.load(f)


def _replay(calls, x=None, streams=()):
    """Runs the recorded `voyager` calls on voyager_compat.  Returns (bytes the built index saved, loaded index)."""
    from audiomuse_ai_b200 import voyager_compat as vc
    by_sha = {_sha(b): b for b in streams}
    built = loaded = saved = None
    for c in calls:
        op = c["op"]
        if op == "Index":
            built = vc.Index(getattr(vc.Space, c["space"]), num_dimensions=c["num_dimensions"], M=c["M"],
                             ef_construction=c["ef_construction"])
        elif op == "add_items":
            # the reference added exactly the regenerated rows (the NULL / short ones skipped) with ids 0..n-1
            assert list(x.shape) == c["shape"] and _sha(x.tobytes()) == c["sha256"]
            ids = np.arange(len(x), dtype=np.int64)
            assert _sha(ids.tobytes()) == c["ids_sha256"]
            built.add_items(x, ids=ids)
        elif op == "save":
            with tempfile.TemporaryDirectory() as d:
                path = os.path.join(d, "index.voy")
                built.save(path)
                with open(path, "rb") as f:
                    saved = f.read()
            assert len(saved) == c["len"] and _sha(saved) == c["sha256"]
            by_sha[_sha(saved)] = saved
        elif op == "load":
            data = by_sha[c["sha256"]]
            if c["raised"]:
                with pytest.raises(Exception) as e:
                    vc.Index.load(io.BytesIO(data))
                assert type(e.value).__name__ == c["raised"]
            else:
                loaded = vc.Index.load(io.BytesIO(data))
        elif op == "set":
            setattr(loaded, c["name"], c["value"])
            assert getattr(loaded, c["name"]) == c["value"]
        elif op == "get":
            assert getattr(loaded, c["name"]) == c["value"]
        else:
            raise AssertionError(f"unknown recorded call {op}")
    return saved, loaded


def test_build_store_load_single_row(trace):
    from audiomuse_ai_b200 import voyager_compat as vc
    g = trace["single_row"]
    cfg = g["config"]
    d, name = cfg["EMBEDDING_DIMENSION"], cfg["INDEX_NAME"]
    x = fill(rh.FakeDB(), 500, d)
    saved, _ = _replay(g["build"], x)
    assert list(g["rows"]) == [name] and g["commits"] == 1
    row = g["rows"][name]
    assert saved[:4] == b"AMIX" and row["sha256"] == _sha(saved) and row["dim"] == d   # the row holds the shim's bytes
    assert row["id_map"] == {"entries": 500, "first": "item0", "last": "item499", "has_skipped_rows": False}
    _, loaded = _replay(g["load"], streams=[saved])
    assert isinstance(loaded, vc.Index) and len(loaded) == 500 and loaded.ef == cfg["VOYAGER_QUERY_EF"]
    assert g["state"] == {"index_loaded": True, "id_map_len": 500, "ef": cfg["VOYAGER_QUERY_EF"]}
    np.testing.assert_array_equal(loaded._rows, x)             # float32 rows survive the round trip bit for bit


def test_build_store_load_segmented_rows(trace):
    """An index larger than VOYAGER_MAX_PART_SIZE is stored as <INDEX_NAME>_<part>_<total> rows (:410-436) and
    reassembled by the loader (:186-283)."""
    g = trace["segmented_rows"]
    cfg = g["config"]
    x = fill(rh.FakeDB(), 4000, cfg["EMBEDDING_DIMENSION"])
    saved, _ = _replay(g["build"], x)
    names, rows = g["part_order"], g["rows"]
    total = len(names)
    assert sorted(rows) == sorted(names) and total == -(-len(saved) // (1 << 20)) >= 3
    assert names == [f"{cfg['INDEX_NAME']}_{i}_{total}" for i in range(1, total + 1)]
    parts, off = [], 0
    for n in names:                                               # the rows are the shim's bytes, cut in order
        parts.append(saved[off:off + rows[n]["len"]])
        off += rows[n]["len"]
        assert _sha(parts[-1]) == rows[n]["sha256"] and rows[n]["len"] <= (1 << 20)
    assert off == len(saved)
    assert rows[names[0]]["id_map"]["entries"] == 4000 and all(rows[n]["id_map"] == "" for n in names[1:])
    _, loaded = _replay(g["load"], streams=[b"".join(parts)])
    assert len(loaded) == 4000 and g["state"]["index_loaded"] and g["state"]["id_map_len"] == 4000
    np.testing.assert_array_equal(loaded._rows, x)
    # a missing segment aborts the load before any bytes reach the index (:224-227): reference behaviour, recorded
    # (no call into the shim to replay)
    assert g["load_missing_part"] == [] and g["state_missing_part"]["index_loaded"] is False


def test_an_old_hnsw_blob_is_refused_and_the_loader_survives(trace):
    from audiomuse_ai_b200 import voyager_compat as vc
    g = trace["old_hnsw_blob"]
    assert [c["op"] for c in g["load"]] == ["load"] and g["load"][0]["raised"]
    _replay(g["load"], streams=[OLD_HNSW_BLOB])                # the shim raises what it raised for the reference
    assert g["state"]["index_loaded"] is False                  # which logged it and left the cache empty: rebuild path
    with pytest.raises(RuntimeError):
        vc.Index.load(io.BytesIO(OLD_HNSW_BLOB))


def test_not_loaded_errors_match_the_reference_contract(trace):
    """tests/unit/test_voyager_manager.py:420-473 of the reference: querying without a loaded index raises before any
    call reaches the index.  Reference behaviour only, pinned as recorded: the shim is not exercised here."""
    g = trace["not_loaded"]
    assert g["raised"] == {"find_nearest_neighbors_by_vector": "RuntimeError", "find_nearest_neighbors_by_id": "RuntimeError",
                           "get_max_distance_for_id": "RuntimeError"}
    assert g["calls"] == []


def test_integration_patch_applies_to_the_reference_modules(trace):
    from audiomuse_ai_b200 import clap_analyzer as b200_clap, clustering_gpu as b200_cg, integration
    from audiomuse_ai_b200 import voyager_compat as vc
    g = trace["integration"]
    integration.install_voyager_shim()
    assert sys.modules["voyager"] is vc
    # stand-ins with the attributes the reference modules have (recorded from them)
    assert sorted(g["clap_defs"]) == sorted(integration.CLAP_NAMES)   # every patched name exists upstream with that spelling
    ref_clap = types.ModuleType("tasks.clap_analyzer")
    for name in g["clap_defs"]:
        setattr(ref_clap, name, object())
    assert g["voyager_manager_has_filter_by_distance"]
    ref_vm = types.ModuleType("tasks.voyager_manager")
    ref_vm._filter_by_distance = object()
    ref_cg = types.ModuleType("tasks.clustering_gpu")
    for name in g["clustering_names"]:
        setattr(ref_cg, name, object())
    old = os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
    try:
        integration.apply(clap=ref_clap, voyager_manager=ref_vm, clustering=ref_cg)
        assert os.environ.get("B200_ALLOW_SKLEARN_FALLBACK") == "1"        # the reference's silent-fallback contract
    finally:
        os.environ.pop("B200_ALLOW_SKLEARN_FALLBACK", None)
        if old is not None:
            os.environ["B200_ALLOW_SKLEARN_FALLBACK"] = old
    assert all(getattr(ref_clap, n) is getattr(b200_clap, n) for n in integration.CLAP_NAMES)
    assert ref_cg.GPUKMeans is b200_cg.GPUKMeans and ref_cg.check_gpu_available is b200_cg.check_gpu_available
    assert ref_cg.GPUDBSCAN is b200_cg.GPUDBSCAN and ref_cg.GPUPCA is b200_cg.GPUPCA
    assert ref_vm._filter_by_distance.__name__ == "_filter_by_distance_b200"
    # the reference's get_clustering_model / get_pca_model handed out these classes after the patch
    # (clustering_gpu.py:151-278, 338-421), constructed with these arguments
    assert g["factory_results"] == {"kmeans": "GPUKMeans", "dbscan": "GPUDBSCAN", "pca": "GPUPCA"}
    made = {c["class"]: getattr(b200_cg, c["class"])(*c["args"], **c["kwargs"]) for c in g["constructed"]}
    assert made["GPUKMeans"].n_clusters == 7
    assert made["GPUDBSCAN"].eps == 0.5 and made["GPUDBSCAN"].min_samples == 4
    assert made["GPUPCA"].n_components == 12
