"""The radius walk without a GPU: the oracle (oracle/radius_walk.py) against the reference's own playlists
(tests/golden/radius_walk_golden.npz), and the host half of integration.make_radius_walk over a fake index."""
import sys
import types

import numpy as np
import pytest

from oracle import radius_walk as orw
from tests.golden import make_radius_walk_golden as gen

GAP = 1e-6


@pytest.fixture(scope="module")
def golden():
    return gen.load()


def _run(case, mode):
    rows = gen.stored_rows(case["library"], case["space"])
    w = case["walk_in"]
    return orw.radius_walk([rows[v] for v in w["vid"]], rows[int(case["target"][4:])], w["author"], case["n"],
                           case["eliminate_duplicates"], case["max_songs_per_artist"], case["metric"], mode=mode)


def test_golden_covers_the_cases(golden):
    names = {c["name"] for c in golden}
    assert {c[0] for c in gen.CASES} == names
    assert {c["n"] for c in golden} >= {1, 10, 25, 49, 50, 51, 100, 200}
    assert {c["max_songs_per_artist"] for c in golden} == {0, 1, 3}
    assert {c["metric"] for c in golden} == {"angular", "euclidean"}
    assert any(len(c["walk_out"]["vid"]) < c["n"] for c in golden)                        # pool smaller than n
    assert any(c["dropped"] is not None and c["dropped"] in c["cand_in"] for c in golden)
    authors = [a for c in golden for a in c["walk_in"]["author"]]
    assert None in authors and "" in authors
    dup = next(c for c in golden if c["name"] == "cos_n100_duplicate_rows")
    assert len(set(dup["walk_in"]["dist_anchor"])) < len(dup["walk_in"]["dist_anchor"])  # exact ties on the anchor


def test_oracle_reference_mode_reproduces_the_goldens_bit_for_bit(golden):
    for case in golden:
        r = _run(case, "reference")
        w = case["walk_in"]
        assert [w["vid"][p] for p in r["positions"]] == case["walk_out"]["vid"], case["name"]
        assert r["distances"] == case["walk_out"]["distance"], case["name"]


def test_oracle_float64_mode_gives_the_golden_order_where_the_gap_allows(golden):
    checked = 0
    for case in golden:
        if min(case["sort_gap"], case["score_gap"]) <= GAP:
            continue
        r = _run(case, "float64")
        assert [case["walk_in"]["vid"][p] for p in r["positions"]] == case["walk_out"]["vid"], case["name"]
        np.testing.assert_allclose(r["distances"], case["walk_out"]["distance"], rtol=1e-6, atol=2e-6)
        checked += 1
    assert checked >= 15


# ---------------------------------------------------------------------------------------------- drop-in host logic
class FakeIndex:
    def __init__(self):
        self.calls = []

    def radius_walk(self, anchor, ids, artists, n, eliminate_duplicates, max_songs_per_artist, metric):
        self.calls.append(dict(anchor=anchor, ids=list(ids), artists=list(artists), n=n, ed=eliminate_duplicates,
                               cap=max_songs_per_artist, metric=metric))
        k = min(n, len(ids))
        return np.arange(k)[::-1].astype(np.int32), np.linspace(0.1, 0.2, k)


def _fake_vm(**over):
    vm = types.SimpleNamespace(
        voyager_index=FakeIndex(), reverse_id_map={f"i{k}": k for k in range(10)}, MAX_SONGS_PER_ARTIST=3,
        VOYAGER_METRIC="angular", MOOD_SIMILARITY_ENABLE=False,
        _filter_by_distance=lambda res, db: res,
        _deduplicate_and_filter_neighbors=lambda res, db, det: res,
        _filter_by_mood_similarity=lambda res, tid, db: res[:-1],
        _get_cached_vector=lambda item: np.ones(4, np.float32) if item == "anchor" else None)
    vm.__dict__.update(over)
    return vm


@pytest.fixture
def app_helper(monkeypatch):
    meta = {f"i{k}": {"item_id": f"i{k}", "title": f"T{k}", "author": a}
            for k, a in enumerate(["A", "B", None, "A", "", "C", "B", "A", "D", "E"])}
    mod = types.ModuleType("app_helper")
    mod.get_score_data_by_ids = lambda ids: [meta[i] for i in ids if i in meta]
    monkeypatch.setitem(sys.modules, "app_helper", mod)
    return mod


def _results(keys):
    return [{"item_id": k, "distance": 0.1 * j} for j, k in enumerate(keys)]


def test_dropin_candidates_keep_the_filters_and_drop_unknown_ids(app_helper):
    from audiomuse_ai_b200 import integration
    seen = {}

    def filt(res, db):
        seen["filter"] = [r["item_id"] for r in res]
        return res[:1] + res[2:]      # keeps the prepended target, drops i0

    vm = _fake_vm(_filter_by_distance=filt)
    cand, _ = integration.make_radius_walk(vm)
    out = cand("anchor", None, _results(["i0", "i1", "zz", "i2", "i3"]), None, {}, True, mood_similarity=True)
    assert seen["filter"][0] == "anchor"
    # i0 was dropped by the distance filter (it followed the prepended target), i3 by the mood filter, "zz" has no row
    assert [c["item_id"] for c in out] == ["i1", "i2"]
    assert out[0] == {"item_id": "i1", "row": 1, "title": "T1", "author": "B"}
    assert all("vector" not in c and "dist_anchor" not in c for c in out)
    assert cand("anchor", None, [], None, {}, True) == []


def test_dropin_candidates_fall_through_failing_filters_as_the_reference_does(app_helper):
    from audiomuse_ai_b200 import integration

    def boom(*a):
        raise RuntimeError("db down")

    vm = _fake_vm(_filter_by_distance=boom, _deduplicate_and_filter_neighbors=boom, _filter_by_mood_similarity=boom,
                  MOOD_SIMILARITY_ENABLE=True)
    cand, _ = integration.make_radius_walk(vm)
    out = cand("anchor", None, _results(["i0", "i1", "i2"]), None, {}, True)
    assert [c["item_id"] for c in out] == ["i0", "i1", "i2"]
    app_helper.get_score_data_by_ids = boom
    out = cand("anchor", None, _results(["i0", "i1"]), None, {}, True)
    assert [(c["title"], c["author"]) for c in out] == [(None, None), (None, None)]


def test_dropin_walk_maps_authors_and_reads_config_at_call_time():
    from audiomuse_ai_b200 import integration
    vm = _fake_vm()
    _, walk = integration.make_radius_walk(vm)
    assert walk("anchor", 10, []) == []
    cd = [{"item_id": f"i{k}", "row": k, "title": None, "author": a}
          for k, a in enumerate(["A", "B", None, "A", "", "C", "B"])]
    vm.MAX_SONGS_PER_ARTIST, vm.VOYAGER_METRIC = None, "euclidean"
    out = walk("anchor", 3, cd, None, True)
    call = vm.voyager_index.calls[-1]
    assert call["artists"] == [0, 1, -1, 0, -1, 2, 1]
    assert call["ids"] == list(range(7)) and call["n"] == 3 and call["ed"] is True
    assert call["cap"] is None and call["metric"] == "euclidean"
    assert [r["item_id"] for r in out] == ["i2", "i1", "i0"]
    assert all(isinstance(r["distance"], float) for r in out)


def test_apply_patches_the_walk_pair_only_when_asked():
    from audiomuse_ai_b200 import integration
    names = set(integration.RADIUS_WALK_NAMES) | {"_filter_by_distance"}

    def module():
        m = types.SimpleNamespace(**{k: object() for k in names})
        return m, dict(vars(m))

    m, before = module()
    integration.apply(voyager_manager=m)
    changed = {k for k in names if getattr(m, k) is not before[k]}
    assert changed == {"_filter_by_distance"}
    m, before = module()
    integration.apply(radius_walk=m)
    changed = {k for k in names if getattr(m, k) is not before[k]}
    assert changed == {"_radius_walk_get_candidates", "_execute_radius_walk"}
