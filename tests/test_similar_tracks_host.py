"""The device similar-tracks requests' host side without a GPU: the float64 oracle (oracle/similar_tracks.py) against
the reference's recorded requests (tests/golden/similar_tracks_golden.npz), the drop-ins over an index whose similar and
farthest are the oracle, validation, the mood parsing, integration.apply(similar=, ...) and the configuration read at
call time."""
import sys
import types

import numpy as np
import pytest

from audiomuse_ai_b200 import by_vector, integration, similar_tracks as st, voyager_compat as vc
from oracle import knn as oknn
from oracle import similar_tracks as osim
from tests.golden import make_similar_tracks_golden as gen
from tests.test_song_path_host import KNN_BOUND, thr_bound

# The device's float64 distances differ from the oracle's in the last bits: a float32 rounding or an order decided by
# more than this cannot change.
FAR_BOUND = 1e-12


@pytest.fixture(scope="module")
def cases():
    return gen.load()


def test_golden_covers_the_issue_cases(cases):
    ids = [c for c in cases if c["kind"] == "by_id"]
    vecs = [c for c in cases if c["kind"] == "by_vector"]
    lists = ids + vecs
    assert {c["config"]["VOYAGER_METRIC"] for c in lists} == {"angular", "euclidean"}
    assert {c["config"]["LOOKBACK"] for c in ids} == {0, 1} and {c["config"]["LOOKBACK"] for c in vecs} == {0, 1}
    assert {c["config"]["MAX_SONGS_PER_ARTIST"] for c in ids} == {0, 1, 3}
    assert {c["config"]["MAX_SONGS_PER_ARTIST"] for c in vecs} == {0, 1, 3}
    assert {c["request"]["n"] for c in ids} == {1, 10, 100, 500} == {c["request"]["n"] for c in vecs}
    assert {c["request"].get("eliminate_duplicates", True) for c in lists} == {True, False}
    moody = [c for c in ids if any("mood_distance" in r for r in c["result"])]
    assert len(moody) >= 4 and any(len(c["result"]) > 50 for c in moody)
    assert any(c["request"].get("mood_similarity") and not any("mood_distance" in r for r in c["result"])
               and c["result"] for c in ids)   # a target without mood features: no stage
    assert any(not c["request"].get("mood_similarity") and c["config"]["MOOD_SIMILARITY_ENABLE"]
               and any("mood_distance" in r for r in c["result"]) for c in ids)
    assert any(c["library"] == "small" and 0 < len(c["result"]) < c["request"]["n"] for c in lists)
    maxes = {c["name"]: c["result"] for c in cases if c["kind"] == "max"}
    assert maxes["max_ties_euc"]["farthest_item_id"] == "item2"      # smaller float64 distance beats the lower row
    assert maxes["max_ties_cos"]["farthest_item_id"] == "item1"      # exact ties: the lower row
    assert maxes["max_single"] == {"max_distance": 0.0, "farthest_item_id": None} and maxes["max_unknown"] is None


def test_oracle_reproduces_every_golden(cases):
    for c in cases:
        o = gen.run_oracle(osim, c)
        assert o["result"] == c["result"], c["name"]
        for g in ("filter_gap", "knn_gap", "far_gap"):
            if g in c:
                assert o[g] == c[g], (c["name"], g)


def test_every_margin_exceeds_its_bound(cases):
    for c in cases:
        if c["kind"] == "max":
            assert c["far_gap"] > FAR_BOUND, c["name"]
        else:
            assert c["filter_gap"] > thr_bound(c["config"]), c["name"]
            assert c["knn_gap"] > KNN_BOUND, c["name"]


# ------------------------------------------------------------------------------------------------ the drop-ins
class OracleIndex:
    """The device index's surface for the drop-ins over the golden's stored rows, with Index.similar and
    Index.farthest answered by the oracle."""

    def __init__(self, rows, space):
        self.rows, self.space, self.calls = rows, space, []

    def __len__(self):
        return len(self.rows)

    def get_vector(self, i):
        return self.rows[int(i)].copy()

    def query(self, vec, k):
        if k > len(self.rows):
            raise vc.RecallError("too many")
        ids, dist = oknn.topk(self.rows, np.asarray(vec, np.float32)[None, :], int(k),
                              metric=oknn.COSINE if self.space == "cosine" else oknn.EUCLIDEAN)
        return ids[0].astype(np.uint64), dist[0]

    def similar(self, cfg, target_id, target_sig, cand_ids, cand_sig, cand_raw, n_sig, n, mood=None, mood_ok=None,
                target_mood=None):
        self.calls.append("similar")
        assert max(list(cand_sig) + [target_sig], default=-1) < n_sig
        return osim.similar_keys(self.rows, cfg, -1 if target_id is None else target_id, target_sig, cand_ids,
                                 cand_sig, cand_raw, n, mood, mood_ok, target_mood)

    def farthest(self, id):
        self.calls.append("farthest")
        if not 0 <= int(id) < len(self.rows):
            raise KeyError(f"id {id} not in index")
        r, _ =osim.max_distance(self.rows, self.space, f"item{int(id)}")
        return (0.0, None) if r["farthest_item_id"] is None else (r["max_distance"], int(r["farthest_item_id"][4:]))


def fake_modules(idx, table, cfg):
    """A voyager_manager stand-in holding the golden's configuration, and app_helper over `table`."""
    vm = types.ModuleType("similar_tracks_test_vm")
    vm.voyager = vc
    vm.voyager_index = idx
    vm.id_map = {i: f"item{i}" for i in range(len(idx))}
    vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
    gen.configure(vm, cfg)
    ah = types.ModuleType("app_helper")
    ah.reads = []

    def get_score_data_by_ids(ids):
        ah.reads.append(len(ids))
        return [dict(table[i]) for i in ids if i in table]

    ah.get_score_data_by_ids = get_score_data_by_ids
    ah.get_db = lambda: None
    return vm, ah


def run(c, idx, monkeypatch, fns=None):
    """Replays golden case c through the drop-ins (or through `fns`, name -> function built over the returned vm)."""
    vm, ah = fake_modules(idx, gen.score_table(c["library"]), c["config"])
    monkeypatch.setitem(sys.modules, "app_helper", ah)
    if fns is None:
        fns = {"by_id": st.make_find_nearest_neighbors_by_id, "by_vector": st.make_find_nearest_neighbors_by_vector,
               "max": st.make_get_max_distance_for_id}
    fn = fns[c["kind"]](vm)
    req = c["request"]
    if c["kind"] == "by_id":
        return fn(req["target"], n=req["n"], eliminate_duplicates=req.get("eliminate_duplicates"),
                  mood_similarity=req.get("mood_similarity"), radius_similarity=False), ah
    if c["kind"] == "by_vector":
        return fn(np.asarray(req["vector"], np.float32), n=req["n"],
                  eliminate_duplicates=req.get("eliminate_duplicates")), ah
    return fn(req["target"]), ah


def test_dropins_over_the_oracle_return_every_recorded_answer(cases, monkeypatch):
    for c in cases:
        idx = OracleIndex(gen.stored_rows(c["library"], c["space"]), c["space"])
        got, ah = run(c, idx, monkeypatch)
        assert got == c["result"], c["name"]
        if c["kind"] != "max" and got:
            assert idx.calls == ["similar"] and len(ah.reads) == (2 if c["kind"] == "by_id" else 1), c["name"]
        if c["kind"] == "max" and got is not None:
            assert idx.calls == ["farthest"], c["name"]


def test_mood_distances_are_the_references_bits(cases):
    for c in cases:
        for r in c["result"] if c["kind"] == "by_id" else []:
            if "mood_distance" in r:
                assert isinstance(r["mood_distance"], float) and r["mood_distance"] <= c["config"][
                    "MOOD_SIMILARITY_THRESHOLD"]


# ------------------------------------------------------------------------------------------------ parsing
@pytest.mark.parametrize("text,want", [
    ("danceable:0.5,aggressive:0.25", {"danceable": 0.5, "aggressive": 0.25}),
    (" danceable : 0.5 , happy:1e-3, no_colon", {"danceable": 0.5, "happy": 0.001}),
    ("danceable:abc,happy:0.5", {}),
    ("", {}),
    ("no pairs at all", {}),
    ("a:1:2", {}),
    (None, {}),
])
def test_parse_follows_the_reference(text, want):
    assert st.parse_mood_features(text) == want
    assert osim.parse_mood(text) == want


def test_mood_row_fills_missing_features_with_zero():
    assert st.mood_row({"happy": 0.25, "tempo": 9.0}) == [0.0, 0.0, 0.25, 0.0, 0.0, 0.0]


# ------------------------------------------------------------------------------------------------ validation
def test_index_similar_checks_its_arrays_before_the_library():
    idx = vc.Index(vc.Space.Cosine, num_dimensions=4)
    idx.add_items(np.eye(4, dtype=np.float32))
    cfg = st._lib.SimilarCfg(metric=0, filter_lookback=1, filter_batch=50, cap=0, filter_threshold=0.01,
                             mood_threshold=0.15)
    with pytest.raises(ValueError):
        idx.similar(cfg, None, -1, [0, 1], [0], [0, 0], 1, 5)
    with pytest.raises(ValueError):
        idx.similar(cfg, None, -1, [0, 1], [0, 1], [0, 0], 2, 5, mood=np.zeros((2, 6)), mood_ok=[1],
                    target_mood=np.zeros(6))
    with pytest.raises(KeyError):
        idx.similar(cfg, 17, 0, [0, 1], [0, 1], [0, 0], 2, 5)
    with pytest.raises(KeyError):
        idx.farthest(17)


def test_by_id_and_by_vector_query_sizes_follow_the_reference():
    assert st.by_id_query_size(10, True, False, None, 10**6) == 10 + 30 + 1
    assert st.by_id_query_size(10, False, False, None, 10**6) == 10 + 3 + 1
    assert st.by_id_query_size(100, False, True, None, 10**6) == 100 + 300 + 1
    assert st.by_id_query_size(500, True, False, True, 10**6) == 4501
    assert st.by_id_query_size(500, False, False, True, 10**6) == 2501
    assert st.by_id_query_size(500, True, False, True, 3000) == 3000
    assert by_vector.query_size(100, True, 10**6) == 500 and by_vector.query_size(100, False, 10**6) == 120


# ------------------------------------------------------------------------------------------------ the early returns
def test_early_returns(monkeypatch):
    rows = gen.stored_rows("small", "cosine")
    idx = OracleIndex(rows, "cosine")
    vm, ah = fake_modules(idx, gen.score_table("small"), gen.BASE)
    monkeypatch.setitem(sys.modules, "app_helper", ah)
    by_id, by_vec, far = (st.make_find_nearest_neighbors_by_id(vm), st.make_find_nearest_neighbors_by_vector(vm),
                          st.make_get_max_distance_for_id(vm))
    assert by_id("item999") == [] and far("item999") is None
    assert by_vec(rows[0], n=0) == []
    vm.reverse_id_map["ghost"] = 999
    ah.get_score_data_by_ids = lambda ids: [{"item_id": i, "title": "t", "author": "a"} for i in ids]
    assert by_id("ghost") == []                                   # get_vector fails
    assert far("ghost") is None

    def recall(*a, **k):
        raise vc.RecallError("sparse")

    idx.query = recall
    assert by_id("item1") == [] and by_vec(rows[0]) == []
    vm.voyager_index = None
    for fn, arg in ((by_id, "item1"), (by_vec, rows[0]), (far, "item1")):
        with pytest.raises(RuntimeError):
            fn(arg)


def test_radius_similarity_hands_off_to_the_walk_looked_up_at_call_time(monkeypatch):
    rows = gen.stored_rows("small", "cosine")
    vm, ah = fake_modules(OracleIndex(rows, "cosine"), gen.score_table("small"), gen.BASE)
    monkeypatch.setitem(sys.modules, "app_helper", ah)
    fn = st.make_find_nearest_neighbors_by_id(vm)
    seen = {}

    def cands(**kw):
        seen["cands"] = kw
        return ["c"]

    def walk(**kw):
        seen["walk"] = kw
        return [{"item_id": "walked", "distance": 0.5}]

    vm._radius_walk_get_candidates, vm._execute_radius_walk = cands, walk
    assert fn("item3", n=5, radius_similarity=True) == [{"item_id": "walked", "distance": 0.5}]
    assert seen["walk"]["candidate_data"] == ["c"] and seen["walk"]["n"] == 5
    assert all(r["item_id"] != "item3" for r in seen["cands"]["initial_results"])
    vm.SIMILARITY_RADIUS_DEFAULT = True
    seen.clear()
    fn("item3", n=5)
    assert "walk" in seen


def test_configuration_is_read_at_call_time(cases, monkeypatch):
    c = next(c for c in cases if c["name"] == "id_n100_mood")
    idx = OracleIndex(gen.stored_rows(c["library"], c["space"]), c["space"])
    vm, ah = fake_modules(idx, gen.score_table(c["library"]), gen.BASE)
    monkeypatch.setitem(sys.modules, "app_helper", ah)
    fn = st.make_find_nearest_neighbors_by_id(vm)
    gen.configure(vm, c["config"])
    assert fn("item12", n=100, mood_similarity=True, radius_similarity=False) == c["result"]
    other = next(c for c in cases if c["name"] == "id_wide_thr")
    gen.configure(vm, other["config"])
    assert fn("item21", n=100, mood_similarity=True, radius_similarity=False) == other["result"]


# ------------------------------------------------------------------------------------------------ integration.apply
def test_apply_replaces_the_three_names_where_they_are_bound():
    vm = types.ModuleType("vm")
    app_voyager, sonic, app_path = (types.ModuleType(n) for n in ("app_voyager", "sonic", "app_path"))
    for m in (vm, app_voyager):
        for name in integration.SIMILAR_NAMES:
            setattr(m, name, None)
    sonic.find_nearest_neighbors_by_vector = app_path.find_nearest_neighbors_by_vector = None
    app_path.find_path_between_songs = "reference"
    integration.apply(similar=vm, app_voyager=app_voyager, sonic_fingerprint=sonic, app_path=app_path)
    for name in integration.SIMILAR_NAMES:
        assert getattr(vm, name).__name__ == name and getattr(app_voyager, name) is getattr(vm, name)
    assert sonic.find_nearest_neighbors_by_vector is vm.find_nearest_neighbors_by_vector
    assert app_path.find_nearest_neighbors_by_vector is vm.find_nearest_neighbors_by_vector
    assert app_path.find_path_between_songs == "reference"


def test_apply_rules():
    m = types.ModuleType("m")
    with pytest.raises(ValueError):
        integration.apply(app_voyager=m)
    with pytest.raises(ValueError):
        integration.apply(sonic_fingerprint=m)
    with pytest.raises(ValueError):
        integration.apply(app_path=m)
    vm = types.ModuleType("vm")
    vm.find_nearest_neighbors_by_id = "reference"
    integration.apply(voyager_manager=types.SimpleNamespace(), radius_walk=None)
    assert vm.find_nearest_neighbors_by_id == "reference"   # nothing changes without similar=
