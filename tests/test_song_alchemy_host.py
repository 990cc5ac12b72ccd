"""The device Song Alchemy's host side without a GPU: the float64 oracle (oracle/song_alchemy.py) against the
reference's recorded requests (tests/golden/song_alchemy_golden.npz), the sampling, the whole drop-in over an index
whose am_knn_alchemy is the oracle, validation, and integration.apply(alchemy=, app_alchemy=)."""
import random
import sys
import types

import numpy as np
import pytest

from audiomuse_ai_b200 import alchemy as al
from oracle import knn as oknn
from oracle import song_alchemy as osa
from tests.golden import make_song_alchemy_golden as gen
from tests.test_song_path_host import KNN_BOUND, thr_bound

# The drop-in's centroid distances are float64 like the reference's, in another summation order: they differ by a few
# ulps, and arccos amplifies that near 0.  A sampling draw or a temperature-0 order whose gap exceeds this cannot
# change; neither can a subtract decision.
DECISION_BOUND = 1e-9


@pytest.fixture(scope="module")
def cases():
    return gen.load()


def test_golden_covers_the_issue_cases(cases):
    sides = {(side, it["type"]) for c in cases for side in ("add", "sub") for it in (c[side] or [])}
    assert sides == {(s, t) for s in ("add", "sub") for t in ("song", "artist", "anchor", "mood")}
    assert {c["temperature"] for c in cases} == {0.0, 0.5, 1.0}
    assert any(k.startswith("find_nearest_neighbors_by_id") for c in cases for k in c["calls"])
    assert {(c["config"]["VOYAGER_METRIC"], c["config"]["PATH_DISTANCE_METRIC"]) for c in cases} == {
        ("angular", "angular"), ("angular", "euclidean"), ("euclidean", "euclidean"), ("euclidean", "angular")}
    assert {c["config"]["LOOKBACK"] for c in cases} == {0, 1}
    assert {c["config"]["MAX_SONGS_PER_ARTIST"] for c in cases} == {0, 1, 3}
    assert {c["config"]["ELIMINATE_DUPLICATES"] for c in cases} == {True, False}
    assert {c["n"] for c in cases} == {1, 10, 100, 200}
    assert any(c["library"] == "small" and c["queries"] and c["queries"][0][1] == 40 for c in cases)
    assert {c["result"].get("projection") for c in cases} >= {"none", "pca", "discriminant"}
    assert any(c["map"] == "partial" and c["result"].get("projection") == "discriminant" for c in cases)
    assert sum(len(c["result"]["filtered_out"]) for c in cases) > 20
    assert any(c["add_ids"] for c in cases) and any(not c["result"]["results"] for c in cases)


def test_oracle_reproduces_every_golden(cases):
    for c in cases:
        rows = gen.stored_rows(c["library"], c["space"])
        got = gen.check_with_oracle(osa, rows, gen.score_table(c["library"]), c)   # asserts the ids and distances
        assert got["candidates"] == c["candidates"] and got["distances"] == c["distances"], c["name"]
        for g in ("filter_gap", "sub_gap", "knn_gap", "sample_gap"):
            assert got[g] == c[g], (c["name"], g)


def test_every_margin_exceeds_its_bound(cases):
    for c in cases:
        assert c["filter_gap"] > thr_bound(c["config"]), c["name"]
        assert c["knn_gap"] > KNN_BOUND, c["name"]
        assert c["sub_gap"] > DECISION_BOUND and c["sample_gap"] > DECISION_BOUND, c["name"]


def test_sampling_from_the_recorded_distances_gives_the_recorded_order(cases):
    for c in cases:
        distances = dict(zip(c["candidates"], c["distances"]))
        random.seed(c["random_seed"])
        got = al.sample(c["candidates"], distances, c["temperature"], c["n"])
        assert got == [r["item_id"] for r in c["result"]["results"]], c["name"]


def test_sampling_draws_like_the_reference():
    ids = ["a", "b", "c", "d"]
    dist = {"a": 0.1, "b": 0.1, "c": 0.3, "d": float("inf")}
    assert al.sample(ids, dist, 0.0, 3) == ["a", "b", "c"]      # stable on ties
    random.seed(5)
    got = al.sample(ids, dist, 1.0, 4)
    random.seed(5)
    assert got == osa.sample(ids, dist, 1.0, 4, 5)[0] and sorted(got) == ids
    assert al.sample(ids, {"a": 0.1}, 1.0, 2) == ["a", "b"]     # a KeyError falls back to the sorted order
    assert al.sample([], dist, 1.0, 3) == []


# ------------------------------------------------------------------------------------------------ the drop-in
class OracleIndex:
    """The device index's surface for the drop-in over the golden's stored rows, with Index.alchemy answered by the
    oracle from the keys the drop-in built."""

    def __init__(self, rows, space):
        self.rows, self.space, self.calls = rows, space, []

    def __len__(self):
        return len(self.rows)

    def get_vector(self, i):
        return self.rows[int(i)].copy()

    def query(self, vec, k):
        ids, dist = oknn.topk(self.rows, np.asarray(vec, np.float32)[None, :], int(k),
                              metric=oknn.COSINE if self.space == "cosine" else oknn.EUCLIDEAN)
        return ids[0].astype(np.uint64), dist[0]

    def alchemy(self, cfg, add_c, sub_c, cand_ids, cand_sig, cand_raw, n_sig, excl_ids, rows=False):
        self.calls.append(dict(n=cfg.n, skip_chain=cfg.skip_chain, rows=rows, m=len(cand_ids)))
        items = [f"item{i}" for i in cand_ids]
        keyed = {it: (s, None if r < 0 else r) for it, s, r in zip(items, cand_sig, cand_raw) if s >= 0}
        ocfg = {"VOYAGER_METRIC": "angular" if cfg.voyager_metric == 0 else "euclidean",
                "THRESHOLD_COSINE": cfg.filter_threshold, "THRESHOLD_EUCLIDEAN": cfg.filter_threshold,
                "LOOKBACK": cfg.filter_lookback, "BATCH": cfg.filter_batch, "MAX_SONGS_PER_ARTIST": cfg.voyager_cap,
                "ELIMINATE_DUPLICATES": True}
        metric = "angular" if cfg.path_metric == 0 else "euclidean"
        o = osa.candidates(self.rows, keyed, ocfg, metric, add_c, sub_c, cfg.subtract_threshold, items,
                           {f"item{i}" for i in excl_ids}, cfg.n, bool(cfg.skip_chain))
        pos = [items.index(it) for it in o["chain"]]
        status = [1 if it in o["distances"] else 2 if it in o["filtered_out"] else 0 for it in o["chain"]]
        dsub = [o["dsub"].get(it, 0.0) for it in o["chain"]]
        dadd = [o["distances"].get(it, 0.0) for it in o["chain"]]
        got = self.rows[[int(it[4:]) for it in o["chain"]]] if rows else None
        return np.array(pos, np.int32), np.array(status, np.uint8), np.array(dsub), np.array(dadd), got


def _replay(c, name, convert=lambda v: v):
    def fn(*args, **kwargs):
        key = gen.call_key(name, args, kwargs)
        assert key in c["calls"], f"{c['name']}: {name} called with arguments the reference did not use"
        rec = c["calls"][key]
        if "raises" in rec:
            raise RuntimeError(rec["raises"])
        return convert(rec["value"])
    fn.__name__ = name
    return fn


def modules(c, index, tag="song_alchemy_test"):
    """Stand-ins for the reference's song_alchemy, voyager_manager, app_helper and app_helper_artist over `index`
    and the golden's table, map, anchors and artists; the reference helpers replay the recorded calls (the local
    projections check that their input vectors hash as recorded)."""
    lib, space = c["library"], c["space"]
    table = gen.score_table(lib)
    vm = types.ModuleType(tag + "_vm")
    vm.voyager_index = index
    vm.id_map = {i: f"item{i}" for i in range(len(index))}
    vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
    sa = types.ModuleType(tag)
    sa.config = types.SimpleNamespace()
    gen.configure(vm, sa.config, c["config"])

    def get_score_data_by_ids(ids):
        return [dict(table[i]) for i in ids if i in table]

    def arr(v):
        return None if v is None else np.array(v, dtype=float)

    sa.get_score_data_by_ids = get_score_data_by_ids
    sa.get_vector_by_id = lambda i: index.get_vector(vm.reverse_id_map[i]) if i in vm.reverse_id_map else None
    sa.load_map_projection = lambda name: gen.main_map(lib, c["map"])
    sa._compute_centroid_from_items = _replay(c, "_compute_centroid_from_items", arr)
    sa._get_artist_gmm_vectors_and_weights = _replay(c, "_get_artist_gmm_vectors_and_weights",
                                                     lambda v: ([np.array(m) for m in v[0]], v[1]))
    sa._get_mood_centroid_vector = _replay(c, "_get_mood_centroid_vector", arr)
    sa._get_mood_label = _replay(c, "_get_mood_label")
    sa.find_nearest_neighbors_by_id = _replay(c, "find_nearest_neighbors_by_id",
                                              lambda v: [{"item_id": i, "distance": 0.0} for i in v])
    sa._project_with_discriminant = _replay(c, "_project_with_discriminant", lambda v: [tuple(p) for p in v])
    sa._project_to_2d = _replay(c, "_project_to_2d", lambda v: [tuple(p) for p in v])
    ah = types.ModuleType("app_helper")
    ah.get_score_data_by_ids = get_score_data_by_ids
    ah.get_alchemy_anchor_by_id = lambda a: gen.anchor(lib, space, a)
    ah.ARTIST_PROJECTION_CACHE = gen.artist_projection_cache()
    aha = types.ModuleType("app_helper_artist")
    aha.get_artist_name_by_id = gen.artist_name
    return sa, vm, ah, aha


@pytest.fixture
def helper_modules(monkeypatch):
    def install(ah, aha):
        monkeypatch.setitem(sys.modules, "app_helper", ah)
        monkeypatch.setitem(sys.modules, "app_helper_artist", aha)
    return install


def run(c, index, helper_modules, fn=None):
    sa, vm, ah, aha = modules(c, index)
    helper_modules(ah, aha)
    fn = fn or al.make_song_alchemy(sa, vm)
    random.seed(c["random_seed"])
    np.random.seed(c["np_random_seed"])
    return gen.jsonable(fn(add_items=c["add"], subtract_items=c["sub"], add_ids=c["add_ids"], subtract_ids=c["sub_ids"],
                           n_results=c["n"], subtract_distance=c["subtract_distance"], temperature=c["temperature"]))


def test_dropin_over_the_oracle_returns_every_recorded_dict(cases, helper_modules):
    for c in cases:
        idx = OracleIndex(gen.stored_rows(c["library"], c["space"]), c["space"])
        assert run(c, idx, helper_modules) == c["result"], c["name"]
        if c["result"]["results"]:
            assert len(idx.calls) == 1, c["name"]   # one device call per request
            assert idx.calls[0]["rows"] == (c["map"] != "full"), c["name"]


def test_dropin_validation_and_empty_answers(cases, helper_modules):
    c = next(c for c in cases if c["name"] == "songs_t1")
    sa, vm, ah, aha = modules(c, OracleIndex(gen.stored_rows("main", "cosine"), "cosine"))
    helper_modules(ah, aha)
    fn = al.make_song_alchemy(sa, vm)
    with pytest.raises(ValueError):
        fn(add_items=[])
    with pytest.raises(ValueError):
        fn()
    sa._compute_centroid_from_items = lambda items: None
    assert fn(add_items=[{"type": "song", "id": "nope"}]) == {"results": [], "filtered_out": [], "centroid_2d": None}
    sa._compute_centroid_from_items = lambda items: np.ones(gen.D)
    vm.voyager_index = None
    with pytest.raises(RuntimeError):
        fn(add_items=[{"type": "mood", "id": "x"}])


def test_index_alchemy_validates_before_the_library():
    from audiomuse_ai_b200 import _lib, voyager_compat as vc
    idx = vc.Index(vc.Space.Euclidean, 4)
    idx.add_items(np.eye(4, dtype=np.float32))
    cfg = _lib.AlchemyCfg(n=3)
    args = dict(cfg=cfg, add_centroid=np.zeros(4), sub_centroid=None, cand_ids=[0, 1], cand_sig=[0, 1],
                cand_author_raw=[-1, 0], n_sig=2, excl_ids=[])
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, cand_sig=[0]))
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, add_centroid=np.zeros(3)))
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, sub_centroid=np.zeros(5)))
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, cfg=_lib.AlchemyCfg(n=_lib.ALCHEMY_MAX_N + 1)))
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, cfg=_lib.AlchemyCfg(n=0)))
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, cand_ids=list(range(3001)), cand_sig=[0] * 3001, cand_author_raw=[0] * 3001))
    with pytest.raises(ValueError):
        idx.alchemy(**dict(args, cfg=_lib.AlchemyCfg(n=1, skip_chain=1)))
    with pytest.raises(KeyError):
        idx.alchemy(**dict(args, excl_ids=[7]))


def test_config_reads_both_modules():
    vm = types.SimpleNamespace(SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT=False, MAX_SONGS_PER_ARTIST=3,
                               VOYAGER_METRIC="euclidean", DUPLICATE_DISTANCE_CHECK_LOOKBACK=2,
                               BATCH_SIZE_VECTOR_OPS=50, DUPLICATE_DISTANCE_THRESHOLD_COSINE=0.01,
                               DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN=0.15)
    sa = types.SimpleNamespace(config=types.SimpleNamespace(PATH_DISTANCE_METRIC="angular",
                                                            ALCHEMY_SUBTRACT_DISTANCE_ANGULAR=0.2,
                                                            ALCHEMY_SUBTRACT_DISTANCE_EUCLIDEAN=5.0))
    cfg = al.config(sa, vm, 30, None, False)
    assert (cfg.voyager_metric, cfg.path_metric, cfg.voyager_cap, cfg.filter_lookback, cfg.n) == (1, 0, 0, 2, 30)
    assert (cfg.filter_threshold, cfg.subtract_threshold) == (0.15, 0.2)
    vm.SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT = True
    sa.config.PATH_DISTANCE_METRIC = "euclidean"
    cfg = al.config(sa, vm, 30, 0.7, True)
    assert (cfg.voyager_cap, cfg.path_metric, cfg.subtract_threshold, cfg.skip_chain) == (3, 1, 0.7, 1)


def test_apply_patches_song_alchemy_and_app_alchemy_only_when_asked():
    from audiomuse_ai_b200 import integration, projection
    vm = types.ModuleType("fake_song_alchemy_vm")
    sys.modules[vm.__name__] = vm
    try:
        def find_nearest_neighbors_by_id(item_id, n=10):
            return []

        find_nearest_neighbors_by_id.__module__ = vm.__name__
        ref = lambda *a, **k: None  # noqa: E731
        sa = types.SimpleNamespace(find_nearest_neighbors_by_id=find_nearest_neighbors_by_id, song_alchemy=ref,
                                   _project_with_umap=ref)
        app = types.SimpleNamespace(song_alchemy=ref)
        with pytest.raises(ValueError):
            integration.apply(app_alchemy=app)
        assert app.song_alchemy is ref
        integration.apply(song_alchemy=sa)   # the UMAP projection only
        assert sa.song_alchemy is ref and sa._project_with_umap is projection.project_with_umap
        integration.apply(alchemy=sa)
        assert sa.song_alchemy is not ref and app.song_alchemy is ref
        sa.song_alchemy = ref
        integration.apply(alchemy=sa, app_alchemy=app)
        assert sa.song_alchemy is app.song_alchemy is not ref
        assert sa.song_alchemy.__qualname__.startswith("make_song_alchemy")
    finally:
        del sys.modules[vm.__name__]

