"""The device Song Path's host side without a GPU: the float64 oracle (oracle/song_path.py) against the reference's
recorded paths (tests/golden/song_path_golden.npz), the job planning against the recorded query vectors, the
drop-in's keys and validation, and integration.apply(path_manager=, app_path=)."""
import math
import sys
import types

import numpy as np
import pytest

from audiomuse_ai_b200 import song_path as sp
from oracle import song_path as osp
from tests.golden import make_song_path_golden as gen

# float32 error of one direct distance of the reference (unit or raw rows, d = 64): the dot products and norms are
# sums of 64 float32 products, so |float32 - exact| <= 64 * 2^-24 relative; arccos(cos) / pi amplifies an error in
# cos by 1 / (pi sin(pi t)) at the angular threshold t.  k-NN orders are float64 on both sides.
GAMMA = 64 * 2.0 ** -24
KNN_BOUND = 1e-12


def thr_bound(cfg):
    t = cfg["THRESHOLD_COSINE"]
    return max(GAMMA * max(1.0, cfg["THRESHOLD_EUCLIDEAN"]), GAMMA / (math.pi * math.sin(math.pi * t)))


@pytest.fixture(scope="module")
def cases():
    return gen.load()


def test_golden_covers_the_issue_cases(cases):
    assert {c["Lreq"] for c in cases} == {3, 5, 25, 60}
    assert {c["path_fix_size"] for c in cases} == {True, False}
    assert {c["config"]["MAX_SONGS_PER_ARTIST"] for c in cases} == {0, 1, 3}
    assert {c["config"]["LOOKBACK"] for c in cases} == {0, 1, 3}
    assert {(c["config"]["VOYAGER_METRIC"], c["config"]["PATH_DISTANCE_METRIC"]) for c in cases} == {
        ("angular", "angular"), ("angular", "euclidean"), ("euclidean", "euclidean"), ("euclidean", "angular")}
    assert {c["config"]["ELIMINATE_DUPLICATES"] for c in cases} == {True, False}
    merged = [c for c in cases if c["path_fix_size"] and any(not f for _, _, f in c["jobs"])]
    assert len(merged) >= 8
    assert any(len(c["path"]) < c["Lreq"] and c["path_fix_size"] for c in cases)   # a failing last job
    assert any(c["library"] == "small" and max(k for _, k in c["queries"]) == 40 for c in cases)


def test_oracle_reproduces_every_golden(cases):
    for c in cases:
        rows = gen.stored_rows(c["library"], c["space"])
        o = osp.song_path(rows, c["space"], gen.score_table(c["library"]), c["config"], c["start"], c["end"],
                          c["Lreq"], c["path_fix_size"], *c["neighbours"])
        assert o["path"] == c["path"], c["name"]
        assert o["jobs"] == c["jobs"], c["name"]
        assert [k for _, k in o["queries"]] == [k for _, k in c["queries"]], c["name"]
        assert all(np.array_equal(a, b) for (a, _), (b, _) in zip(o["queries"], c["queries"])), c["name"]
        assert o["total"] == pytest.approx(c["total"], rel=5e-5), c["name"]
        assert o["thr_gap"] == c["thr_gap"] and o["knn_gap"] == c["knn_gap"]


def test_every_margin_exceeds_the_float32_bound(cases):
    for c in cases:
        assert c["thr_gap"] > thr_bound(c["config"]), c["name"]
        assert c["knn_gap"] > KNN_BOUND, c["name"]


def test_host_jobs_give_the_recorded_query_vectors_bit_for_bit(cases):
    """Replays the planning and the merges the golden's job sequence implies, without any walk."""
    for c in cases:
        if c["Lreq"] <= 2:
            continue
        rows = gen.stored_rows(c["library"], c["space"])
        metric = c["config"]["PATH_DISTANCE_METRIC"]
        s, e = int(c["start"][4:]), int(c["end"][4:])
        inter = sp.interpolate_centroids(rows[s], rows[e], c["Lreq"], metric)[1:-1]
        jobs = sp.plan_jobs(inter, sp.initial_job_count(c["Lreq"] - 2, *c["neighbours"]), c["path_fix_size"])
        ed, n = c["config"]["ELIMINATE_DUPLICATES"], len(rows)
        got, i = [], 0
        for k, need, found in c["jobs"]:
            job = jobs[i]
            assert (job["k"], job["need"]) == (k, need), c["name"]
            got.append((np.asarray(job["vector"], np.float32), sp.query_size(k, ed, n)))
            if found or not c["path_fix_size"]:
                i += 1
            elif i + 1 < len(jobs):
                sp.merge_jobs(jobs, i, inter, metric)
        assert len(got) == len(c["queries"]), c["name"]
        for (a, ka), (b, kb) in zip(got, c["queries"]):
            assert ka == kb and a.dtype == b.dtype and np.array_equal(a, b), c["name"]


def test_interpolation_falls_back_to_straight_lines():
    z = np.zeros(4)
    v = np.array([1.0, 2.0, 0.0, 0.0])
    assert np.array_equal(sp.interpolate_centroids(z, v, 5, "angular"), np.linspace(z, v, 5))
    assert np.allclose(sp.interpolate_centroids(v, 3 * v, 4, "angular"), np.linspace(v, 3 * v, 4))
    mid = sp.interpolate_centroids(np.array([1.0, 0.0]), np.array([0.0, 2.0]), 3, "angular")[1]
    assert np.allclose(mid, 1.5 * np.array([1.0, 1.0]) / np.sqrt(2))


def test_planning_rules():
    assert sp.query_size(10, True, 10_000) == 50 and sp.query_size(10, False, 10_000) == 12
    assert sp.query_size(20, True, 40) == 40
    assert sp.initial_job_count(23, ["a", "b", "c"], ["c", "d"]) == 1       # intersection 1 -> max(1, 0)
    assert sp.initial_job_count(23, list("abcdef"), list("ghij")) == 5       # no intersection: union 10
    assert sp.initial_job_count(23, [], []) == 23
    inter = np.arange(23 * 2, dtype=float).reshape(23, 2)
    jobs = sp.plan_jobs(inter, 5, True)
    assert [j["indices"][0] for j in jobs] == [0, 5, 9, 14, 18] and sum(j["need"] for j in jobs) == 23
    assert all(j["k"] == 46 for j in jobs)
    assert [j["need"] for j in sp.plan_jobs(inter, 5, False)] == [1] * 23
    sp.merge_jobs(jobs, 3, inter, "euclidean")
    assert len(jobs) == 4 and jobs[3]["indices"] == list(range(14, 23)) and jobs[3]["k"] == 92
    assert np.array_equal(jobs[3]["vector"], (inter[14] + inter[22]) / 2)


def test_keys_and_signatures():
    assert sp.signature({"author": "  The Band ", "title": "SONG "}) == sp.signature({"author": "the band",
                                                                                     "title": " song"})
    assert sp.signature({"author": None, "title": None}) == sp.signature({"author": "", "title": " "}) == ("", "")
    k = sp.Keys()
    assert [k("a"), k("b"), k("a"), k("c")] == [0, 1, 0, 2] and len(k) == 3


def _request():
    vm = types.SimpleNamespace(reverse_id_map={"s": 0, "e": 1, "x": 2}, SIMILARITY_ELIMINATE_DUPLICATES_DEFAULT=True)
    return sp._Request(vm, {"author": " A ", "title": "T"}, {"author": None, "title": "U"}, "s", "e")


def test_request_state_and_candidate_keys():
    req = _request()
    assert req.used_ids == [0, 1] and req.path_ids == [0] and req.end_row == 1
    assert req.used_sig.tolist() == [1, 1] and req.author_count.tolist() == [1]   # a falsy end author is not counted
    captured = {}

    class Index:
        def song_path(self, cfg, off, k, need, cand, sig, author, raw, *rest):
            captured.update(off=off, cand=cand, sig=sig, author=author, raw=raw, used_sig=rest[1].copy(),
                            counts=rest[2].copy())
            return np.array([1]), np.array([1]), None, [0, 1, 2], [0, 2], np.array([0.5, 0.25])

    req.vm.voyager_index = Index()
    req.add_details([{"item_id": "x", "author": "a", "title": " t "}, {"item_id": "y", "author": "B", "title": "v"}])
    jobs = [{"k": 10, "need": 1, "items": ["y", "x", "z"]}]
    found, taken, failed, dist = req.walk(jobs, None)
    assert captured["off"] == [0, 3] and captured["cand"] == [-1, 2, -1]   # y and z have no row: no vector
    assert captured["sig"] == [2, 0, -1]                                    # x repeats the start's signature
    assert captured["author"][:2] == [1, 0] and captured["raw"] == [0, 1, -1]
    assert captured["used_sig"].tolist() == [1, 1, 0] and captured["counts"].tolist() == [1, 0, 0]
    assert taken == ["x"] and failed is None and req.path_ids == [0, 2]


def test_index_song_path_validates_its_arrays():
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Euclidean, 4)
    idx.add_items(np.eye(4, dtype=np.float32))
    args = dict(cfg=None, job_off=[0, 2], job_n=[10], job_need=[1], cand_ids=[0, 1], cand_sig=[0, 1],
                cand_author=[0, 0], cand_author_raw=[-1, 0], used_ids=[2, 3], used_sig=np.zeros(2, np.uint8),
                author_count=np.zeros(1, np.int32), path_ids=[2], end_id=3)
    with pytest.raises(ValueError):
        idx.song_path(**dict(args, cand_sig=[0]))
    with pytest.raises(ValueError):
        idx.song_path(**dict(args, job_off=[0, 1]))
    with pytest.raises(ValueError):
        idx.song_path(**dict(args, job_need=[1, 1]))
    with pytest.raises(ValueError):
        idx.song_path(**dict(args, author_count=np.zeros(1, np.int64)))


def test_apply_patches_path_manager_and_app_path_only_when_asked():
    from audiomuse_ai_b200 import integration
    vm = types.ModuleType("fake_song_path_vm")
    sys.modules[vm.__name__] = vm
    try:
        def get_vector_by_id(item_id):
            return None

        get_vector_by_id.__module__ = vm.__name__
        ref = lambda *a, **k: None  # noqa: E731
        pm = types.SimpleNamespace(get_vector_by_id=get_vector_by_id, find_path_between_songs=ref)
        app = types.SimpleNamespace(find_path_between_songs=ref)
        integration.apply(voyager_manager=None)
        assert pm.find_path_between_songs is ref and app.find_path_between_songs is ref
        with pytest.raises(ValueError):
            integration.apply(app_path=app)
        assert app.find_path_between_songs is ref
        integration.apply(path_manager=pm)
        assert pm.find_path_between_songs is not ref and app.find_path_between_songs is ref
        pm.find_path_between_songs = ref
        integration.apply(path_manager=pm, app_path=app)
        assert pm.find_path_between_songs is app.find_path_between_songs is not ref
        assert pm.find_path_between_songs.__qualname__.startswith("make_song_path")
    finally:
        del sys.modules[vm.__name__]
