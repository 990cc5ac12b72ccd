"""am_knn_song_path on the GPU: the reference's paths (tests/golden/song_path_golden.npz) through the drop-in and
through integration.apply, the round trips of one request, and seeded 100 k-row libraries against the float64 oracle
(oracle/song_path.py)."""
import sys
import types

import numpy as np
import pytest

from oracle import song_path as osp
from tests import ref_harness as rh
from tests.golden import make_song_path_golden as gen
from tests.test_song_path_host import KNN_BOUND, thr_bound

pytestmark = pytest.mark.gpu

# The reference sums Lreq - 1 float32 distances, each within 64 * 2^-24 relative of the exact one (x 1 / sin(angle)
# for arccos, angles between path songs are > 0.1 rad here), in a float32 running sum (Lreq * 2^-24 relative): for
# Lreq <= 100 all of it stays below 5e-5 of the total.
TOTAL_RTOL = 5e-5


def _index(x, space, stored):
    """The device index of the golden's space over the raw library; it stores the same rows as the recording index."""
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Cosine if space == "cosine" else vc.Space.Euclidean, num_dimensions=x.shape[1])
    idx.add_items(x, ids=np.arange(len(x)))
    sample = np.arange(0, len(x), max(1, len(x) // 500))
    assert np.array_equal(idx.get_vectors(sample), stored[sample])
    return idx


class Calls:
    def __init__(self):
        self.query = self.walk = 0
        self.details = []


def _modules(idx, table, cfg, neighbours, calls, tag="song_path_test_vm"):
    """Stand-ins for the reference's voyager_manager, path_manager and app_helper over the device index and an
    in-memory table; the index's query and walk and get_score_data_by_ids are counted."""
    vm = types.ModuleType(tag)
    vm.voyager_index = idx
    vm.id_map = {i: f"item{i}" for i in range(len(idx))}
    vm.reverse_id_map = {v: k for k, v in vm.id_map.items()}
    pm = types.ModuleType(tag + "_pm")
    gen.configure(vm, pm, cfg)
    pm.PATH_CANDIDATES_PER_STEP, pm.PATH_DEFAULT_LENGTH, pm.PATH_FIX_SIZE = 25, 25, False
    query, walk = idx.query, idx.song_path

    def counted_query(*a, **k):
        calls.query += 1
        return query(*a, **k)

    def counted_walk(*a, **k):
        calls.walk += 1
        return walk(*a, **k)

    idx.query, idx.song_path = counted_query, counted_walk

    def get_vector_by_id(item_id):
        return idx.get_vector(int(item_id[4:]))

    get_vector_by_id.__module__ = vm.__name__
    nb = iter(neighbours)
    pm.get_vector_by_id = get_vector_by_id
    pm.find_nearest_neighbors_by_id = lambda item_id, n=10: [{"item_id": i} for i in next(nb)]

    def create_path(ids):
        ids = list(dict.fromkeys(ids))
        return [dict(table[i]) for i in ids if i in table]

    pm._create_path_from_ids = create_path

    def get_score_data_by_ids(ids):
        calls.details.append(list(ids))
        return [dict(table[i]) for i in ids if i in table]

    app_helper = types.ModuleType("app_helper")
    app_helper.get_score_data_by_ids = get_score_data_by_ids
    return vm, pm, app_helper


@pytest.fixture
def app_helper_slot(monkeypatch):
    def install(mod):
        monkeypatch.setitem(sys.modules, "app_helper", mod)
        monkeypatch.setitem(sys.modules, mod.__name__, mod)
    return install


def _golden_run(c, indexes, app_helper_slot, through_apply=False):
    from audiomuse_ai_b200 import integration, song_path
    key = (c["library"], c["space"])
    if key not in indexes:
        indexes[key] = _index(gen.library(c["library"]), c["space"], gen.stored_rows(*key))
    calls = Calls()
    vm, pm, ah = _modules(indexes[key], gen.score_table(c["library"]), c["config"], c["neighbours"], calls)
    app_helper_slot(ah)
    sys.modules[vm.__name__] = vm
    try:
        if through_apply:
            app = types.ModuleType("app_path")
            integration.apply(path_manager=pm, app_path=app)
            fn = app.find_path_between_songs
        else:
            fn = song_path.make_song_path(vm, pm)
        details, total = fn(c["start"], c["end"], c["Lreq"], path_fix_size=c["path_fix_size"])
    finally:
        del sys.modules[vm.__name__]
        idx = indexes[key]
        del idx.query, idx.song_path
    return [d["item_id"] for d in details], total, calls


def test_golden_paths_through_the_dropin(app_helper_slot):
    indexes = {}
    for c in gen.load():
        ids, total, calls = _golden_run(c, indexes, app_helper_slot)
        assert ids == c["path"], c["name"]
        assert total == pytest.approx(c["total"], rel=TOTAL_RTOL), c["name"]
        merged = any(not f for _, _, f in c["jobs"]) and c["path_fix_size"]
        if not merged:   # one query, one details read over the candidates, one walk
            assert (calls.query, calls.walk) == (1 if c["Lreq"] > 2 else 0, 1), c["name"]
            assert len(calls.details) == 2 + (c["Lreq"] > 2), c["name"]
        else:            # one more of each per merge
            fails = sum(1 for _, _, f in c["jobs"] if not f)
            assert calls.walk == 1 + fails - (len(c["path"]) < c["Lreq"]), c["name"]


def test_golden_paths_through_integration_apply(app_helper_slot):
    indexes = {}
    for c in gen.load()[::3]:
        ids, total, _ = _golden_run(c, indexes, app_helper_slot, through_apply=True)
        assert ids == c["path"], c["name"]
        assert total == pytest.approx(c["total"], rel=TOTAL_RTOL), c["name"]


def _library(seed, N, d):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((64, d)).astype(np.float32)
    x = (base[rng.integers(0, 64, N)] + 0.6 * rng.standard_normal((N, d)).astype(np.float32)).astype(np.float32)
    x[N - 50:] = x[:50]   # exact duplicates
    return x


@pytest.mark.parametrize("N,d,space", [(100_000, 512, "cosine"), (100_000, 200, "euclidean")])
def test_large_libraries_match_the_oracle(N, d, space, app_helper_slot):
    from audiomuse_ai_b200 import song_path
    from oracle import knn as oknn
    x = _library(d, N, d)
    rows = oknn.normalize_rows(x) if space == "cosine" else x
    idx = _index(x, space, rows)
    table = rh.make_score_table(N, seed=d)
    for i in range(0, N, 97):
        table[f"item{i}"]["author"] = None if i % 2 else ""
    rng = np.random.default_rng(N + d)
    checked = 0
    for Lreq, fix, cap, lookback in ((10, False, 3, 1), (25, True, 3, 1), (25, True, 1, 3), (40, False, 0, 0)):
        cfg = gen.case_config(("", "", space, "angular" if space == "cosine" else "euclidean", Lreq, fix, cap, lookback,
                               True, 0.01, 1.0, "", ""))
        s, e = (int(v) for v in rng.choice(N, 2, replace=False))
        start, end = f"item{s}", f"item{e}"
        q = np.stack([rows[s], rows[e]])
        nb = [[f"item{int(i)}" for i in r] for r in idx.query(q, 25)[0]]
        o = osp.song_path(rows, space, table, cfg, start, end, Lreq, fix, *nb)
        calls = Calls()
        vm, pm, ah = _modules(idx, table, cfg, nb, calls)
        app_helper_slot(ah)
        try:
            details, total = song_path.make_song_path(vm, pm)(start, end, Lreq, path_fix_size=fix)
        finally:
            del idx.query, idx.song_path
        assert [dd["item_id"] for dd in details] == o["path"], (Lreq, fix, cap, lookback)
        assert total == pytest.approx(o["total"], rel=1e-12)
        assert o["thr_gap"] > thr_bound(cfg) and o["knn_gap"] > KNN_BOUND
        checked += 1
    assert checked == 4


def test_two_calls_are_bit_identical(app_helper_slot):
    from audiomuse_ai_b200 import song_path
    c = next(c for c in gen.load() if c["name"] == "ang_l60_fix")
    idx = _index(gen.library(c["library"]), c["space"], gen.stored_rows(c["library"], c["space"]))
    outs = []
    for _ in range(2):
        vm, pm, ah = _modules(idx, gen.score_table(c["library"]), c["config"], c["neighbours"], Calls())
        app_helper_slot(ah)
        try:
            details, total = song_path.make_song_path(vm, pm)(c["start"], c["end"], c["Lreq"], path_fix_size=True)
        finally:
            del idx.query, idx.song_path
        outs.append(([d["item_id"] for d in details], total))
    assert outs[0][0] == outs[1][0] == c["path"]
    assert np.float64(outs[0][1]).tobytes() == np.float64(outs[1][1]).tobytes()
