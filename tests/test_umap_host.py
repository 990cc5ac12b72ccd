"""Host-side contracts of the GPU UMAP projection (audiomuse_ai_b200.projection) and of the float64 oracle it is tested
against (oracle/umap.py).  No GPU compute is issued here."""
import ast
import json
import os
import sys
import types

import numpy as np
import pytest

from oracle import umap as ou

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_map_golden  # noqa: E402


def test_ab_params_of_the_defaults():
    from audiomuse_ai_b200 import projection
    for a, b in (ou.find_ab_params(), projection.find_ab_params()):
        assert a == pytest.approx(1.57694, abs=5e-5) and b == pytest.approx(0.89506, abs=5e-5)


def test_oracle_bisection_reaches_the_target_or_the_floor():
    rng = np.random.default_rng(0)
    X = np.concatenate([rng.standard_normal((400, 8)), np.zeros((20, 8)), rng.standard_normal((80, 8)) * 1e-4])
    k = 15
    ids, dist = ou.knn(X.astype(np.float32), k)
    sigma, rho, ok = ou.smooth_knn_dist(dist, k)
    assert ok.all()
    t = dist[:, 1:] - rho[:, None]
    psum = np.where(t > 0, np.exp(-np.maximum(t, 0) / sigma[:, None]), 1.0).sum(1)
    hit = np.abs(psum - np.log2(k)) < 1e-5
    mean_row, mean_all = dist.mean(1), dist.mean()
    floor = ou.MIN_K_DIST_SCALE * np.where(rho > 0, mean_row, mean_all)
    assert np.all(hit | (sigma == floor)) and (~hit).any()
    assert np.all(ids[:, 0] == np.arange(len(X))) and np.all(dist[:, 0] == 0)


def test_oracle_graph_is_a_symmetric_pruned_union():
    X = np.random.default_rng(1).standard_normal((300, 5)).astype(np.float32)
    g = ou.fuzzy_graph(X, n_epochs=200)
    W = g["W"]
    assert abs(W - W.T).max() == 0 and W.diagonal().max() == 0
    assert W.data.min() >= W.data.max() / 200 and W.data.max() <= 1.0
    np.testing.assert_allclose(g["eps"], W.data.max() / W.data)
    assert ou.effective_neighbors(10) == 9 and ou.effective_neighbors(16) == 15
    with pytest.raises(ValueError):
        ou.effective_neighbors(1)


def test_drop_in_contract_before_any_device_work(monkeypatch):
    from audiomuse_ai_b200 import _lib, projection

    def no_library():
        raise AssertionError("validation must not reach the library")

    monkeypatch.setattr(_lib, "load", no_library)
    assert projection.project_with_umap([]) == []
    v = [np.ones(4), np.zeros(4), np.arange(4.0)]
    with pytest.raises(ValueError):
        projection.project_with_umap(v, n_components=3)
    for bad in (np.nan, np.inf, -np.inf):
        w = [x.copy() for x in v]
        w[1][2] = bad
        with pytest.raises(ValueError, match="NaN or infinity"):
            projection.project_with_umap(w)
    with pytest.raises(ValueError):
        projection.umap_fit_transform(np.ones((1, 4)))
    with pytest.raises(ValueError, match="NaN or infinity"):
        projection.umap_fit_transform(np.full((5, 3), 1e39))


def test_no_device_raises(monkeypatch):
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("GPU present")
    except ImportError:
        pass
    from audiomuse_ai_b200 import _lib, projection
    with pytest.raises(_lib.B200Error):
        projection.project_with_umap([np.arange(3.0), np.ones(3), np.zeros(3)])


@pytest.fixture(scope="module")
def map_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "map_golden.npz"))


def test_map_golden_kwargs_and_row_order(map_golden):
    """app_helper.build_and_store_map_projection as recorded: UMAP(n_components=2, random_state=None, n_jobs=-1) -- the
    2-component default layout the drop-in computes -- over the rows that have an embedding, in database order"""
    g = map_golden
    kwargs = {str(n): ast.literal_eval(str(v)) for n, v in zip(g["umap_kwarg_names"], g["umap_kwarg_values"])}
    assert kwargs == {"n_components": 2, "random_state": None, "n_jobs": -1}
    ids = [str(i) for i in g["item_ids"]]
    skipped = set(g["null_rows"].tolist()) | set(g["empty_rows"].tolist())
    kept = [i for i in range(len(ids)) if i not in skipped]
    assert json.loads(str(g["id_map_json"])) == [ids[i] for i in kept] == [str(i) for i in g["cache_ids"]]
    _, emb = make_map_golden.library()
    assert g["matrix"].dtype == np.float32 and g["matrix"].shape == (len(kept), 200)
    np.testing.assert_array_equal(g["matrix"], emb[kept])
    assert str(g["index_name"]) == "main_map" and int(g["embedding_dimension"]) == 2


def test_map_golden_replays_through_the_drop_in(map_golden, monkeypatch):
    """project_with_umap on the recorded matrix, with the layout replaced by the array the reference's UMAP returned:
    the coordinates and the map_projection_data blob are the reference's, byte for byte"""
    from audiomuse_ai_b200 import projection
    g = map_golden
    seen = {}

    def recorded_layout(X, **kw):
        seen["X"] = X
        return g["umap_output"].copy()

    monkeypatch.setattr(projection, "umap_fit_transform", recorded_layout)
    out = projection.project_with_umap([v for v in g["matrix"]], n_components=2)
    np.testing.assert_array_equal(seen["X"], g["matrix"])
    proj = np.array(out, dtype=np.float32)            # what build_and_store_map_projection does with the list
    np.testing.assert_array_equal(proj, g["projection"])
    assert proj.astype(np.float32).tobytes() == g["blob"].tobytes()
    assert projection.scale_to_unit(np.ones((3, 2), np.float32)) == [(0.0, 0.0)] * 3


def test_integration_patches_song_alchemy_and_app_map():
    from audiomuse_ai_b200 import integration, projection
    sa = types.ModuleType("tasks.song_alchemy")
    am = types.ModuleType("app_map")
    sentinel = object()
    for m in (sa, am):
        m._project_with_umap = sentinel
        m._project_to_2d = sentinel
    integration.apply(song_alchemy=sa, app_map=am, allow_sklearn_fallback=False)
    assert sa._project_with_umap is projection.project_with_umap
    assert am._project_with_umap is projection.project_with_umap
    assert sa._project_to_2d is sentinel and am._project_to_2d is sentinel     # the PCA fallback stays the reference's


def test_initial_layout_random_branch_is_seeded_and_rescaled():
    import scipy.sparse as sp
    from audiomuse_ai_b200 import projection
    W = sp.csr_matrix((3, 3))
    a = projection.initial_layout(np.zeros((3, 2), np.float32), W, seed=4)
    b = projection.initial_layout(np.zeros((3, 2), np.float32), W, seed=4)
    assert a.tobytes() == b.tobytes() and a.dtype == np.float32
    np.testing.assert_allclose(a.min(0), 0.0)
    np.testing.assert_allclose(a.max(0), 10.0, rtol=1e-6)
