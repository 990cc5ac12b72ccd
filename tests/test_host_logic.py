"""Host-side contracts that need no GPU."""
import os

import numpy as np
import pytest


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not _no_gpu(), reason="exercises the no-device failure path")
def test_gpukmeans_fallback_contract_both_settings(monkeypatch):
    """tasks/clustering_gpu.py:130-148: a failing GPU k-means falls back to scikit-learn silently.  Here that is opt-in
    (B200_ALLOW_SKLEARN_FALLBACK=1, set by integration.apply for deployments); the default is to fail loudly so that a
    missing CUDA library can never pass for the GPU path in this repository's own tests."""
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    x = np.random.default_rng(0).standard_normal((300, 8)).astype(np.float32)
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    m = cg.GPUKMeans(n_clusters=3, n_init=1, random_state=0)
    with pytest.raises(_lib.B200Error):
        m.fit_predict(x)
    assert m.using_gpu is False
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    m = cg.GPUKMeans(n_clusters=3, n_init=1, random_state=0)
    labels = m.fit_predict(x)
    assert labels.shape == (300,) and m.using_gpu is False and m.cluster_centers_.shape == (3, 8)
    assert (m.labels_ == labels).all()
    assert cg.check_gpu_available() is False


@pytest.mark.skipif(not _no_gpu(), reason="exercises the no-device failure path")
def test_gpudbscan_and_gpupca_fallback_contract(monkeypatch):
    """Same contract for the two other classes of tasks/clustering_gpu.py:151-278: loud by default, scikit-learn (the
    reference's own CPU branch) when the deployment switch is set -- and then with scikit-learn's attributes."""
    from sklearn.cluster import DBSCAN
    from sklearn.decomposition import PCA
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.standard_normal((150, 6)) * 0.2 + 3, rng.standard_normal((150, 6)) * 0.2 - 3]).astype(np.float32)
    monkeypatch.delenv("B200_ALLOW_SKLEARN_FALLBACK", raising=False)
    with pytest.raises(_lib.B200Error):
        cg.GPUDBSCAN(0.8, 4).fit_predict(x)
    with pytest.raises(_lib.B200Error):
        cg.GPUPCA(3).fit_transform(x)
    monkeypatch.setenv("B200_ALLOW_SKLEARN_FALLBACK", "1")
    d = cg.get_clustering_model("dbscan", {"eps": 0.8, "min_samples": 4}, use_gpu=True)
    assert np.array_equal(d.fit_predict(x), DBSCAN(eps=0.8, min_samples=4).fit_predict(x)) and d.using_gpu is False
    p = cg.get_pca_model(3, use_gpu=True)
    y = p.fit_transform(x)
    ref = PCA(n_components=3).fit(x)
    assert p.using_gpu is False and y.shape == (300, 3) and p.n_components_ == 3
    np.testing.assert_allclose(p.explained_variance_ratio_, ref.explained_variance_ratio_, rtol=1e-6)
    np.testing.assert_allclose(p.inverse_transform(y), x, atol=1.5)   # 3 of 6 components: a projection, not the identity
    assert isinstance(cg.get_clustering_model("dbscan", {"eps": 0.8, "min_samples": 4}, use_gpu=False), DBSCAN)


def test_voyager_compat_host_side_contract(tmp_path):
    """Everything of the Index duck type that lives on the host: ids, in-place update of an existing id (voyager
    replaces the stored vector), O(1) id lookup with arbitrary ids, save / load round trip, RecallError before any
    device work."""
    from audiomuse_ai_b200 import voyager_compat as vc
    rng = np.random.default_rng(1)
    x = rng.standard_normal((50, 16)).astype(np.float32)
    idx = vc.Index(vc.Space.Cosine, num_dimensions=16, M=64, ef_construction=1024)
    assert idx.add_items(x[:40], ids=np.arange(100, 140)) == list(range(100, 140))
    idx.add_items(x[40:45], ids=[100, 101, 300, 301, 302])          # two existing ids, three new ones
    assert len(idx) == 43 and 300 in idx and 100 in idx and 7 not in idx
    np.testing.assert_array_equal(idx._rows[idx._row_of(100)], x[40])  # replaced in place, not appended
    np.testing.assert_array_equal(idx._rows[idx._row_of(302)], x[44])
    assert sorted(idx.ids) == sorted(list(range(100, 140)) + [300, 301, 302])
    with pytest.raises(KeyError):
        idx._row_of(9999)
    # the vectorised lookup: -1 for a missing id, or KeyError naming the first missing id; any shape
    ids = np.array([[300, 7, 100], [9999, 139, 302]], dtype=np.uint64)
    np.testing.assert_array_equal(idx._rows_of(ids, strict=False), [[40, -1, 0], [-1, 39, 42]])
    with pytest.raises(KeyError, match="id 7 not in index"):
        idx._rows_of(ids, strict=True)
    ident = vc.Index(vc.Space.Cosine, num_dimensions=16)
    ident.add_items(x[:5])
    np.testing.assert_array_equal(ident._rows_of([4, 5, -1, 0], strict=False), [4, -1, -1, 0])
    assert ident._rows_of([], strict=True).shape == (0,)
    with pytest.raises(vc.RecallError):
        idx.query(x[0], k=44)
    p = tmp_path / "i.amix"
    idx.save(str(p))
    back = vc.Index.load(str(p))
    assert len(back) == 43 and back.ids == idx.ids and back.space == vc.Space.Cosine
    np.testing.assert_array_equal(back._rows, idx._rows)
    plain = vc.Index(vc.Space.Euclidean, num_dimensions=16)
    assert plain.add_items(x[:3]) == [0, 1, 2] and plain.add_item(x[3]) == 3 and plain._identity_ids


def test_numa_binding_is_best_effort_without_a_gpu():
    """dist.bind_to_gpu_numa_node never raises: no CUDA device / no sysfs topology -> None and the affinity is untouched"""
    import os
    from audiomuse_ai_b200 import dist as amdist
    before = os.sched_getaffinity(0)
    assert amdist.bind_to_gpu_numa_node(0) is None
    assert os.sched_getaffinity(0) == before
