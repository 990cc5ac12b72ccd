"""The per-phase device times the library reports (CUDA events around each phase): after one small call, every phase
of the spectral and UMAP plans, of am_gmm_fit for each covariance type and of the artist-GMM sweep has taken a finite,
positive time."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _blobs(n, d, k, seed):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((k, d)) * 3.0
    return (c[rng.integers(0, k, n)] + rng.standard_normal((n, d))).astype(np.float32)


def _check(where, times):
    for name, ms in times.items():
        assert math.isfinite(ms) and ms > 0.0, f"{where}: {name} = {ms}"


def test_every_phase_time_is_finite_and_positive():
    from audiomuse_ai_b200 import artist_gmm as ag, clustering_gpu as cg, projection

    X = _blobs(1000, 16, 4, 0)
    det = {}
    cg.spectral_embedding(X, 4, n_neighbors=10, seed=0, details=det)
    _check("am_spectral_plan_info", {k: det[k] for k in ("knn_ms", "graph_ms")})
    det = {}
    projection.umap_fit_transform(X, n_epochs=20, seed=0, details=det)
    _check("am_umap_plan_info", {k: det[k] for k in ("knn_ms", "graph_ms", "layout_ms")})
    for cov in ("full", "tied", "diag", "spherical"):
        f = cg.gmm_fit(X.astype(np.float64), 4, n_init=2, max_iter=3, random_state=0, covariance_type=cov)
        assert len(f.phase_ms) == 5
        _check(f"am_gmm_fit ({cov})", f.phase_ms)
    timings = {}
    ag.fit_artist_gmms([_blobs(60, 16, 2, 1), _blobs(40, 16, 3, 2)], timings=timings)
    _check("am_artist_gmm_fit", timings)
