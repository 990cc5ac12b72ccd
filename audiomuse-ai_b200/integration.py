"""The patch a maintainer applies to AudioMuse-AI (INTEGRATION.md section 3), as code.

    from audiomuse_ai_b200 import integration
    integration.install_voyager_shim()      # BEFORE `import tasks.voyager_manager` / `tasks.clap_text_search`
    import tasks.clap_analyzer, tasks.voyager_manager, tasks.clustering_gpu
    integration.apply(clap=tasks.clap_analyzer, voyager_manager=tasks.voyager_manager, clustering=tasks.clustering_gpu)

Nothing in the reference tree is modified; every assignment below replaces a module attribute that the reference's
own callers look up at call time (tasks/analysis.py:883 imports analyze_audio_file as clap_analyze from the module,
tasks/voyager_manager.py:1594 calls the module-level _filter_by_distance, clustering_helper.py:21 calls
get_clustering_model).  tests/test_reference_shims.py applies exactly this to the stub-imported reference modules.
"""
from __future__ import annotations

import os
import sys

CLAP_NAMES = ("compute_mel_spectrogram", "analyze_audio_file", "initialize_clap_audio_model", "get_clap_audio_model",
              "unload_clap_audio_only", "unload_clap_model", "is_clap_model_loaded", "is_clap_audio_loaded")


def install_voyager_shim() -> None:
    """`import voyager` in tasks/voyager_manager.py:12 and tasks/clap_text_search.py resolves to the flat exact index:
    Index(space, num_dimensions, M, ef_construction), add_items, query, get_vector, len, .ef, save / load,
    Space.Cosine, RecallError."""
    from . import voyager_compat

    sys.modules["voyager"] = voyager_compat


def make_filter_by_distance(vm):
    """voyager_manager._filter_by_distance (tasks/voyager_manager.py:526-617) on the vectors already in HBM: one
    device walk instead of O(k) get_vector calls + Python distance loops.  Keeps exactly the items upstream keeps
    (tests/golden/filter_golden.npz)."""

    def _filter_by_distance_b200(song_results, db_conn):
        if vm.DUPLICATE_DISTANCE_CHECK_LOOKBACK <= 0 or not song_results:
            return song_results
        ids = [vm.reverse_id_map.get(s["item_id"], -1) for s in song_results]   # unknown item -> dropped, as upstream
        thr = (vm.DUPLICATE_DISTANCE_THRESHOLD_COSINE if vm.VOYAGER_METRIC == "angular"
               else vm.DUPLICATE_DISTANCE_THRESHOLD_EUCLIDEAN)
        keep = vm.voyager_index.filter_by_distance([-1 if i is None else i for i in ids], thr,
                                                   lookback=vm.DUPLICATE_DISTANCE_CHECK_LOOKBACK,
                                                   batch=vm.BATCH_SIZE_VECTOR_OPS)
        return [s for s, k in zip(song_results, keep) if k]

    return _filter_by_distance_b200


METRIC_NAMES = ("silhouette_score", "davies_bouldin_score", "calinski_harabasz_score")


def apply(clap=None, voyager_manager=None, clustering=None, allow_sklearn_fallback: bool = True,
          clustering_helper=None, song_alchemy=None, app_map=None, artist_gmm_manager=None,
          gaussian_mixture=None) -> None:
    """clap / voyager_manager / clustering / clustering_helper: the reference's already imported tasks.* modules (pass
    only the ones to patch).  allow_sklearn_fallback keeps the reference's contract that a failing GPU k-means silently
    falls back to scikit-learn (tasks/clustering_gpu.py:130-148); this repository's own tests run with it off so a
    missing CUDA library can never pass as the GPU path.  clustering_helper imports the three scores by name at module
    level (tasks/clustering_helper.py:16) and looks them up at call time (:462-470), so replacing the module attributes
    moves the fitness scoring to the GPU.  song_alchemy / app_map get the GPU UMAP projection as _project_with_umap:
    app_helper imports it from tasks.song_alchemy at call time (app_helper.py:1320, 1437), app_map binds it when it is
    imported (app_map.py:13), so both modules are patched.  artist_gmm_manager gets the GPU fit_artist_gmm and
    select_optimal_gmm_components; build_and_store_artist_index looks both up at call time (:556, :185), and the
    reference's own functions are kept for the B200_ALLOW_SKLEARN_FALLBACK=1 path.  That module runs `import voyager`
    when it is imported, so install_voyager_shim() must come before `import tasks.artist_gmm_manager` and before
    `import tasks.analysis`, which imports it.  gaussian_mixture (the reference's tasks.clustering_gpu again) gets the
    GPU GPUGaussianMixture; get_clustering_model looks the class up at call time (:385).  clustering= alone leaves
    that class to the reference."""
    if clap is not None:
        from . import clap_analyzer as b200_clap

        for name in CLAP_NAMES:
            setattr(clap, name, getattr(b200_clap, name))
    if voyager_manager is not None:
        voyager_manager._filter_by_distance = make_filter_by_distance(voyager_manager)
    if clustering is not None:
        from . import clustering_gpu as b200_cg

        clustering.GPUKMeans = b200_cg.GPUKMeans
        clustering.GPUDBSCAN = b200_cg.GPUDBSCAN   # get_clustering_model / get_pca_model look the classes up at call time
        clustering.GPUPCA = b200_cg.GPUPCA
        clustering.GPUSpectralClustering = b200_cg.GPUSpectralClustering
        clustering.check_gpu_available = b200_cg.check_gpu_available
    if gaussian_mixture is not None:
        from . import clustering_gpu as b200_cg

        gaussian_mixture.GPUGaussianMixture = b200_cg.GPUGaussianMixture
    if clustering_helper is not None:
        from . import cluster_metrics as b200_cm

        for name in METRIC_NAMES:
            setattr(clustering_helper, name, getattr(b200_cm, name))
    for mod in (song_alchemy, app_map):
        if mod is not None:
            from . import projection

            mod._project_with_umap = projection.project_with_umap
    if artist_gmm_manager is not None:
        from . import artist_gmm

        artist_gmm.capture_originals(artist_gmm_manager)
        artist_gmm_manager.fit_artist_gmm = artist_gmm.fit_artist_gmm
        artist_gmm_manager.select_optimal_gmm_components = artist_gmm.select_optimal_gmm_components
    if (clustering is not None or clustering_helper is not None or artist_gmm_manager is not None
            or gaussian_mixture is not None) and allow_sklearn_fallback:
        os.environ.setdefault("B200_ALLOW_SKLEARN_FALLBACK", "1")
