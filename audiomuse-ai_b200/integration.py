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

import logging
import os
import sys

logger = logging.getLogger(__name__)

CLAP_NAMES = ("compute_mel_spectrogram", "analyze_audio_file", "initialize_clap_audio_model", "get_clap_audio_model",
              "unload_clap_audio_only", "unload_clap_model", "is_clap_model_loaded", "is_clap_audio_loaded")


def _apply_clap_text(text_module, clap_module) -> None:
    from . import clap_analyzer as b200_clap

    def _load_text_model():
        path = text_module.config.CLAP_TEXT_MODEL_PATH
        logger.info("Loading CLAP text model from %s on the GPU", path)
        return b200_clap.B200TextSession(path=path)

    text_module._load_text_model = _load_text_model
    if clap_module is None:
        return
    unload_audio, audio_loaded = clap_module.unload_clap_model, clap_module.is_clap_model_loaded

    def unload_clap_model() -> bool:
        freed = unload_audio()
        session = text_module._text_session
        if session is not None:
            try:
                close = getattr(session, "close", None)
                if close is not None:
                    close()
            finally:
                text_module._text_session = None
                text_module._tokenizer = None
            freed = True
        return freed

    def is_clap_model_loaded() -> bool:
        return audio_loaded() or text_module._text_session is not None

    clap_module.unload_clap_model = unload_clap_model
    clap_module.is_clap_model_loaded = is_clap_model_loaded


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


RADIUS_WALK_NAMES = ("_radius_walk_get_candidates", "_execute_radius_walk")


def make_radius_walk(vm):
    """Replacements for voyager_manager._radius_walk_get_candidates (tasks/voyager_manager.py:842-938) and
    _execute_radius_walk (:941-1367), patched as a pair: find_nearest_neighbors_by_id (:1469-1487) is their only
    caller.  The candidate step keeps the reference's three filters and their fallbacks but no longer fetches one vector
    per candidate (each get_vector is a device-to-host copy over the shim) or computes anchor distances on the host: it
    hands on the candidates' index ids, and the walk runs anchor distances, sort, bucketed greedy walk, artist rules
    and the triple-adjacency pass in one device call (am_knn_radius_walk).  Everything is looked up on `vm` at call
    time, as the reference's own module globals are."""

    def _radius_walk_get_candidates_b200(target_item_id, anchor_vector, initial_results, db_conn,
                                         original_song_details, eliminate_duplicates, mood_similarity=None):
        from app_helper import get_score_data_by_ids

        if not initial_results:
            return []
        try:
            temp = vm._filter_by_distance([{"item_id": target_item_id, "distance": 0.0}] + initial_results, db_conn)
            results = [s for s in temp if s["item_id"] != target_item_id]
        except Exception:
            logger.exception("Radius walk: distance-based pre-filter failed, continuing with original candidate set.")
            results = initial_results
        try:
            unique = vm._deduplicate_and_filter_neighbors(results, db_conn, original_song_details)
        except Exception:
            logger.exception("Radius walk: name-based dedupe failed, continuing without it.")
            unique = results
        try:
            if vm.MOOD_SIMILARITY_ENABLE if mood_similarity is None else mood_similarity:
                unique = vm._filter_by_mood_similarity(unique, target_item_id, db_conn)
        except Exception:
            logger.exception("Radius walk: mood-based pre-filter failed, continuing without it.")
        if not unique:
            return []
        try:
            details = {d["item_id"]: d for d in get_score_data_by_ids([r["item_id"] for r in unique])}
        except Exception:
            details = {}
        out = []
        for song in unique:
            row = vm.reverse_id_map.get(song["item_id"])
            if row is None:   # _get_cached_vector returns None: the reference drops the candidate
                continue
            info = details.get(song["item_id"], {})
            out.append({"item_id": song["item_id"], "row": row, "title": info.get("title"),
                        "author": info.get("author")})
        return out

    def _execute_radius_walk_b200(target_item_id, n, candidate_data, original_song_details=None,
                                  eliminate_duplicates=False):
        if not candidate_data:
            return []
        anchor = vm._get_cached_vector(target_item_id)
        if anchor is None:
            raise KeyError(f"radius walk: anchor item {target_item_id!r} is not in the loaded index")
        artist_ids = {}
        artists = [artist_ids.setdefault(c["author"], len(artist_ids)) if c.get("author") else -1
                   for c in candidate_data]
        pos, dist = vm.voyager_index.radius_walk(anchor, [c["row"] for c in candidate_data], artists, n,
                                                 eliminate_duplicates, vm.MAX_SONGS_PER_ARTIST, vm.VOYAGER_METRIC)
        return [{"item_id": candidate_data[p]["item_id"], "distance": float(d)} for p, d in zip(pos, dist)]

    return _radius_walk_get_candidates_b200, _execute_radius_walk_b200


SIMILAR_NAMES = ("find_nearest_neighbors_by_id", "find_nearest_neighbors_by_vector", "get_max_distance_for_id")

METRIC_NAMES = ("silhouette_score", "davies_bouldin_score", "calinski_harabasz_score")


def apply(clap=None, voyager_manager=None, clustering=None, allow_sklearn_fallback: bool = True,
          clustering_helper=None, song_alchemy=None, app_map=None, artist_gmm_manager=None,
          gaussian_mixture=None, radius_walk=None, path_manager=None, app_path=None, analysis=None, alchemy=None,
          app_alchemy=None, similar=None, app_voyager=None, sonic_fingerprint=None,
          gmm_all_covariance_types: bool = False, clap_text=None, clustering_batch=None) -> None:
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
    that class to the reference.  With gmm_all_covariance_types=True it gets GPUGaussianMixtureAnyCovariance instead,
    which also fits config.GMM_COVARIANCE_TYPE = 'diag', 'tied' and 'spherical' on the device (GPUGaussianMixture
    refuses them, and the reference's _apply_clustering_model then fits scikit-learn on the CPU).  radius_walk (the
    reference's tasks.voyager_manager again) gets the device radius walk: _radius_walk_get_candidates and _execute_radius_walk are replaced together (make_radius_walk);
    voyager_manager= alone leaves the walk to the reference.  path_manager (the reference's tasks.path_manager) gets the
    device song path as find_path_between_songs (song_path.make_song_path, over the voyager_manager module whose
    functions path_manager imported); app_path binds that name when it is imported (app_path.py:5), so pass it too for
    the Song Path endpoint to use it.  alchemy (the reference's tasks.song_alchemy) gets the device Song Alchemy as
    song_alchemy (alchemy.make_song_alchemy, over the voyager_manager module whose functions song_alchemy imported);
    app_alchemy binds that name when it is imported (app_alchemy.py:4), so pass it too for the Alchemy endpoint to use
    it.  song_alchemy= alone still only replaces _project_with_umap.  similar (the reference's tasks.voyager_manager
    again) gets the device plain similar-tracks requests as find_nearest_neighbors_by_id,
    find_nearest_neighbors_by_vector and get_max_distance_for_id (similar_tracks.make_*); app_voyager
    (app_voyager.py:10-12) and sonic_fingerprint (tasks.sonic_fingerprint_manager, :7) bind those names when they are
    imported, so pass them too for their endpoints to use them, and app_path (app_path.py:6) gets
    find_nearest_neighbors_by_vector when similar= is passed with it.  analysis (the reference's tasks.analysis) gets track_features.LibrosaFacade as
    its `librosa`: analyze_track's beat_track, rms and chroma_stft (:344-348) run on the device, every other librosa use
    of the module goes to the librosa it imported; sys.modules["librosa"] is left alone.  clap_text (the reference's
    tasks.clap_analyzer) gets a _load_text_model that returns a B200TextSession over config.CLAP_TEXT_MODEL_PATH, read
    when it is called; initialize_clap_text_model looks that name up at call time (:300), so text search's query
    embeddings and get_text_embeddings_batch run on the device while the tokenizer, get_text_embedding and
    search_by_text stay the reference's.  With clap= as well, the installed unload_clap_model and is_clap_model_loaded
    also close and clear the module's _text_session (and its tokenizer, as the reference's unload does), so the idle
    unload timer frees the text model too.  clustering_batch (the reference's tasks.clustering) gets
    clustering_batch.make_run_clustering_batch_task as run_clustering_batch_task: RQ resolves
    'tasks.clustering.run_clustering_batch_task' by name when a batch job runs (clustering.py:884-887), and the drop-in
    fits a batch's k-means iterations in one device pass.  It builds the reference's GPUKMeans, so clustering= must
    be passed too."""
    if clustering_batch is not None and clustering is None:
        raise ValueError("clustering_batch= builds the device GPUKMeans that clustering= installs: pass both")
    if gmm_all_covariance_types and gaussian_mixture is None:
        raise ValueError("gmm_all_covariance_types= selects the class installed by gaussian_mixture=: pass both")
    if analysis is not None:
        from . import track_features

        if not isinstance(analysis.librosa, track_features.LibrosaFacade):
            analysis.librosa = track_features.LibrosaFacade(analysis.librosa)
    if clap is not None:
        from . import clap_analyzer as b200_clap

        for name in CLAP_NAMES:
            setattr(clap, name, getattr(b200_clap, name))
    if clap_text is not None:
        _apply_clap_text(clap_text, clap)
    if voyager_manager is not None:
        voyager_manager._filter_by_distance = make_filter_by_distance(voyager_manager)
    if radius_walk is not None:
        for name, fn in zip(RADIUS_WALK_NAMES, make_radius_walk(radius_walk)):
            setattr(radius_walk, name, fn)
    if app_path is not None and path_manager is None and similar is None:
        raise ValueError("app_path= takes the device song path from path_manager=: pass both")
    if (app_voyager is not None or sonic_fingerprint is not None) and similar is None:
        raise ValueError("app_voyager= / sonic_fingerprint= take the device similar-tracks requests from similar=: "
                         "pass it too")
    if similar is not None:
        from . import similar_tracks

        fns = {name: getattr(similar_tracks, "make_" + name)(similar) for name in SIMILAR_NAMES}
        for name, fn in fns.items():
            setattr(similar, name, fn)
            if app_voyager is not None:
                setattr(app_voyager, name, fn)
        if sonic_fingerprint is not None:
            sonic_fingerprint.find_nearest_neighbors_by_vector = fns["find_nearest_neighbors_by_vector"]
        if app_path is not None:
            app_path.find_nearest_neighbors_by_vector = fns["find_nearest_neighbors_by_vector"]
    if path_manager is not None:
        from . import song_path

        fn = song_path.make_song_path(sys.modules[path_manager.get_vector_by_id.__module__], path_manager)
        path_manager.find_path_between_songs = fn
        if app_path is not None:
            app_path.find_path_between_songs = fn
    if app_alchemy is not None and alchemy is None:
        raise ValueError("app_alchemy= takes the device Song Alchemy from alchemy=: pass both")
    if alchemy is not None:
        from . import alchemy as b200_alchemy

        fn = b200_alchemy.make_song_alchemy(alchemy, sys.modules[alchemy.find_nearest_neighbors_by_id.__module__])
        alchemy.song_alchemy = fn
        if app_alchemy is not None:
            app_alchemy.song_alchemy = fn
    if clustering is not None:
        from . import clustering_gpu as b200_cg

        clustering.GPUKMeans = b200_cg.GPUKMeans
        clustering.GPUDBSCAN = b200_cg.GPUDBSCAN   # get_clustering_model / get_pca_model look the classes up at call time
        clustering.GPUPCA = b200_cg.GPUPCA
        clustering.GPUSpectralClustering = b200_cg.GPUSpectralClustering
        clustering.check_gpu_available = b200_cg.check_gpu_available
    if clustering_batch is not None:
        from . import clustering_batch as b200_cb

        clustering_batch.run_clustering_batch_task = b200_cb.make_run_clustering_batch_task(
            clustering_batch, sys.modules[clustering_batch._perform_single_clustering_iteration.__module__])
    if gaussian_mixture is not None:
        from . import clustering_gpu as b200_cg

        gaussian_mixture.GPUGaussianMixture = (b200_cg.GPUGaussianMixtureAnyCovariance if gmm_all_covariance_types
                                               else b200_cg.GPUGaussianMixture)
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
