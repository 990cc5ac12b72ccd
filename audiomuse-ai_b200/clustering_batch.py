"""tasks/clustering.py:112-249 run_clustering_batch_task with every k-means fit of the batch in one device pass.

The reference runs each iteration start to finish: subset, data, parameters, PCA, one KMeans(k, n_init=10) fit, score.
None of the steps before the fit reads what an earlier fit produced, and the fits draw nothing from Python's or numpy's
generators (GPUKMeans seeds its own generator with 0), so the drop-in prepares every iteration in the reference's order
with the reference's own functions, fits all of them with one clustering_gpu.kmeans_fit_batch, and then scores and
reports each iteration in order as the reference does.  Every draw of `random` / `np.random` is the reference's.

    make_run_clustering_batch_task(task_module, helper) -> run_clustering_batch_task
        task_module: the reference's tasks.clustering (the original function, get_current_job, _sanitize_for_json,
        _get_stratified_song_subset);
        helper: its tasks.clustering_helper (the iteration steps, USE_GPU_CLUSTERING, GPU_CLUSTERING_AVAILABLE,
        get_clustering_model, get_pca_model), both read at call time.

The original function runs unchanged when the method is not 'kmeans' or GPU clustering is off or unavailable.  A fit
the device refuses or fails sends those iterations through the reference's _apply_clustering_model, with its own GPU
-> scikit-learn fallback.
"""
from __future__ import annotations

import json
import logging
import uuid

import numpy as np

from . import clustering_gpu

logger = logging.getLogger("tasks.clustering")

# GPUKMeans's defaults, which the reference's get_clustering_model('kmeans', ...) leaves in place
N_INIT, MAX_ITER, TOL, SEED = 10, 300, 1e-4, 0


class _Stop(Exception):
    """raised by the preparation loop: the iterations prepared so far are fitted and reported first"""

    def __init__(self, kind, index, payload=None):
        super().__init__(kind)
        self.kind, self.index, self.payload = kind, index, payload


def make_run_clustering_batch_task(task_module, helper):
    original = task_module.run_clustering_batch_task

    def run_clustering_batch_task(batch_id_str, start_run_idx, num_iterations_in_batch,
                                  genre_to_lightweight_track_data_map_json, target_songs_per_genre,
                                  sampling_percentage_change_per_run, clustering_method, active_mood_labels_for_batch,
                                  num_clusters_min_max_tuple, dbscan_params_ranges_dict, gmm_params_ranges_dict,
                                  spectral_params_ranges_dict, pca_params_ranges_dict, max_songs_per_cluster,
                                  parent_task_id, score_weights_dict, elite_solutions_params_list_json,
                                  exploitation_probability, mutation_config_json, initial_subset_track_ids_json,
                                  enable_clustering_embeddings_param):
        args = (batch_id_str, start_run_idx, num_iterations_in_batch, genre_to_lightweight_track_data_map_json,
                target_songs_per_genre, sampling_percentage_change_per_run, clustering_method,
                active_mood_labels_for_batch, num_clusters_min_max_tuple, dbscan_params_ranges_dict,
                gmm_params_ranges_dict, spectral_params_ranges_dict, pca_params_ranges_dict, max_songs_per_cluster,
                parent_task_id, score_weights_dict, elite_solutions_params_list_json, exploitation_probability,
                mutation_config_json, initial_subset_track_ids_json, enable_clustering_embeddings_param)
        if clustering_method != "kmeans" or not (helper.USE_GPU_CLUSTERING and helper.GPU_CLUSTERING_AVAILABLE):
            return original(*args)

        from app import app
        from app_helper import (redis_conn, save_task_status, get_task_info_from_db,
                                TASK_STATUS_PROGRESS, TASK_STATUS_REVOKED, TASK_STATUS_FAILURE,
                                TASK_STATUS_SUCCESS)

        current_job = task_module.get_current_job(redis_conn)
        current_task_id = current_job.id if current_job else str(uuid.uuid4())
        logger.info(f"Starting clustering batch task {current_task_id} (Batch: {batch_id_str})")
        log_prefix = f"[Batch-{current_task_id}]"

        with app.app_context():
            def _log_and_update(message, progress, details=None, state=TASK_STATUS_PROGRESS):
                logger.info(f"[ClusteringBatchTask-{current_task_id}] {message}")
                db_details = {"batch_id": batch_id_str, "start_run_idx": start_run_idx,
                              "num_iterations_in_batch": num_iterations_in_batch, "status_message": message,
                              **(details or {})}
                if current_job:
                    current_job.meta['progress'] = progress
                    current_job.meta['status_message'] = message
                    current_job.save_meta()
                save_task_status(current_task_id, "clustering_batch", state, parent_task_id=parent_task_id,
                                 sub_type_identifier=batch_id_str, progress=progress, details=db_details)

            try:
                _log_and_update("Batch started.", 0)
                genre_map = json.loads(genre_to_lightweight_track_data_map_json)
                elites = json.loads(elite_solutions_params_list_json)
                mutation_config = json.loads(mutation_config_json)
                state = {"ids": json.loads(initial_subset_track_ids_json), "best": None, "best_score": -1.0,
                         "done": 0}

                # 1. prepare every iteration in the reference's order, until the batch ends or must stop
                prepared, stop = [], None
                try:
                    for i in range(num_iterations_in_batch):
                        run_idx = start_run_idx + i
                        if current_job:
                            task_info = get_task_info_from_db(current_task_id)
                            parent_info = get_task_info_from_db(parent_task_id)
                            if (task_info and task_info.get('status') == TASK_STATUS_REVOKED) or \
                               (parent_info and parent_info.get('status') in [TASK_STATUS_REVOKED,
                                                                               TASK_STATUS_FAILURE]):
                                raise _Stop("revoked", i)
                        pct = 0.0 if i == 0 else sampling_percentage_change_per_run
                        subset = task_module._get_stratified_song_subset(genre_map, target_songs_per_genre,
                                                                    prev_ids=state["ids"], percent_change=pct)
                        item_ids = [t['item_id'] for t in subset]
                        state["ids"] = list(item_ids)
                        if not item_ids:
                            logger.warning(f"No songs in subset for iteration {run_idx}. Skipping.")
                            continue
                        try:
                            it = _prepare(helper, app, run_idx, item_ids, clustering_method,
                                          num_clusters_min_max_tuple, dbscan_params_ranges_dict,
                                          gmm_params_ranges_dict, spectral_params_ranges_dict, pca_params_ranges_dict,
                                          active_mood_labels_for_batch, log_prefix, elites, exploitation_probability,
                                          mutation_config, enable_clustering_embeddings_param)
                        except Exception as e:
                            logger.error(f"{log_prefix} Iteration {run_idx} failed critically", exc_info=True)
                            raise _Stop("error", i, e)
                        prepared.append((i, it))
                except _Stop as s:
                    stop = s

                # 2. one device pass over every k-means fit, 3. score and report each iteration in order
                _fit_all(helper, [it for _, it in prepared], log_prefix)
                for i, it in prepared:
                    result = _score(helper, it, active_mood_labels_for_batch, max_songs_per_cluster,
                                    enable_clustering_embeddings_param, score_weights_dict, log_prefix)
                    state["done"] += 1
                    if result and result.get("fitness_score", -1.0) > state["best_score"]:
                        state["best_score"] = result["fitness_score"]
                        state["best"] = result
                    progress = int(100 * (i + 1) / num_iterations_in_batch)
                    _log_and_update(f"Iteration {start_run_idx + i} complete. Batch best score: "
                                    f"{state['best_score']:.2f}", progress)
                if stop is not None and stop.kind == "revoked":
                    _log_and_update("Stopping batch due to revocation.", stop.index, state=TASK_STATUS_REVOKED)
                    return {"status": "REVOKED", "message": "Batch task revoked."}
                if stop is not None:
                    raise stop.payload

                best = state["best"]
                if best:
                    best = task_module._sanitize_for_json(best)
                final_details = {"best_score_in_batch": state["best_score"],
                                 "iterations_completed_in_batch": state["done"],
                                 "full_best_result_from_batch": best, "final_subset_track_ids": state["ids"]}
                _log_and_update(f"Batch complete. Best score: {state['best_score'] or -1:.2f}", 100,
                                details=final_details, state=TASK_STATUS_SUCCESS)
                return {"status": "SUCCESS", "iterations_completed_in_batch": state["done"],
                        "best_result_from_batch": best, "final_subset_track_ids": state["ids"]}
            except Exception as e:
                logger.error(f"Clustering batch {batch_id_str} failed", exc_info=True)
                _log_and_update(f"Batch failed: {e}", 100, details={"error": str(e)}, state=TASK_STATUS_FAILURE)
                return {"status": "FAILURE", "message": str(e)}

    run_clustering_batch_task.__wrapped__ = original
    return run_clustering_batch_task


def _prepare(helper, app, run_idx, item_ids, method, k_range, dbscan_r, gmm_r, spectral_r, pca_r, moods, log_prefix,
             elites, exploit_p, mutation_cfg, use_embeddings):
    """steps 1-4 of _perform_single_clustering_iteration (tasks/clustering_helper.py:60-96) -> the iteration's state;
    'result' is set when the reference would return before the fit"""
    it = {"run_idx": run_idx, "result": None}
    with app.app_context():
        valid_tracks, X_feat, X_embed = helper._prepare_iteration_data(item_ids, moods, use_embeddings, log_prefix,
                                                                       run_idx)
    if valid_tracks is None:
        it["result"] = {"fitness_score": -1.0}
        return it
    data, scaler = helper._prepare_and_scale_data(X_feat, X_embed, use_embeddings)
    if data is None:
        logger.error(f"{log_prefix} Iteration {run_idx}: Data for clustering is empty after prep. Cannot proceed.")
        it["result"] = {"fitness_score": -1.0}
        return it
    params = helper._generate_evolutionary_parameters(elites, exploit_p, mutation_cfg, method, data, pca_r, k_range,
                                                      dbscan_r, gmm_r, spectral_r, log_prefix, run_idx)
    pca_model, data_after_pca = None, data
    if params['pca_config']['enabled']:
        pca_model = helper.get_pca_model(n_components=params['pca_config']['components'], use_gpu=True)
        data_after_pca = pca_model.fit_transform(data)
        params['pca_config']['components'] = pca_model.n_components_
    it.update(valid_tracks=valid_tracks, X_feat=X_feat, data=data_after_pca, scaler=scaler, params=params,
              pca=pca_model, labels=None, centers=None, model=None)
    if params['clustering_method_config']['params'].get('n_clusters', 0) < 2:
        it["result"] = {"fitness_score": -1.0}      # _apply_clustering_model's rule (:268-270)
    return it


def _fit_all(helper, its, log_prefix):
    """every pending k-means fit in one kmeans_fit_batch; a fit it refuses or fails goes through the reference's
    _apply_clustering_model, one iteration at a time"""
    todo = [it for it in its if it["result"] is None]
    ks = [int(it["params"]['clustering_method_config']['params']['n_clusters']) for it in todo]
    fits = [None] * len(todo)
    # a problem kmeans_fit_batch would refuse (k > N, no features, NaN / inf) takes the per-iteration path alone
    ok = [j for j, it in enumerate(todo) if _fits_batch(it["data"], ks[j])]
    if ok:
        try:
            res = clustering_gpu.kmeans_fit_batch([todo[j]["data"] for j in ok], [ks[j] for j in ok], n_init=N_INIT,
                                                  max_iter=MAX_ITER, tol=TOL, seeds=SEED)
            for j, r in zip(ok, res):
                fits[j] = r
        except Exception as e:
            logger.warning(f"{log_prefix} batched GPU k-means failed, fitting its {len(ok)} iterations one by one: {e}")
    for it, fit in zip(todo, fits):
        mc = it["params"]['clustering_method_config']
        if fit is None:
            it["labels"], it["centers"], it["model"] = helper._apply_clustering_model(it["data"], mc, log_prefix,
                                                                                      it["run_idx"])
            if it["labels"] is None:
                it["result"] = {"fitness_score": -1.0}
            continue
        model = helper.get_clustering_model(mc['method'], mc['params'], use_gpu=True)
        model.cluster_centers_, model.labels_, model.inertia_, model.n_iter_ = fit
        model.using_gpu = True
        it["labels"], it["model"] = model.labels_, model
        it["centers"] = {i: c for i, c in enumerate(model.cluster_centers_)}


def _fits_batch(data, k):
    X = np.asarray(data)
    if X.ndim != 2 or X.shape[1] < 1 or not 1 <= k <= X.shape[0]:
        return False
    with np.errstate(over="ignore"):
        return bool(np.isfinite(X).all() and np.isfinite(X.astype(np.float32)).all())


def _score(helper, it, moods, max_songs, use_embeddings, weights, log_prefix):
    if it["result"] is not None:
        return it["result"]
    return helper._format_and_score_iteration_result(
        it["labels"], it["valid_tracks"], it["X_feat"], it["data"], it["centers"], it["model"], it["pca"],
        it["scaler"], moods, it["params"], max_songs, it["run_idx"], use_embeddings, weights, log_prefix)
