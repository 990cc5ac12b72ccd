"""The run_clustering_batch_task drop-in (clustering_batch.py) on the host, with stand-in task / helper modules and a
recording fake in place of the device fit.  The oracle is `reference_loop`, a restatement of tasks/clustering.py:112-249
over the same helper functions (one _apply_clustering_model per iteration): under the same seeded `random` /
`np.random` both must hand the fit the same (subset, parameters, data bytes) per iteration, make the same status calls
and return the same dict."""
import json
import random
import sys
import types
import uuid

import numpy as np
import pytest

from audiomuse_ai_b200 import clustering_batch, clustering_gpu, integration

N_TRACKS, D_FEAT, D_EMBED = 3000, 9, 24


class Env:
    def __init__(self, revoke_at=None, fail_prepare_at=None):
        rng = np.random.default_rng(0)
        self.feat = {f"t{i}": rng.random(D_FEAT) for i in range(N_TRACKS)}
        self.embed = {f"t{i}": rng.standard_normal(D_EMBED) for i in range(N_TRACKS)}
        self.genre_map = {g: [{"item_id": f"t{i}"} for i in range(g, N_TRACKS, 4)] for g in range(4)}
        self.status, self.fits, self.calls = [], [], 0
        self.revoke_at, self.fail_prepare_at = revoke_at, fail_prepare_at
        self.helper = self._helper()
        self.task = self._task()

    # ---- tasks.clustering_helper stand-in: each step draws from `random` / np.random as the reference's do
    def _helper(self):
        env = self
        h = types.SimpleNamespace(USE_GPU_CLUSTERING=True, GPU_CLUSTERING_AVAILABLE=True)

        def prepare(ids, moods, use_emb, log_prefix, run_idx):
            if env.fail_prepare_at == run_idx:
                raise RuntimeError("database gone")
            tracks = [{"item_id": i} for i in ids]
            X = np.array([env.feat[i] for i in ids])
            return tracks, X, (np.array([env.embed[i] for i in ids]) if use_emb else None)

        def scale(X_feat, X_embed, use_emb):
            src = X_embed if use_emb else X_feat
            return (src - src.mean(0)) / src.std(0), "scaler"

        def params(elites, p, mut, method, data, pca_r, k_range, *rest):
            if elites and random.random() < p:
                e = random.choice(elites)
                k = int(np.clip(e["k"] + random.randint(-3, 3), *k_range))
            else:
                k = random.randint(*k_range)
            pca = random.random() < 0.5
            return {"pca_config": {"enabled": pca, "components": random.randint(2, 6) if pca else 0},
                    "clustering_method_config": {"method": method, "params": {"n_clusters": k}}}

        class PCA:
            def __init__(self, n_components):
                self.n_components_ = n_components

            def fit_transform(self, X):
                return X[:, :self.n_components_] * 2.0

        def apply_model(data, mc, log_prefix, run_idx):
            k = mc["params"]["n_clusters"]
            if k < 2:
                return None, None, None
            env.fits.append(("apply", run_idx, mc["params"]["n_clusters"], np.asarray(data, np.float32).tobytes()))
            lab = fake_labels(data, k)
            return lab, {i: np.zeros(2) for i in range(k)}, types.SimpleNamespace(labels_=lab)

        def score(labels, tracks, X_feat, data, centers, model, pca, scaler, moods, params, *rest):
            return {"fitness_score": float(np.bincount(labels).max()) / len(labels) + params["pca_config"]["components"],
                    "params": params, "ids": [t["item_id"] for t in tracks], "centers": len(centers)}

        h._prepare_iteration_data = prepare
        h._prepare_and_scale_data = scale
        h._generate_evolutionary_parameters = params
        h.get_pca_model = lambda n_components, use_gpu: PCA(n_components)
        h._apply_clustering_model = apply_model
        h._format_and_score_iteration_result = score
        h.get_clustering_model = lambda method, params, use_gpu: clustering_gpu.GPUKMeans(params["n_clusters"])
        return h

    def _task(self):
        env = self
        t = types.SimpleNamespace()

        def subset(genre_map, target, prev_ids=None, percent_change=0.0):
            ids = [x["item_id"] for g in genre_map.values() for x in g]
            return [{"item_id": i} for i in random.sample(ids, min(target, len(ids)))] if target else []

        class Job:
            id = "job1"
            meta = {}

            def save_meta(self):
                pass

        t._get_stratified_song_subset = subset
        t.get_current_job = lambda conn: Job()
        t._sanitize_for_json = lambda o: json.loads(json.dumps(o, default=lambda v: v.tolist()))
        t.run_clustering_batch_task = lambda *a: reference_loop(env, *a)
        return t

    def install_app(self, monkeypatch):
        env = self
        monkeypatch.setitem(sys.modules, "app", types.SimpleNamespace(app=types.SimpleNamespace(
            app_context=lambda: _Ctx())))

        def info(task_id):
            if task_id == "job1":
                env.calls += 1
                if env.revoke_at is not None and env.calls > env.revoke_at:
                    return {"status": "REVOKED"}
            return {"status": "PROGRESS"}

        monkeypatch.setitem(sys.modules, "app_helper", types.SimpleNamespace(
            redis_conn=None, get_task_info_from_db=info,
            save_task_status=lambda *a, **k: env.status.append((a, json.dumps(k, sort_keys=True, default=str))),
            TASK_STATUS_PROGRESS="PROGRESS", TASK_STATUS_REVOKED="REVOKED", TASK_STATUS_FAILURE="FAILURE",
            TASK_STATUS_SUCCESS="SUCCESS"))


class _Ctx:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def fake_labels(data, k):
    X = np.asarray(data, np.float32)
    return (np.arange(len(X)) % k).astype(np.int32)


def reference_loop(env, batch_id_str, start_run_idx, num_iterations_in_batch, genre_map_json, target, pct_change,
                   method, moods, k_range, dbscan_r, gmm_r, spectral_r, pca_r, max_songs, parent_task_id, weights,
                   elites_json, exploit_p, mutation_json, initial_ids_json, use_emb):
    """tasks/clustering.py:112-249 with _perform_single_clustering_iteration (clustering_helper.py:45-114) inlined"""
    from app_helper import save_task_status, get_task_info_from_db
    h, t = env.helper, env.task
    job = t.get_current_job(None)
    tid = job.id

    def log(message, progress, details=None, state="PROGRESS"):
        d = {"batch_id": batch_id_str, "start_run_idx": start_run_idx, "num_iterations_in_batch": num_iterations_in_batch,
             "status_message": message, **(details or {})}
        save_task_status(tid, "clustering_batch", state, parent_task_id=parent_task_id, sub_type_identifier=batch_id_str,
                         progress=progress, details=d)

    try:
        log("Batch started.", 0)
        genre_map, elites = json.loads(genre_map_json), json.loads(elites_json)
        ids = json.loads(initial_ids_json)
        best, best_score, done = None, -1.0, 0
        for i in range(num_iterations_in_batch):
            run_idx = start_run_idx + i
            ti, pi = get_task_info_from_db(tid), get_task_info_from_db(parent_task_id)
            if (ti and ti.get("status") == "REVOKED") or (pi and pi.get("status") in ["REVOKED", "FAILURE"]):
                log("Stopping batch due to revocation.", i, state="REVOKED")
                return {"status": "REVOKED", "message": "Batch task revoked."}
            sub = t._get_stratified_song_subset(genre_map, target, prev_ids=ids, percent_change=0.0 if i == 0 else pct_change)
            ids = [x["item_id"] for x in sub]
            if not ids:
                continue
            tracks, X_feat, X_embed = h._prepare_iteration_data(ids, moods, use_emb, "", run_idx)
            data, scaler = h._prepare_and_scale_data(X_feat, X_embed, use_emb)
            params = h._generate_evolutionary_parameters(elites, exploit_p, json.loads(mutation_json), method, data,
                                                         pca_r, k_range, dbscan_r, gmm_r, spectral_r, "", run_idx)
            pca, d2 = None, data
            if params["pca_config"]["enabled"]:
                pca = h.get_pca_model(n_components=params["pca_config"]["components"], use_gpu=True)
                d2 = pca.fit_transform(data)
                params["pca_config"]["components"] = pca.n_components_
            labels, centers, model = h._apply_clustering_model(d2, params["clustering_method_config"], "", run_idx)
            res = {"fitness_score": -1.0} if labels is None else h._format_and_score_iteration_result(
                labels, tracks, X_feat, d2, centers, model, pca, scaler, moods, params, max_songs, run_idx, use_emb,
                weights, "")
            done += 1
            if res and res.get("fitness_score", -1.0) > best_score:
                best_score, best = res["fitness_score"], res
            log(f"Iteration {run_idx} complete. Batch best score: {best_score:.2f}", int(100 * (i + 1) / num_iterations_in_batch))
        if best:
            best = t._sanitize_for_json(best)
        log(f"Batch complete. Best score: {best_score or -1:.2f}", 100, details={
            "best_score_in_batch": best_score, "iterations_completed_in_batch": done,
            "full_best_result_from_batch": best, "final_subset_track_ids": ids}, state="SUCCESS")
        return {"status": "SUCCESS", "iterations_completed_in_batch": done, "best_result_from_batch": best,
                "final_subset_track_ids": ids}
    except Exception as e:
        log(f"Batch failed: {e}", 100, details={"error": str(e)}, state="FAILURE")
        return {"status": "FAILURE", "message": str(e)}


def batch_args(env, method="kmeans", k_range=(40, 100), use_emb=False, elites=(), target=250, n=20):
    return ("b0", 100, n, json.dumps(env.genre_map), target, 0.2, method, ["happy"], k_range, {}, {}, {}, {}, 50,
            "parent", {}, json.dumps(list(elites)), 0.7, json.dumps({}), json.dumps([]), use_emb)


def run_both(monkeypatch, fail_fit=False, **kw):
    out = []
    env_kw = {k: kw.pop(k) for k in ("revoke_at", "fail_prepare_at") if k in kw}
    for drop_in in (False, True):
        env = Env(**env_kw)
        env.install_app(monkeypatch)

        def fake_batch(problems, k, n_init, max_iter, tol, seeds):
            assert (n_init, max_iter, tol, seeds) == (10, 300, 1e-4, 0)
            if fail_fit:
                raise RuntimeError("device lost")
            res = []
            for X, kk in zip(problems, k):
                # the rows reach the device as kmeans_fit casts them: float64 data rounded to float32
                env.fits.append(("apply", None, kk, np.asarray(X, np.float32).tobytes()))
                res.append((np.zeros((kk, X.shape[1]), np.float32), fake_labels(X, kk), 1.0, 3))
            return res

        monkeypatch.setattr(clustering_gpu, "kmeans_fit_batch", fake_batch)
        random.seed(7)
        np.random.seed(7)
        fn = clustering_batch.make_run_clustering_batch_task(env.task, env.helper) if drop_in else \
            env.task.run_clustering_batch_task
        ret = fn(*batch_args(env, **kw))
        out.append((ret, env))
    return out


def _same(a, b):
    (ra, ea), (rb, eb) = a, b
    assert json.dumps(ra, sort_keys=True, default=str) == json.dumps(rb, sort_keys=True, default=str)
    assert [f[2:] for f in ea.fits] == [f[2:] for f in eb.fits]
    assert ea.status == eb.status


@pytest.mark.parametrize("use_emb", [False, True])
@pytest.mark.parametrize("elites", [(), ({"k": 60},)])
def test_fit_inputs_status_and_result_match_the_reference_loop(monkeypatch, use_emb, elites):
    ref, new = run_both(monkeypatch, use_emb=use_emb, elites=elites)
    _same(ref, new)
    assert ref[0]["status"] == "SUCCESS" and ref[0]["iterations_completed_in_batch"] == 20
    assert len(new[1].fits) == 20


def test_k_below_two_and_empty_subset(monkeypatch):
    ref, new = run_both(monkeypatch, k_range=(1, 3), n=12)
    _same(ref, new)
    assert len(ref[1].fits) < 12                     # some iterations drew k = 1 and were scored -1
    ref, new = run_both(monkeypatch, target=0, n=5)  # every subset empty: nothing is fitted or counted
    _same(ref, new)
    assert ref[0]["iterations_completed_in_batch"] == 0


def test_revocation_and_failure_mid_batch(monkeypatch):
    ref, new = run_both(monkeypatch, revoke_at=7)
    _same(ref, new)
    assert ref[0]["status"] == "REVOKED"
    ref, new = run_both(monkeypatch, fail_prepare_at=105)
    _same(ref, new)
    assert ref[0]["status"] == "FAILURE"


def test_fit_failure_falls_back_per_iteration(monkeypatch):
    ref, new = run_both(monkeypatch, fail_fit=True)
    _same(ref, new)
    assert new[0]["status"] == "SUCCESS"


def test_other_methods_and_gpu_off_delegate(monkeypatch):
    env = Env()
    seen = []
    env.task.run_clustering_batch_task = lambda *a: seen.append(a) or {"status": "ORIGINAL"}
    fn = clustering_batch.make_run_clustering_batch_task(env.task, env.helper)
    assert fn(*batch_args(env, method="gmm")) == {"status": "ORIGINAL"}
    env.helper.USE_GPU_CLUSTERING = False
    assert fn(*batch_args(env)) == {"status": "ORIGINAL"}
    env.helper.USE_GPU_CLUSTERING, env.helper.GPU_CLUSTERING_AVAILABLE = True, False
    assert fn(*batch_args(env)) == {"status": "ORIGINAL"}
    assert len(seen) == 3 and seen[0] == batch_args(env, method="gmm")


def test_apply_needs_clustering(monkeypatch):
    env = Env()
    with pytest.raises(ValueError, match="clustering="):
        integration.apply(clustering_batch=env.task, allow_sklearn_fallback=False)
    helper_mod = types.ModuleType("fake_clustering_helper_" + uuid.uuid4().hex)
    monkeypatch.setitem(sys.modules, helper_mod.__name__, helper_mod)

    def perform():
        pass

    perform.__module__ = helper_mod.__name__
    env.task._perform_single_clustering_iteration = perform
    integration.apply(clustering_batch=env.task, clustering=types.SimpleNamespace(), allow_sklearn_fallback=False)
    assert env.task.run_clustering_batch_task.__module__ == clustering_batch.__name__
