#!/usr/bin/env python
"""Golden record of the clustering task's fitness scoring as the reference computes it.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_cluster_metrics_golden.py
    # writes tests/golden/cluster_metrics_golden.npz

Runs, UNMODIFIED and on the CPU, tasks.clustering_helper._apply_clustering_model and _format_and_score_iteration_result
(:261-590) with all three score weights on, for a k-means labelling and a DBSCAN labelling with noise, on seeded
StandardScaler-ed track features (600 x 13).  The module's silhouette_score / davies_bouldin_score /
calinski_harabasz_score are wrapped so that the (X, labels) the reference passes and scikit-learn's returns are
recorded, together with the resulting fitness_score and the names the module defines (integration.apply replaces three
of them).  tests/test_cluster_metrics_host.py and tests/test_gpu_cluster_metrics.py replay the record.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import ref_harness as rh  # noqa: E402

METRICS = ("silhouette_score", "davies_bouldin_score", "calinski_harabasz_score")
WEIGHTS = {"mood_diversity": 2.0, "mood_purity": 1.0, "other_feature_diversity": 0.0, "other_feature_purity": 0.0,
           "silhouette": 0.6, "davies_bouldin": 0.3, "calinski_harabasz": 0.4}
CASES = {"kmeans": {"method": "kmeans", "params": {"n_clusters": 8}},
         "dbscan": {"method": "dbscan", "params": {"eps": 1.1, "min_samples": 5}}}


def load_clustering_helper():
    """tasks.clustering_helper with inert stand-ins for the packages it imports but scoring never uses."""
    if rh.REF not in sys.path:
        sys.path.insert(0, rh.REF)
    for k in [k for k in sys.modules if k == "tasks" or k.startswith("tasks.") or k == "config"]:
        del sys.modules[k]
    rh._stub("psycopg2", extras=None, OperationalError=Exception)
    rh._stub("psycopg2.extras", DictCursor=object)
    sys.modules["psycopg2"].extras = sys.modules["psycopg2.extras"]
    rh._stub("rq")
    rh._stub("rq.job", Job=object)
    rh._stub("rq.exceptions", NoSuchJobError=Exception)
    tasks_pkg = rh._stub("tasks")
    tasks_pkg.__path__ = [os.path.join(rh.REF, "tasks")]
    import config  # noqa: F401  (the reference's config.py: environment defaults only)
    return rh._load("tasks.clustering_helper", "tasks/clustering_helper.py")


def features(n=600, k=8, seed=11):
    """track features laid out as score_vector makes them: tempo, energy, 5 moods, 6 other features, all in [0, 1]"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(0.1, 0.9, (k, 13))
    lab = rng.integers(0, k, n)
    x = np.clip(centres[lab] + 0.05 * rng.standard_normal((n, 13)), 0.0, 1.0)
    m = rng.random(n) < 0.04                                   # a few scattered tracks: DBSCAN noise
    x[m] = rng.uniform(0.0, 1.0, (int(m.sum()), 13))
    return x


def main():
    from sklearn.preprocessing import StandardScaler
    assert rh.available(), "set AUDIOMUSE_REFERENCE to a checkout of the reference"
    ch = load_clustering_helper()
    import config
    active_moods = list(config.MOOD_LABELS[:5])
    x_feat = features()
    scores = rh.make_score_table(len(x_feat), seed=4)
    tracks = [scores[f"item{i}"] for i in range(len(x_feat))]
    scaler = StandardScaler()
    data = scaler.fit_transform(x_feat)
    out = {"helper_names": np.array(sorted(n for n in vars(ch) if not n.startswith("__") and callable(getattr(ch, n)))),
           "weight_names": np.array(sorted(WEIGHTS)), "weights": np.array([WEIGHTS[k] for k in sorted(WEIGHTS)])}
    originals = {n: getattr(ch, n) for n in METRICS}
    np.random.seed(5)                                           # KMeans(random_state=None) draws from numpy's global state
    for case, method_config in CASES.items():
        calls = []

        def recording(name):
            def f(X, labels):
                v = originals[name](X, labels)
                calls.append((name, np.array(X, copy=True), np.array(labels, copy=True), float(v)))
                return v
            return f

        for n in METRICS:
            setattr(ch, n, recording(n))
        labels, centers, model = ch._apply_clustering_model(data, method_config, "[golden]", 0)
        params = {"pca_config": {"enabled": False, "components": 0}, "clustering_method_config": method_config}
        res = ch._format_and_score_iteration_result(labels, tracks, x_feat, data, centers, model, None, scaler,
                                                    active_moods, params, 40, 0, False, WEIGHTS, "[golden]")
        assert [c[0] for c in calls] == list(METRICS), f"{case}: the reference scored {[c[0] for c in calls]}"
        X0, l0 = calls[0][1], calls[0][2]
        assert all(np.array_equal(c[1], X0) and np.array_equal(c[2], l0) for c in calls)
        if case == "dbscan":
            assert (l0 == -1).sum() > 0 and len(set(l0.tolist()) - {-1}) >= 2, "the DBSCAN case needs clusters and noise"
        out[f"{case}_X"] = X0
        out[f"{case}_labels"] = l0
        for name, _, _, v in calls:
            out[f"{case}_{name}"] = np.float64(v)
        out[f"{case}_fitness"] = np.float64(res["fitness_score"])
        print(case, {name: v for name, _, _, v in calls}, "fitness", res["fitness_score"])
    for n in METRICS:
        setattr(ch, n, originals[n])
    path = os.path.join(HERE, "cluster_metrics_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
