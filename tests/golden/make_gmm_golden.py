#!/usr/bin/env python
"""Golden record of the clustering task's Gaussian mixture as the reference runs it.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_gmm_golden.py
    # writes tests/golden/gmm_golden.npz

Runs, UNMODIFIED and on the CPU:
  - tasks.clustering_gpu.get_clustering_model('gmm', params, use_gpu=True): the class it hands out and the arguments
    it gives scikit-learn's GaussianMixture (clustering_gpu.py:284-309, 385-392);
  - tasks.clustering_helper._apply_clustering_model (:261-335) after np.random.seed(SEED) (the reference passes
    random_state=None, so numpy's global generator drives k-means++) on seeded, StandardScaler-ed track features
    (600 x 13, 6 groups): the labels and the centres it returns (the model's means_).
tests/test_gmm_host.py and tests/test_gpu_gmm.py replay the record.
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from tests import ref_harness as rh  # noqa: E402
from make_cluster_metrics_golden import load_clustering_helper  # noqa: E402

PARAMS = {"n_components": 6}
SEED = 2468
CTOR = ("n_components", "covariance_type", "init_params", "n_init", "random_state", "reg_covar")


def features(n=600, k=6, seed=33):
    """track features in [0, 1] around k well separated centres"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(0.1, 0.9, (k, 13))
    lab = np.arange(n) % k
    return np.clip(centres[lab] + 0.04 * rng.standard_normal((n, 13)), 0.0, 1.0)


def main():
    from sklearn.preprocessing import StandardScaler
    assert rh.available(), "set AUDIOMUSE_REFERENCE to a checkout of the reference"
    ch = load_clustering_helper()
    spec = importlib.util.spec_from_file_location("tasks.clustering_gpu", os.path.join(rh.REF, "tasks", "clustering_gpu.py"))
    ref_cg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_cg)
    model = ref_cg.get_clustering_model("gmm", dict(PARAMS), use_gpu=True)
    sk_params = model.model.get_params()
    data = StandardScaler().fit_transform(features())
    np.random.seed(SEED)
    labels, centers, fitted = ch._apply_clustering_model(data, {"method": "gmm", "params": dict(PARAMS)}, "[golden]", 0)
    assert type(fitted).__name__ == "GaussianMixture"
    keys = sorted(centers)
    assert keys == list(range(PARAMS["n_components"]))
    out = {"class_name": np.array(type(model).__name__),
           "ctor_names": np.array(CTOR),
           "ctor_values": np.array([repr(sk_params[n]) for n in CTOR]),
           "n_components": np.int64(PARAMS["n_components"]), "seed": np.int64(SEED),
           "X": data, "labels": np.asarray(labels, dtype=np.int64), "centers": np.stack([centers[c] for c in keys])}
    print(out["class_name"], dict(zip(CTOR, out["ctor_values"])), np.bincount(out["labels"]))
    path = os.path.join(HERE, "gmm_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
