#!/usr/bin/env python
"""Golden record of the clustering task's Gaussian mixture for the covariance types other than 'full', as the
reference runs it.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_gmm_types_golden.py
    # writes tests/golden/gmm_types_golden.npz

A deployment picks the type with the environment variable GMM_COVARIANCE_TYPE, which the reference's config.py reads
when it is imported (config.py:140).  For each of 'diag', 'tied' and 'spherical' this script sets
os.environ["GMM_COVARIANCE_TYPE"] and then imports the reference's config, tasks.clustering_helper and
tasks.clustering_gpu afresh (load_clustering_helper drops the cached modules first), and runs, UNMODIFIED and on the
CPU:
  - tasks.clustering_gpu.get_clustering_model('gmm', params, use_gpu=True): the class it hands out and the arguments
    it gives scikit-learn's GaussianMixture (clustering_gpu.py:284-309, 385-392);
  - tasks.clustering_helper._apply_clustering_model (:261-335) after np.random.seed(SEED[type]) (random_state=None, so
    numpy's global generator drives k-means++) on seeded, StandardScaler-ed track features (600 x 13, 6 groups): the
    labels and the centres it returns (the model's means_).
Keys are prefixed with the type ("diag/labels", ...).  tests/test_gmm_covariance_types_host.py and
tests/test_gpu_gmm_covariance_types.py replay the record.
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
from make_gmm_golden import CTOR, PARAMS, features  # noqa: E402

TYPES = ("diag", "tied", "spherical")
SEED = {"diag": 1357, "tied": 2468, "spherical": 3579}


def record(cov_type, data):
    os.environ["GMM_COVARIANCE_TYPE"] = cov_type       # before the reference's config is imported, as a deployment does
    ch = load_clustering_helper()
    assert ch.GMM_COVARIANCE_TYPE == cov_type
    spec = importlib.util.spec_from_file_location("tasks.clustering_gpu", os.path.join(rh.REF, "tasks", "clustering_gpu.py"))
    ref_cg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_cg)
    model = ref_cg.get_clustering_model("gmm", dict(PARAMS), use_gpu=True)
    sk_params = model.model.get_params()
    assert sk_params["covariance_type"] == cov_type
    np.random.seed(SEED[cov_type])
    labels, centers, fitted = ch._apply_clustering_model(data, {"method": "gmm", "params": dict(PARAMS)}, "[golden]", 0)
    assert type(fitted).__name__ == "GaussianMixture" and fitted.covariance_type == cov_type
    keys = sorted(centers)
    assert keys == list(range(PARAMS["n_components"]))
    out = {"class_name": np.array(type(model).__name__),
           "ctor_names": np.array(CTOR),
           "ctor_values": np.array([repr(sk_params[n]) for n in CTOR]),
           "seed": np.int64(SEED[cov_type]),
           "labels": np.asarray(labels, dtype=np.int64), "centers": np.stack([centers[c] for c in keys])}
    print(cov_type, out["class_name"], dict(zip(CTOR, out["ctor_values"])), np.bincount(out["labels"]))
    return {f"{cov_type}/{k}": v for k, v in out.items()}


def main():
    from sklearn.preprocessing import StandardScaler
    assert rh.available(), "set AUDIOMUSE_REFERENCE to a checkout of the reference"
    data = StandardScaler().fit_transform(features())
    out = {"X": data, "n_components": np.int64(PARAMS["n_components"]), "types": np.array(TYPES),
           "how": np.array("os.environ['GMM_COVARIANCE_TYPE'] set before the reference's config is imported")}
    for t in TYPES:
        out.update(record(t, data))
    path = os.path.join(HERE, "gmm_types_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
