"""Spectral clustering on the GPU (csrc/spectral.cu + clustering_gpu.GPUSpectralClustering) at clustering-task sizes,
next to scikit-learn's SpectralClustering on the box's CPU cores.  One JSON line.
    python tools/spectral_bench.py [--sklearn-max-n 20000]

Per (N, d), n_clusters = 60, n_neighbors = 20, n_init = 10 (the reference's SpectralClustering arguments,
tasks/clustering_gpu.py:312-335): d = 13 is a StandardScaler-ed mixture of 60 overlapping Gaussian groups (a connected
k-NN graph, closely packed eigenvalues); d = 200 is 60 well separated blobs (60 components).
  stages: k-NN lists and CSR build (CUDA events inside am_spectral_plan_create), the eigensolver (host clock around
          the outer iterations, every one of which ends in a device synchronise; outer iterations and SpMM count),
          k-means on the embedding (host clock around am_kmeans_fit);
  spmm:   device time of cheb_spmm_kernel (am_profile_enable, a separate run) and its algorithmic bytes per SpMM,
          nnz * 12 (i32 index + f64 value) + nnz * ld * 8 (gathered rows) + 3 * N * ld * 8 (own row, previous
          iterate, output), ld = the block width rounded up to 32;
  host-API total: GPUSpectralClustering.fit_predict, median of 3 after a warm-up;
  scikit-learn: one SpectralClustering.fit_predict with the same arguments for N <= --sklearn-max-n, and the ARI
          between the two labellings.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from audiomuse_ai_b200 import _lib, clustering_gpu as cg  # noqa: E402
from cluster_metrics_bench import card  # noqa: E402

K, NN = 60, 20


def data(n, d, seed):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, K, n)
    if d == 13:
        from sklearn.preprocessing import StandardScaler
        c = rng.standard_normal((K, d))
        return StandardScaler().fit_transform(c[lab] + rng.standard_normal((n, d))).astype(np.float32)
    c = rng.standard_normal((K, d)) * 10.0
    return (c[lab] + rng.standard_normal((n, d))).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sklearn-max-n", type=int, default=20_000)
    args = ap.parse_args()
    out = {"metric": "spectral_clustering", **card(), "cpu_cores": os.cpu_count(), "n_clusters": K, "n_neighbors": NN,
           "runs": []}
    cg.GPUSpectralClustering(n_clusters=4, n_neighbors=NN, random_state=0).fit_predict(data(2000, 13, 1))  # warm-up
    for n, d in ((5_000, 13), (5_000, 200), (20_000, 13), (20_000, 200), (100_000, 13), (100_000, 200)):
        x = data(n, d, n + d)
        det = {}
        emb, ev = cg.spectral_embedding(x, K, n_neighbors=NN, seed=1, details=det)
        t0 = time.perf_counter()
        _, labels, _, _ = cg.kmeans_fit(emb.astype(np.float32), K, n_init=10, seed=1)
        km_ms = 1e3 * (time.perf_counter() - t0)
        _lib.profile_enable(True)
        _lib.profile_report()
        cg.spectral_embedding(x, K, n_neighbors=NN, seed=1)
        prof = _lib.profile_report()
        _lib.profile_enable(False)
        m = cg.GPUSpectralClustering(n_clusters=K, n_neighbors=NN, random_state=1)
        m.fit_predict(x)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got = m.fit_predict(x)
            ts.append(time.perf_counter() - t0)
        ld = -(-det["block"] // 32) * 32
        nnz = det["nnz"]
        spmm = next((v for k, v in prof.items() if k.endswith("cheb_spmm_kernel")), {"ms": float("nan"), "count": 0})
        spmm_ms = spmm["ms"] / max(1, spmm["count"])
        spmm_bytes = nnz * 12 + nnz * ld * 8 + 3 * n * ld * 8
        run = {"n": n, "d": d, "block": det["block"], "nnz": nnz, "knn_ms": round(det["knn_ms"], 2),
               "csr_ms": round(det["graph_ms"], 2), "eigensolver_ms": round(det["eigensolver_ms"], 1),
               "outer_iterations": det["outer_iterations"], "n_spmm": det["n_spmm"], "kmeans_ms": round(km_ms, 1),
               "spmm_ms": round(spmm_ms, 4), "spmm_bytes": spmm_bytes,
               "spmm_gb_per_s": round(spmm_bytes / (spmm_ms * 1e-3) / 1e9, 1),
               "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items()},
               "host_api_s": round(float(np.median(ts)), 4), "lambda_max": float(ev[-1]),
               "max_residual": float(det["residuals"].max())}
        if n <= args.sklearn_max_n:
            from sklearn.cluster import SpectralClustering
            from sklearn.metrics import adjusted_rand_score
            t0 = time.perf_counter()
            ref = SpectralClustering(n_clusters=K, affinity="nearest_neighbors", n_neighbors=NN, random_state=1,
                                     n_init=10).fit_predict(x)
            run["sklearn_s"] = round(time.perf_counter() - t0, 2)
            run["ari_vs_sklearn"] = round(float(adjusted_rand_score(ref, got)), 4)
        else:
            run["sklearn_s"] = "not measured"
        out["runs"].append(run)
        print(json.dumps(run), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
