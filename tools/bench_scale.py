#!/usr/bin/env python
"""Scale cases of SURVEY.md section 8(d) that bench.py's single JSON line does not carry (GPU box only):

  config 3  k-NN over 100 k x 512: QPS at query batches 1 / 32 / 256 / 4096 for k = 50, k = 500 at batch 256,
            one k = N full scan, and the exact-id match rate against the float64 oracle
  config 4  k-means, 1 M x 512, k = 128, n_init = 1: time, iterations, inertia; parity on a 100 k subsample
            from identical initial centres against sklearn (inertia ratio, adjusted Rand index)
  config 5  query mix over a 1 M x 512 library through the voyager-compatible Index (host API, single queries
            like the reference's callers): 50 % Sonic-Fingerprint style (mean of 20 rows, k = 400), 50 % Song-Path
            style (get_vector + k cycling 101 / 10 / 30 / 100 / 300 / 1000): p50 / p99 latency, queries/s;
            and the same mix in batches of 256

Prints ONE JSON object; `python tools/bench_scale.py > scale.json`.  The oracle is used here only
as the checker of ids / inertia, never as the thing measured.
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import audiomuse_ai_b200 as am  # noqa: E402,F401
from audiomuse_ai_b200 import clustering_gpu as cg, corpus, voyager_compat as vc  # noqa: E402
from oracle import knn as oknn  # noqa: E402


def timed(fn, reps):
    t0 = time.perf_counter()
    for r in range(reps):
        fn(r)
    return (time.perf_counter() - t0) / reps


def config3():
    x = corpus.knn_library(100_000, 512, 1234)
    q = corpus.knn_queries(x, 10_000, 1_000, 4321)
    idx = vc.Index(vc.Space.Cosine, num_dimensions=512, M=64, ef_construction=1024)
    idx.add_items(x)
    idx.query(q[:4096], 50)
    out = {"library": "100000 x 512 f32 unit rows; queries: 10000 near (row + 0.3 noise) + 1000 random"}
    for nq, reps in ((1, 200), (32, 50), (256, 20), (4096, 5)):
        dt = timed(lambda r: idx.query(q[(r * nq) % 4096:(r * nq) % 4096 + nq] if nq > 1 else q[r], 50), reps)
        out[f"qps_k50_batch{nq}"] = nq / dt
    idx.query(q[:256], 500)
    out["qps_k500_batch256"] = 256 / timed(lambda r: idx.query(q[r * 256:(r + 1) * 256], 500), 10)
    idx.query(q[0], len(idx))
    out["full_scan_k_eq_N_ms"] = 1e3 * timed(lambda r: idx.query(q[r], len(idx)), 3)
    # exact ids vs the float64 oracle: the first 32 near + the last 32 random queries
    sample = np.concatenate([q[:32], q[-32:]], 0)
    ids, dist = idx.query(sample, 50)
    want_ids, want_dist = oknn.topk(x, sample, 50)
    out["id_match_rate_vs_f64_oracle"] = float(np.mean(np.asarray(ids, dtype=np.int64) == np.asarray(want_ids)))
    out["max_abs_distance_error"] = float(np.max(np.abs(np.asarray(dist, np.float64) - np.asarray(want_dist))))
    return out


def config4():
    from sklearn.cluster import KMeans
    from sklearn.metrics import adjusted_rand_score
    t0 = time.perf_counter()
    x, lab, centers = corpus.kmeans_library(1_000_000, 512, 128, 7)
    gen_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    c, labels, inertia, n_iter = cg.kmeans_fit(x, 128, n_init=1, max_iter=300, tol=1e-4, seed=0)
    fit_s = time.perf_counter() - t0
    out = {"shape": [1_000_000, 512], "k": 128, "n_init": 1, "fit_seconds_incl_h2d": fit_s, "iterations": n_iter,
           "inertia": inertia, "ari_vs_generating_labels": float(adjusted_rand_score(lab[:200_000], labels[:200_000])),
           "host_generation_seconds": gen_s}
    # parity on a 100 k subsample from identical initial centres
    sub = x[:100_000]
    init = sub[np.random.default_rng(3).choice(100_000, 128, replace=False)].copy()
    t0 = time.perf_counter()
    c_g, l_g, in_g, it_g = cg.kmeans_fit(sub, 128, n_init=1, max_iter=300, tol=1e-4, seed=0, init_centers=init)
    out["subsample_fit_seconds"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    km = KMeans(n_clusters=128, init=init, n_init=1, max_iter=300, tol=1e-4, algorithm="lloyd").fit(sub.astype(np.float64))
    out["subsample_sklearn_seconds"] = time.perf_counter() - t0
    out["subsample_inertia_ratio_vs_sklearn"] = float(in_g / km.inertia_)
    out["subsample_ari_vs_sklearn"] = float(adjusted_rand_score(km.labels_, l_g))
    out["subsample_iterations"] = [int(it_g), int(km.n_iter_)]
    return out, x


def config5(x):
    rng = np.random.default_rng(99)
    n = x.shape[0]
    idx = vc.Index(vc.Space.Cosine, num_dimensions=512, M=64, ef_construction=1024)
    t0 = time.perf_counter()
    idx.add_items(x)
    idx.query(x[0], 10)
    build_s = time.perf_counter() - t0
    tasks = []  # (vector or row id, k)
    for i in range(5000):  # Sonic-Fingerprint style: weighted mean of 20 library rows, k = 5 n with n = 80
        rows = rng.integers(0, n, 20)
        w = rng.random(20).astype(np.float32) + 0.1
        v = (x[rows] * w[:, None]).sum(0)
        tasks.append((v / np.linalg.norm(v), 400))
    ks = (101, 10, 30, 100, 300, 1000)
    for p in range(200):  # Song-Path style: 2 by-id queries, then 23 centroid queries along a SLERP-like path
        a, b = rng.integers(0, n, 2)
        tasks.append((int(a), 101))
        tasks.append((int(b), 101))
        for s in range(23):
            t = (s + 1) / 24.0
            v = (1 - t) * x[a] + t * x[b]
            tasks.append((v / np.linalg.norm(v), ks[s % len(ks)]))
    order = rng.permutation(len(tasks))
    lat = []
    t_all = time.perf_counter()
    for i in order:
        v, k = tasks[i]
        t0 = time.perf_counter()
        if isinstance(v, int):
            v = idx.get_vector(v)
        idx.query(v, k)
        lat.append(time.perf_counter() - t0)
    total = time.perf_counter() - t_all
    lat = np.sort(np.asarray(lat))
    out = {"library": [int(n), 512], "index_build_seconds_incl_h2d": build_s, "queries": len(tasks),
           "single_query_qps": len(tasks) / total, "latency_ms_p50": 1e3 * float(lat[len(lat) // 2]),
           "latency_ms_p99": 1e3 * float(lat[int(len(lat) * 0.99)])}
    # the same mix in batches of 256 per k
    by_k = {}
    for v, k in tasks:
        by_k.setdefault(k, []).append(idx.get_vector(v) if isinstance(v, int) else v)
    t0 = time.perf_counter()
    for k, vs in by_k.items():
        vs = np.stack(vs).astype(np.float32)
        for b0 in range(0, len(vs), 256):
            idx.query(vs[b0:b0 + 256], k)
    out["batched_256_qps"] = len(tasks) / (time.perf_counter() - t0)
    return out


def main():
    res = {"config3_knn_100k": config3()}
    c4, x = config4()
    res["config4_kmeans_1M"] = c4
    res["config5_query_mix_1M"] = config5(x)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
