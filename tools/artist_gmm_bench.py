"""Times the artist-similarity GMM sweep (audiomuse_ai_b200.artist_gmm) on a seeded library of 100 000 x 200 tracks
over about 8 000 artists with Pareto-distributed sizes: the whole library in one fit_artist_gmms batch (device ms of
the fit and selection phases from CUDA events, and wall time with the copies), fit_artist_gmm called once per artist
as build_and_store_artist_index calls it (on a seeded sample of artists, scaled to the library), and scikit-learn's
sweep on a smaller sample (scaled likewise; both scaled figures are labelled extrapolated).  Also the EM flops and row
bytes the batch needs, counted from the shapes and the iteration counts it returned.  Prints one JSON object; needs a
CUDA device.

    python tools/artist_gmm_bench.py [--tracks 100000] [--artists 8000] [--loop-sample 400] [--sklearn-sample 40]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def library(tracks, artists, d=200, seed=0):
    rng = np.random.default_rng(seed)
    w = rng.pareto(1.1, artists) + 1.0
    sizes = np.maximum(1, np.round(w / w.sum() * tracks)).astype(int)
    sizes[np.argmax(sizes)] += tracks - sizes.sum()
    out = []
    for n in sizes:
        g = 1 + int(rng.integers(0, 5))
        c = rng.standard_normal((g, d))
        out.append((c[rng.integers(0, g, n)] + rng.uniform(0.3, 1.2) * rng.standard_normal((n, d))).astype(np.float32))
    return out


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=100000)
    ap.add_argument("--artists", type=int, default=8000)
    ap.add_argument("--loop-sample", type=int, default=400)
    ap.add_argument("--sklearn-sample", type=int, default=40)
    a = ap.parse_args()
    from audiomuse_ai_b200 import artist_gmm as ag

    lib = library(a.tracks, a.artists)
    d = lib[0].shape[1]
    ag.fit_artist_gmms([lib[0]])                                  # context and module load
    timings = {}
    t = time.perf_counter()
    fits = ag.fit_artist_gmms(lib, timings=timings)
    wall = time.perf_counter() - t

    em_flops = rows_bytes = 0.0
    for X, f in zip(lib, fits):
        n = len(X)
        for K in range(f.k_range[0], f.k_range[1] + 1):
            if f.failed.get(K, True):
                continue
            iters = f.n_iter[K - 1].astype(np.float64)
            passes = 2 * iters + 1                     # an E and an M pass per iteration, then the score
            em_flops += float((4.0 * n * d * K * passes).sum())
            rows_bytes += float((4.0 * n * d * passes).sum())

    rng = np.random.default_rng(1)
    sample = rng.choice(len(lib), min(a.loop_sample, len(lib)), replace=False)
    t = time.perf_counter()
    for i in sample:
        ag.fit_artist_gmm(f"artist {i}", list(lib[i]))
    loop_s = (time.perf_counter() - t) * len(lib) / len(sample)

    from sklearn.mixture import GaussianMixture
    warnings.filterwarnings("ignore")
    sk_sample = rng.choice(len(lib), min(a.sklearn_sample, len(lib)), replace=False)
    t = time.perf_counter()
    for i in sk_sample:
        X = lib[i]
        if len(X) < 5:
            continue
        for K in range(1, ag.max_feasible(len(X)) + 1):
            GaussianMixture(K, covariance_type="diag", max_iter=100, n_init=3, random_state=42).fit(X).bic(X)
    sk_s = (time.perf_counter() - t) * len(lib) / len(sk_sample)

    sizes = np.array([len(X) for X in lib])
    print(json.dumps({
        "gpu": gpu_info(),
        "library": {"tracks": int(sizes.sum()), "artists": len(lib), "d": d, "largest_artist": int(sizes.max()),
                    "artists_fitted": int((sizes >= 5).sum())},
        "batch_device_ms": {"fit": round(timings["fit_ms"], 2), "select": round(timings["select_ms"], 3)},
        "batch_wall_s": round(wall, 3),
        "per_artist_loop_s_extrapolated": round(loop_s, 2), "per_artist_loop_sample": len(sample),
        "sklearn_sweep_s_extrapolated": round(sk_s, 1), "sklearn_sample": len(sk_sample),
        "em_gflop": round(em_flops / 1e9, 2), "em_row_gbytes": round(rows_bytes / 1e9, 2),
        "em_gflops_per_s": round(em_flops / 1e6 / timings["fit_ms"], 1),
    }))


if __name__ == "__main__":
    main()
