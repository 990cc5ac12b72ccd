"""Quality floor of the GPU UMAP (tests/test_gpu_umap.py): the sequential oracle (oracle/umap.py: umap's
single-threaded SGD order over the float64 restatement of its graph and spectral initialisation) on seeded datasets,
seeds 0-4, scored by trustworthiness@15, 2-D k-NN recall@15 and, where there are labels, the 2-D silhouette of the
true labels.  Runs on the CPU:

    python tests/golden/make_umap_golden.py      # -> tests/golden/umap_golden.json

The datasets are rebuilt from their seeds by the functions below; the GPU test imports them from here.
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SEEDS = (0, 1, 2, 3, 4)


def blobs(n=5000, d=200, k=60, seed=0):
    """k well-separated Gaussian blobs"""
    rng = np.random.default_rng(seed)
    lab = np.arange(n) % k
    c = rng.standard_normal((k, d)) * 6.0
    return (c[lab] + rng.standard_normal((n, d))).astype(np.float32), lab


def mixture(n=5000, d=13, k=30, seed=1):
    """k overlapping Gaussian groups, StandardScaler-ed"""
    from sklearn.preprocessing import StandardScaler
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((k, d)) * 1.5
    lab = rng.integers(0, k, n)
    return StandardScaler().fit_transform(c[lab] + rng.standard_normal((n, d))).astype(np.float32), lab


def curve(n=3000, d=200, seed=2):
    """a noisy closed curve (a trefoil-like loop) embedded in d dimensions by a random orthonormal map"""
    rng = np.random.default_rng(seed)
    t = np.sort(rng.uniform(0, 2 * np.pi, n))
    P = np.stack([np.sin(t) + 2 * np.sin(2 * t), np.cos(t) - 2 * np.cos(2 * t), -np.sin(3 * t)], 1)
    Q, _ = np.linalg.qr(rng.standard_normal((d, 3)))
    return (P @ Q.T * 5.0 + 0.05 * rng.standard_normal((n, d))).astype(np.float32), None


def mixture200(n, seed=3):
    """overlapping groups in 200 dimensions, for the row counts on either side of the 200 / 500 epoch switch"""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((40, 200)) * 0.6
    lab = rng.integers(0, 40, n)
    return (c[lab] + rng.standard_normal((n, 200))).astype(np.float32), lab


def clique(seed=4):
    """2000 mixture rows and 40 copies of one row far from all of them: the copies form a second component"""
    X, lab = mixture(2000, 13, 10, seed)
    far = np.full((40, 13), 50.0, np.float32)
    return np.concatenate([X, far]), np.concatenate([lab, np.full(40, 10)])


DATASETS = {
    "blobs": lambda: blobs(),
    "mixture": lambda: mixture(),
    "curve": lambda: curve(),
    "rows10000": lambda: mixture200(10000),
    "rows10001": lambda: mixture200(10001),
    "clique": lambda: clique(),
}


def main():
    sys.path.insert(0, ROOT)
    from oracle import umap as ou
    a, b = ou.find_ab_params()
    out = {"a": a, "b": b, "seeds": list(SEEDS), "sets": {}}
    for name, make in DATASETS.items():
        t0 = time.time()
        X, lab = make()
        g = ou.fuzzy_graph(X)
        vec_cache = {}

        def vectors(G, dim):            # the eigenvectors do not depend on the seed: solve each graph once
            key = (G.shape[0], G.nnz, float(G.data.sum()))
            if key not in vec_cache:
                vec_cache[key] = ou._laplacian_vectors(G, dim)
            return vec_cache[key]

        rows = []
        for seed in SEEDS:
            Y0 = ou.initial_layout(X, g["W"], np.random.default_rng(seed), vectors=vectors)
            Y = ou.sgd_sequential(Y0, g["W"], g["eps"], g["n_epochs"], a, b, seed).astype(np.float32)
            rows.append(ou.quality(X, Y, lab))
        out["sets"][name] = {"N": int(X.shape[0]), "d": int(X.shape[1]), "n_epochs": g["n_epochs"], "nnz": int(g["W"].nnz),
                             "scores": rows,
                             "min": {m: min(r[m] for r in rows) for m in rows[0]}}
        print(name, out["sets"][name]["min"], f"{time.time() - t0:.0f} s", flush=True)
    with open(os.path.join(ROOT, "tests", "golden", "umap_golden.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
