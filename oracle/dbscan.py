"""Oracle: exact DBSCAN on float32 input.  TEST INFRASTRUCTURE ONLY.

Restates what ``tasks/clustering_gpu.py:151-199`` asks of GPUDBSCAN: the labels of
sklearn.cluster.DBSCAN (the reference's CPU branch, ``tasks/clustering_helper.py:295``)
on the same points.  The decision rule is written out here instead of borrowed from
scikit-learn, so that a disagreement points at one side:

  * neighbours: the squared distance of two float32 rows, formed from float64
    differences of their coordinates and summed in float64, is ``<= eps * eps`` in
    float64 (eps itself is a Python float, as the reference draws it:
    ``round(uniform(0.1, 0.5), 2)``, clustering_helper.py:196).  Every point is its
    own neighbour;
  * a point is core when it has at least ``min_samples`` neighbours, itself included;
  * clusters grow by scikit-learn's index-ordered depth-first expansion: the lowest
    unlabelled core index starts the next cluster, so clusters are numbered by their
    lowest core index, and a border point joins the first cluster that reaches it --
    the one with the smallest label among its core neighbours.  Noise is -1.

Neighbourhoods come from chunked float64 brute force (a Gram-matrix prefilter with a
generous margin, then the exact differences for every candidate pair), or, for more
than 10 000 rows in at most 16 dimensions, from scipy's cKDTree with a slightly
inflated radius and the same exact recheck.  The case generators at the bottom build
the inputs of tests/test_gpu_cluster_extra_exact.py; tests/test_cluster_extra_host.py
checks that each has the property it is meant to test.
"""
from __future__ import annotations

import numpy as np


# ---------------------------------------------------------------- the oracle
def sq_dist(a, b):
    """exact-as-float64 squared distance between float32 rows a [.., d] and b [.., d]"""
    t = np.asarray(a, np.float32).astype(np.float64) - np.asarray(b, np.float32).astype(np.float64)
    return (t * t).sum(-1)


def neighbourhoods(X, eps):
    """-> (indptr i64[N + 1], indices i64[nnz]): the eps-neighbourhood of every row (itself included), ascending"""
    X = np.asarray(X, np.float32)
    N, d = X.shape
    X64 = X.astype(np.float64)
    eps2 = float(eps) * float(eps)
    rows, cols = [], []
    if N > 10_000 and d <= 16:
        from scipy.spatial import cKDTree
        pairs = cKDTree(X64).query_pairs(float(eps) * (1 + 1e-6) + 1e-300, output_type="ndarray")
        keep = sq_dist(X[pairs[:, 0]], X[pairs[:, 1]]) <= eps2
        p = pairs[keep]
        rows += [p[:, 0], p[:, 1], np.arange(N)]
        cols += [p[:, 1], p[:, 0], np.arange(N)]
    else:
        nx = (X64 * X64).sum(1)
        chunk = max(1, (1 << 23) // N)
        for r0 in range(0, N, chunk):
            r1 = min(N, r0 + chunk)
            g = nx[r0:r1, None] + nx[None, :] - 2.0 * (X64[r0:r1] @ X64.T)
            # the Gram form is off by at most ~ (d + 2) 2^-53 (|x|^2 + |y|^2): 1e-9 of that is far more than enough
            r, c = np.nonzero(g <= eps2 * (1 + 1e-9) + 1e-9 * (nx[r0:r1, None] + nx[None, :]))
            r = r + r0
            keep = sq_dist(X[r], X[c]) <= eps2
            rows.append(r[keep])
            cols.append(c[keep])
    r = np.concatenate(rows)
    c = np.concatenate(cols)
    order = np.lexsort((c, r))
    r, c = r[order], c[order]
    indptr = np.zeros(N + 1, np.int64)
    np.cumsum(np.bincount(r, minlength=N), out=indptr[1:])
    return indptr, c.astype(np.int64)


def expand(indptr, indices, min_samples):
    """scikit-learn's index-ordered depth-first expansion over given neighbourhoods -> (labels i32[N], n_clusters)"""
    N = len(indptr) - 1
    core = np.diff(indptr) >= min_samples
    labels = np.full(N, -1, np.int32)
    n = 0
    for i0 in range(N):
        if labels[i0] != -1 or not core[i0]:
            continue
        stack = [i0]
        labels[i0] = n
        while stack:
            i = stack.pop()
            if not core[i]:
                continue
            for j in indices[indptr[i]:indptr[i + 1]]:
                if labels[j] == -1:
                    labels[j] = n
                    stack.append(j)
        n += 1
    return labels, n


def dbscan(X, eps, min_samples):
    """-> (labels i32[N], n_clusters)"""
    indptr, indices = neighbourhoods(X, eps)
    return expand(indptr, indices, min_samples)


# ---------------------------------------------------------------- generated cases
RAGGED_N = (1, 2, 31, 32, 33, 63, 64, 65, 129)      # around the 32-bit word and the 64-row tile
RAGGED_D = (1, 3, 31, 33, 513)                      # around the 32-wide k-slab


def ragged(n, d, seed=0):
    """three blobs and a few uniform points; eps halfway between two neighbouring pair distances near the 20th percentile
    (so no pair is close to it), min_samples 3 -> (X, eps, min_samples)"""
    rng = np.random.default_rng(1000 * n + d + seed)
    centres = rng.standard_normal((3, d)) * 2.0
    x = centres[rng.integers(0, 3, n)] + 0.4 * rng.standard_normal((n, d))
    m = rng.random(n) < 0.1
    x[m] = rng.uniform(-4, 4, (int(m.sum()), d))
    x = x.astype(np.float32)
    if n == 1:
        return x, 0.5, 1
    s = np.sqrt(np.unique(sq_dist(x[:, None, :], x[None, :, :])[np.triu_indices(n, 1)]))
    q = min(len(s) - 2, int(0.2 * len(s))) if len(s) > 1 else 0
    eps = float(0.5 * (s[q] + s[q + 1])) if len(s) > 1 else float(s[0] * 1.5 + 0.1)
    return x, eps, 3


def degenerate():
    """-> [(name, X, eps, min_samples)]: every point core, every point noise, identical rows, blocks of duplicates"""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((100, 5)).astype(np.float32)
    same = np.tile(rng.standard_normal((1, 3)).astype(np.float32), (70, 1))
    blocks = np.repeat(rng.uniform(-20, 20, (12, 4)).astype(np.float32), np.arange(1, 13), axis=0)   # sizes 1 .. 12
    blocks = blocks[rng.permutation(len(blocks))]
    return [
        ("min_samples_1", x, 1.1, 1),
        ("min_samples_above_n", x, 1.1, 101),
        ("identical_rows", same, 0.05, 5),
        ("identical_rows_all_noise", same, 0.05, 71),
        ("duplicate_blocks", blocks, 0.5, 6),
    ]


def probe(d, k, sign, seed=0):
    """a blob of 4 identical core rows and one probe at squared distance eps^2 (1 + sign 2^-k)^2 from it; eps is derived
    from the float32 rows, so the margin is what it says up to float64 rounding.  min_samples 4: the probe joins the
    blob's cluster exactly when it is inside -> (X, eps, min_samples, inside)"""
    rng = np.random.default_rng(d * 100 + k)
    c = rng.standard_normal(d).astype(np.float32)
    u = rng.standard_normal(d)
    p = (c + 0.37 * u / np.linalg.norm(u)).astype(np.float32)
    far = (c + 50.0).astype(np.float32)                       # an unrelated noise row after the blob
    x = np.stack([c, c, far, c, p, c]).astype(np.float32)
    eps = float(np.sqrt(sq_dist(p, c))) / (1.0 + sign * 2.0 ** -k)
    return x, eps, 4, sign < 0


def lattice(dim, side):
    """every point of a dim-dimensional grid of spacing float32(0.1), coordinates i * float32(0.1) rounded to float32"""
    g = np.arange(side, dtype=np.float32) * np.float32(0.1)
    return np.stack(np.meshgrid(*([g] * dim), indexing="ij"), -1).reshape(-1, dim).astype(np.float32)


# (dim, side, eps, min_samples): eps 0.1 / 0.2 / 0.3 are the values whose float32 square differs from the float64 one on
# lattice pairs; min_samples is set where that difference changes which points are core.  0.23 and 0.5 are controls.
LATTICE_CASES = [
    (2, 20, 0.10, 3), (2, 20, 0.20, 12), (2, 20, 0.30, 28), (2, 20, 0.23, 9), (2, 20, 0.50, 20),
    (3, 10, 0.10, 3), (3, 10, 0.20, 31), (3, 10, 0.30, 109), (3, 10, 0.23, 27), (3, 10, 0.50, 60),
]


def border_between_clusters():
    """cluster A (indices 0-4) and cluster B (5-9) on a line; row 10 is a border point within eps of one core row of each,
    nearer to B's.  scikit-learn gives it A's label 0, the first cluster to reach it -> (X, eps, min_samples, labels)"""
    xs = [0.0, 0.1, 0.2, 0.3, 0.4, 2.27, 2.37, 2.47, 2.57, 2.67, 1.35]
    x = np.zeros((len(xs), 2), np.float32)
    x[:, 0] = xs
    x[:, 1] = 0.25
    return x, 1.0, 4, np.array([0] * 5 + [1] * 5 + [0], np.int32)


def chain(n, order, seed=0):
    """n points 0.5 apart on a line, eps 0.6, min_samples 3: one cluster whose two ends are border points.  order:
    'random', 'ascending' or 'descending' index order along the line -> (X, eps, min_samples)"""
    x = np.zeros((n, 2), np.float32)
    x[:, 0] = np.arange(n, dtype=np.float32) * np.float32(0.5)
    if order == "random":
        x = x[np.random.default_rng(seed).permutation(n)]
    elif order == "descending":
        x = x[::-1].copy()
    return x, 0.6, 3


def band(length, seed=0):
    """a 3 x length grid of spacing 0.5 in random index order, eps 0.6 (axis neighbours only), min_samples 3: one
    cluster -> (X, eps, min_samples)"""
    g = np.stack(np.meshgrid(np.arange(length), np.arange(3), indexing="ij"), -1).reshape(-1, 2)
    x = (g * 0.5).astype(np.float32)
    return x[np.random.default_rng(seed).permutation(len(x))], 0.6, 3


def task_blobs(n, d, seed=0):
    """StandardScaled blobs with scattered points, shaped like the clustering task's input (PCA-reduced or raw
    embeddings scaled to unit variance): tight blobs so that eps on the reference's 0.1-0.5 grid finds clusters"""
    rng = np.random.default_rng(seed + 7 * d)
    k = max(2, n // 100)
    centres = rng.standard_normal((k, d))
    spread = 0.12 / np.sqrt(d) * rng.uniform(0.5, 1.5, k)
    lab = rng.integers(0, k, n)
    x = centres[lab] + spread[lab, None] * rng.standard_normal((n, d))
    m = rng.random(n) < 0.05
    x[m] = rng.standard_normal((int(m.sum()), d))
    x = (x - x.mean(0)) / x.std(0)
    return x.astype(np.float32)


TASK_CASES = [(8, 0.12, 5), (8, 0.27, 20), (58, 0.19, 5), (58, 0.25, 20)]   # (d, eps, min_samples), N = 20 003
