"""Oracle: Lloyd k-means.  TEST INFRASTRUCTURE ONLY.

Restates what ``tasks/clustering_gpu.py:96-148`` asks of its backends
(cuml.cluster.KMeans on GPU, sklearn.cluster.KMeans on CPU; both third-party):
``fit_predict(X) -> labels`` plus ``cluster_centers_``.  The reference has no numeric
test for it (test_clustering_helper.py patches USE_GPU_CLUSTERING False), so the bar
is the sklearn branch itself: same inertia (within 1 %) and label agreement from an
identical initialisation.  ``lloyd`` below is the plain algorithm (float64) used for
small deterministic cases; ``sklearn_fit`` wraps the reference's CPU branch.

The rest of the module is the float64 oracle of ONE Lloyd step as the kernels take it
(tests/test_gpu_kmeans_exact.py, checked on the host by tests/test_kmeans_oracle_host.py).

Distances.  ``D[i, j] = ||x_i - c_j||^2`` in float64, by the expansion after both X and C
are shifted by the column mean of X rounded to an integer: the shift removes any common
offset (the expansion's cancellation grows with ||x||^2), and an integer shift keeps
integer operands integers, so that D is exact for the lattice cases.

Acceptance rule (``accept``).  Both Lloyd paths must be no worse than the fp32 step
``exact_argmin`` (kmeans_tc.cuh): per centre, ``a_j = x.c_j`` by lane-strided ``fmaf``
chains of ceil(d/32) terms and a 5-level shuffle tree, ``cn_j = ||c_j||^2`` the same way,
``v_j = cn_j - 2 a_j``; the label is the lowest index of the smallest ``v_j``.  A dot
product of n terms accumulated through m = ceil(d/32) + 5 roundings in any tree shape has
``|a~ - x.c| <= gamma_m sum_i |x_i c_i|`` with ``gamma_m = m u / (1 - m u)``, u = 2^-24
(Higham, Accuracy and Stability, 3.1); the same for ``cn~`` with ``sum c_i^2``; the final
subtraction adds one rounding, ``u |cn - 2 a|`` to first order.  So the computed v_j obeys
``|v~_j - v_j| <= e_j = gamma_m (||c_j||^2 + 2 sum_i |x_i c_ji|) + u (||c_j||^2 + 2 |x.c_j|)``.
Since ``D_j = ||x||^2 + v_j`` (the row norm is common to every centre), a label l chosen
as the argmin of v~ satisfies ``D_l - D_j* <= e_l + e_j*`` for the float64 argmin j*.  That
is the rule; it gives the tensor-core step no slack of its own (its recheck band exists to
make it as good as this step), so a band that is too narrow fails instead of loosening a
tolerance.  On an exact float64 tie at the minimum the label must be the lowest index.

Per-element bounds for the other outputs (``dist_bound``, ``sums_bound``, inertia by
``inertia_bound``): ``dist = max(v~_l + xn~, 0)`` carries e_l, the rounding of xn~
(gamma_m ||x||^2) and one final rounding; the tensor-core step adds its documented claim
``|v~ - v| <= 2^-12 ||x|| max_j ||c_j||`` on rows it does not recheck.  Column sums of n
rows in fp32, in any order, are within ``gamma_(n-1) sum |x|``; counts are exact given the
labels; the inertia is the float64 sum of dist-like terms, within the sum of the dist
bounds, plus the rounding to float32.

The case generators at the bottom (``lattice``, ``probes``, ``blobs``, ``uniform``) build
the operands of the GPU tests.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24                 # unit roundoff of fp32
TC_V_CLAIM = 2.0 ** -12        # documented |v~ - v| <= 2^-12 ||x|| cmax of the tensor-core step (kmeans_tc.cu)


def assign(X, C):
    X = np.asarray(X, dtype=np.float64)
    C = np.asarray(C, dtype=np.float64)
    d2 = (X * X).sum(1)[:, None] - 2.0 * X @ C.T + (C * C).sum(1)[None, :]
    labels = d2.argmin(1)
    return labels.astype(np.int32), float(np.maximum(d2[np.arange(len(X)), labels], 0).sum())


def lloyd(X, init_centers, max_iter=300, tol=1e-4):
    """Lloyd iterations from fixed initial centers.  Empty clusters keep their center.
    Stops when the squared center shift <= tol * mean feature variance (sklearn's rule)."""
    X = np.asarray(X, dtype=np.float64)
    C = np.array(init_centers, dtype=np.float64)
    thr = tol * X.var(axis=0).mean()
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        labels, _ = assign(X, C)
        newC = C.copy()
        for j in range(len(C)):
            m = labels == j
            if m.any():
                newC[j] = X[m].mean(0)
        shift = ((newC - C) ** 2).sum()
        C = newC
        if shift <= thr:
            break
    labels, inertia = assign(X, C)
    return C, labels, inertia, n_iter


def sklearn_fit(X, k, init, n_init=1, max_iter=300, tol=1e-4, random_state=0):
    """The reference's CPU branch (clustering_gpu.py:135-142) with an explicit init."""
    from sklearn.cluster import KMeans

    km = KMeans(n_clusters=k, init=init, n_init=n_init, max_iter=max_iter, tol=tol,
                random_state=random_state, algorithm="lloyd")
    labels = km.fit_predict(X)
    return km.cluster_centers_, labels.astype(np.int32), float(km.inertia_), km.n_iter_


# ---------------------------------------------------------------- the one-step oracle
def chain_terms(d):
    """m: roundings in a lane-strided fmaf chain of ceil(d / 32) terms plus the 5-level shuffle tree"""
    return -(-int(d) // 32) + 5


def gamma(m):
    return m * U / (1.0 - m * U)


def _f64(a):
    return np.asarray(a, np.float32).astype(np.float64)


def distances(X, C):
    """exact-as-float64 D f64[N, k] = ||x_i - c_j||^2 (expansion after an integer shift by the column mean of X)"""
    return _distances64(_f64(X), _f64(C))


def fp32_errors(X, C):
    """e f64[N, k]: the bound on |v~_j - v_j| of the fp32 step for every (row, centre) (module docstring)"""
    X, C = _f64(X), _f64(C)
    g = gamma(chain_terms(X.shape[1]))
    cn = (C * C).sum(1)[None, :]
    return g * (cn + 2.0 * (np.abs(X) @ np.abs(C).T)) + U * (cn + 2.0 * np.abs(X @ C.T))


def oracle_labels(D):
    """float64 argmin, lowest index on exact ties"""
    return D.argmin(1).astype(np.int32)


def accept(X, C, labels, D=None, E=None):
    """-> bool[N]: each label passes the acceptance rule of the module docstring"""
    D = distances(X, C) if D is None else D
    E = fp32_errors(X, C) if E is None else E
    labels = np.asarray(labels, np.int64)
    r = np.arange(len(labels))
    if labels.min(initial=0) < 0 or labels.max(initial=0) >= D.shape[1]:
        return np.zeros(len(labels), bool) if len(labels) else np.ones(0, bool)
    js = D.argmin(1)
    Dl, Dm = D[r, labels], D[r, js]
    ok = Dl - Dm <= E[r, labels] + E[r, js]
    ok &= ~((Dl == Dm) & (labels != js))         # an exact tie at the minimum goes to the lowest index
    return ok


def margins(D, E):
    """(second - best) float64 gap of each row over the two smallest D, and the rule's slack e_best + e_second"""
    order = np.argsort(D, axis=1, kind="stable")[:, :2]
    r = np.arange(D.shape[0])
    if D.shape[1] == 1:
        return np.full(D.shape[0], np.inf), np.zeros(D.shape[0])
    return D[r, order[:, 1]] - D[r, order[:, 0]], E[r, order[:, 0]] + E[r, order[:, 1]]


def dist_bound(X, C, labels, tensor_cores):
    """per-row bound on |dist - D_label| (module docstring)"""
    X, C = _f64(X), _f64(C)
    labels = np.asarray(labels, np.int64)
    g = gamma(chain_terms(X.shape[1]))
    c = C[labels]
    xn, cn = (X * X).sum(1), (c * c).sum(1)
    xc = (X * c).sum(1)
    axc = (np.abs(X) * np.abs(c)).sum(1)
    b = g * (cn + 2.0 * axc) + g * xn + 2.0 * U * (xn + cn + 2.0 * np.abs(xc))
    if tensor_cores:
        b = b + TC_V_CLAIM * np.sqrt(xn) * np.sqrt((C * C).sum(1).max())
    return b


def sums_exact(X, labels, k):
    """float64 column sums and counts of the rows of each label"""
    X = _f64(X)
    labels = np.asarray(labels, np.int64)
    S = np.zeros((k, X.shape[1]))
    np.add.at(S, labels, X)
    return S, np.bincount(labels, minlength=k).astype(np.float64)


def sums_bound(X, labels, k):
    """per-element bound on fp32 column sums added in any order: gamma_(n_j - 1) sum |x| over the n_j rows"""
    A, n = sums_exact(np.abs(_f64(X)), labels, k)
    return np.array([gamma(max(int(c) - 1, 0)) for c in n])[:, None] * A


def inertia_bound(X, C, labels, tensor_cores, D=None):
    """-> (float64 sum of D_label, bound on |inertia - that| including the rounding to float32)"""
    D = distances(X, C) if D is None else D
    labels = np.asarray(labels, np.int64)
    tot = float(D[np.arange(len(labels)), labels].sum())
    return tot, float(dist_bound(X, C, labels, tensor_cores).sum()) + 2.0 * U * tot


def lloyd_step(X, C):
    """one float64 Lloyd step as scikit-learn's lloyd_iter_chunked_dense takes it: E-step (lowest index on ties),
    M-step sums, _relocate_empty_clusters_dense on float64 copies, then division (as _average_centers does it, a
    cluster still empty -- relocation returns early when every row sits on its centre -- moves to the centre of the
    first largest cluster).  -> (labels, new centres f64[k, d], counts before relocation)"""
    from sklearn.cluster._k_means_common import _relocate_empty_clusters_dense

    X64, C64 = _f64(X), np.asarray(C, np.float64)
    k = C64.shape[0]
    labels = oracle_labels(_distances64(X64, C64))
    S, n = sums_exact(X64, labels, k)
    n0 = n.copy()
    _relocate_empty_clusters_dense(np.ascontiguousarray(X64), np.ones(len(X64)), np.ascontiguousarray(C64), S, n,
                                   labels)
    newC = S / np.maximum(n, 1.0)[:, None]
    newC[n == 0] = newC[int(np.argmax(n))]
    return labels, newC, n0


def _distances64(X64, C64):
    s = np.rint(X64.mean(0))
    Xs, Cs = X64 - s, C64 - s
    return np.maximum((Xs * Xs).sum(1)[:, None] - 2.0 * (Xs @ Cs.T) + (Cs * Cs).sum(1)[None, :], 0.0)


def lloyd_trajectory(X, C, steps):
    """[(labels, centres after the step, counts before relocation, gap between each row's two nearest centres)] for
    `steps` float64 oracle Lloyd steps from the centres C (kept in float64 between steps)"""
    out = []
    C = np.asarray(C, np.float64)
    for _ in range(steps):
        D = np.sort(_distances64(_f64(X), C), axis=1)
        gap = D[:, 1] - D[:, 0] if C.shape[0] > 1 else np.full(len(D), np.inf)
        labels, newC, n0 = lloyd_step(X, C)
        out.append((labels, newC, n0, gap))
        C = newC
    return out


# ---------------------------------------------------------------- fp32 restatement of exact_argmin (host checks)
def fp32_step(X, C):
    """numpy float32 run of exact_argmin's arithmetic: lane-strided fma chains (float64 product + one rounding to
    float32 = one fmaf), the xor-shuffle tree, v = cn - 2 a, strict "<" in index order.  -> (labels, v f32[N, k],
    dist f32[N])"""
    X = np.asarray(X, np.float32)
    C = np.asarray(C, np.float32)
    N, d = X.shape
    k = C.shape[0]
    L = -(-d // 32) * 32
    Xp = np.zeros((N, L), np.float32); Xp[:, :d] = X
    Cp = np.zeros((k, L), np.float32); Cp[:, :d] = C

    def chains(A, B):  # A [n, L], B [k, L] -> fp32 [n, k] dot products in the kernel's order
        acc = np.zeros((A.shape[0], B.shape[0], 32), np.float32)
        for t in range(0, L, 32):
            acc = (acc.astype(np.float64) + A[:, None, t:t + 32].astype(np.float64)
                   * B[None, :, t:t + 32].astype(np.float64)).astype(np.float32)
        lanes = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            acc = (acc + acc[..., lanes ^ o]).astype(np.float32)
        return acc[..., 0]

    cn = np.array([chains(Cp[j:j + 1], Cp[j:j + 1])[0, 0] for j in range(k)], np.float32)
    xn = np.array([chains(Xp[i:i + 1], Xp[i:i + 1])[0, 0] for i in range(N)], np.float32) if N <= 64 else \
        _self_norms(Xp)
    a = np.concatenate([chains(Xp[r:r + 256], Cp) for r in range(0, N, 256)]) if N else np.zeros((0, k), np.float32)
    v = (cn[None, :] - np.float32(2) * a).astype(np.float32)
    labels = v.argmin(1).astype(np.int32)
    best = v[np.arange(N), labels]
    dist = np.maximum((best + xn).astype(np.float32), np.float32(0))
    return labels, v, dist


def _self_norms(Xp):
    acc = np.zeros((Xp.shape[0], 32), np.float32)
    for t in range(0, Xp.shape[1], 32):
        x = Xp[:, t:t + 32].astype(np.float64)
        acc = (acc.astype(np.float64) + x * x).astype(np.float32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, lanes ^ o]).astype(np.float32)
    return acc[:, 0]


# ---------------------------------------------------------------- case generators
def lattice_bound(d):
    """largest |entry| of a lattice case in d dimensions: bf16-exact (<= 256) and every sum of products, norm, v and
    dist below 2^22 in magnitude (4 d B^2 <= 2^24), so fp32 and the split-bf16 GEMM compute them exactly"""
    return int(max(1, min(256, math.isqrt((1 << 22) // max(1, d)))))


def lattice(N, d, k, seed=0):
    """small-integer rows and centres with planted exact ties: centre 1 duplicates centre 0 (when k > 1), and every
    fourth row is equidistant from two centres that differ by 2 in one coordinate.  -> (X f32[N, d], C f32[k, d])"""
    rng = np.random.default_rng(seed)
    B = lattice_bound(d)
    C = rng.integers(-B // 2, B // 2 + 1, (k, d)).astype(np.float64)
    if k > 1:
        C[1] = C[0]
    if k > 3:
        t = int(rng.integers(0, d))
        C[3] = C[2]
        C[3, t] += 2
    X = rng.integers(-B, B + 1, (N, d)).astype(np.float64)
    if k > 3:
        near = np.arange(0, N, 4)
        X[near] = C[2] + rng.integers(-1, 2, (len(near), d)) * (B >= 8)
        X[near, t] = C[2, t] + 1                    # ||x - c_2|| == ||x - c_3||
    elif k > 1:
        X[::4] = C[0] + rng.integers(-1, 2, (len(X[::4]), d))
    X = np.clip(X, -B, B)
    return X.astype(np.float32), C.astype(np.float32)


def probes(d, k=16, per_level=64, levels=range(4, 25), signed=False, seed=0):
    """near-tie probes: each row lies between two centres a, b at a float64 gap D_a - D_b of about
    +-2^-lev ||x|| max||c|| for every level, `per_level` rows each.  Non-negative (aligned) data is the worst case for
    an accumulation error with a bias.  -> (X f32, C f32, target level i32[N])"""
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((k, d)) if signed else 0.25 + 0.75 * rng.random((k, d))  # midpoints stay >= 0.25
    C = C.astype(np.float32).astype(np.float64)
    cmax = np.sqrt((C * C).sum(1).max())
    rows, lev = [], []
    for lv in levels:
        for _ in range(per_level):
            a, b = rng.choice(k, 2, replace=False)
            u = C[b] - C[a]
            m = 0.5 * (C[a] + C[b])
            y = rng.standard_normal(d) * (0.05 * np.sqrt((u * u).sum() / d))
            y -= (y @ u) / (u @ u) * u
            x = m + y
            g = rng.choice((-1.0, 1.0)) * 2.0 ** -lv * np.sqrt(x @ x) * cmax
            x = x + g / (2.0 * (u @ u)) * u        # D_a - D_b = 2 (x - m).u = g
            rows.append(x)
            lev.append(lv)
    return np.asarray(rows).astype(np.float32), C.astype(np.float32), np.asarray(lev, np.int32)


def blobs(N, d, k, seed=0, offset=0.0, spread=1.0):
    """task-shaped data: k Gaussian blobs (unit within-cluster sigma) in standard-scaled units, plus `offset` on every
    coordinate.  -> (X f32, C f32 = the blob centres + offset, true labels)"""
    rng = np.random.default_rng(seed)
    cen = rng.normal(0.0, spread, (k, d))
    lab = rng.integers(0, k, N)
    X = cen[lab] + rng.normal(0.0, 1.0, (N, d))
    return (X + offset).astype(np.float32), (cen + offset).astype(np.float32), lab.astype(np.int32)


def separated(N, d, k, seed=0):
    """well-separated blobs (centres 40 sigma apart along random directions) for Lloyd trajectories"""
    rng = np.random.default_rng(seed)
    cen = rng.standard_normal((k, d))
    cen *= 40.0 / np.linalg.norm(cen, axis=1, keepdims=True)
    cen += rng.normal(0, 5.0, (k, d))
    lab = np.arange(N) % k
    rng.shuffle(lab)
    X = cen[lab] + rng.normal(0.0, 1.0, (N, d))
    return X.astype(np.float32), cen.astype(np.float32), lab.astype(np.int32)


def uniform(N, d, k, seed=0):
    """structureless uniform [0, 1) rows, centres drawn from them: a large share of the rows are near-ties"""
    rng = np.random.default_rng(seed)
    X = rng.random((N, d), dtype=np.float32)
    return X, X[rng.choice(N, k, replace=False)].copy()
