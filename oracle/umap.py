"""Oracle: UMAP with the defaults tasks/song_alchemy._project_with_umap uses.  TEST INFRASTRUCTURE ONLY.

Source.  umap-learn is neither installed nor available where this was written.  The rules below are restated from the
published algorithm (McInnes, Healy & Melville 2018, "UMAP: Uniform Manifold Approximation and Projection for
Dimension Reduction", arXiv:1802.03426) and from umap-learn 0.5's umap_.py / layouts.py / spectral.py as their
maintainer remembers them.  Points marked [unverified] could not be checked against umap-learn's code:

  * n_neighbors = N - 1 when N <= n_neighbors [unverified];
  * the per-column rescale of the initial layout to [0, 10] [unverified: in 0.5.x as remembered];
  * multi_component_layout's details [unverified];
  * a negative sample at zero distance moves nothing [unverified: older versions moved it by 4].

Defaults: n_neighbors 15, min_dist 0.1, spread 1, euclidean, 2 components, learning_rate 1, negative_sample_rate 5,
repulsion_strength 1, set_op_mix_ratio 1, local_connectivity 1, init 'spectral'.

Two layouts:
  * sgd_sequential: umap's single-threaded edge order (numba), each sample applied at once, negatives from a seeded
    generator -- the quality reference;
  * sgd_jacobi: the device's rule restated in float64 -- every vertex moves from the previous epoch's snapshot, and the
    negative samples come from the same counter-based hash -- for short runs compared value by value.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

N_NEIGHBORS, MIN_DIST, SPREAD, NEG_RATE, GAMMA, ALPHA0 = 15, 0.1, 1.0, 5, 1.0, 1.0
SMOOTH_K_TOLERANCE, MIN_K_DIST_SCALE = 1e-5, 1e-3


def find_ab_params(spread=SPREAD, min_dist=MIN_DIST):
    """umap's curve fit: 1 / (1 + a x^(2b)) against 1 below min_dist and exp(-(x - min_dist) / spread) above."""
    from scipy.optimize import curve_fit

    def curve(x, a, b):
        return 1.0 / (1.0 + a * x ** (2 * b))

    xv = np.linspace(0, spread * 3, 300)
    yv = np.zeros(xv.shape)
    yv[xv < min_dist] = 1.0
    yv[xv >= min_dist] = np.exp(-(xv[xv >= min_dist] - min_dist) / spread)
    params, _ = curve_fit(curve, xv, yv)
    return float(params[0]), float(params[1])


def default_epochs(N):
    return 500 if N <= 10000 else 200


def effective_neighbors(N, n_neighbors=N_NEIGHBORS):
    if N < 2:
        raise ValueError(f"UMAP needs at least 2 samples, got {N}")
    return N - 1 if N <= n_neighbors else n_neighbors


def knn(X, k, chunk=1024):
    """(ids i64[N, k], dist f64[N, k]): the row itself first, then its k - 1 nearest other rows (ascending float64
    euclidean distance from the float32 values, ties to the lower id), true (not squared) distances."""
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    N = len(X)
    sq = (X * X).sum(1)
    m = min(N, k + 8)
    ids = np.empty((N, k), np.int64)
    dist = np.empty((N, k))
    for lo in range(0, N, chunk):
        hi = min(N, lo + chunk)
        d2 = sq[lo:hi, None] - 2.0 * X[lo:hi] @ X.T + sq[None, :]
        # candidates: every row within rounding of the m-th smallest expanded distance, so that ties (duplicates) are
        # all re-ranked exactly and the lower ids win
        kth = np.partition(d2, m - 1, axis=1)[:, m - 1] if m < N else np.full(hi - lo, np.inf)
        slack = 1e-9 * (sq[lo:hi] + sq.max()) + 1e-12
        for r in range(hi - lo):
            i = lo + r
            c = np.flatnonzero(d2[r] <= kth[r] + slack[r])
            c = c[c != i]
            de = np.sqrt(((X[c] - X[i]) ** 2).sum(1))
            o = np.lexsort((c, de))[:k - 1]
            ids[i, 0], dist[i, 0] = i, 0.0
            ids[i, 1:], dist[i, 1:] = c[o], de[o]
    return ids, dist


def smooth_knn_dist(dist, k):
    """-> (sigma, rho, converged) f64[N]: umap's bisection, float64, local_connectivity 1."""
    N = dist.shape[0]
    target = np.log2(k)
    mean_all = dist.mean()
    rho, sigma = np.zeros(N), np.zeros(N)
    ok = np.zeros(N, bool)
    for i in range(N):
        d = dist[i]
        nz = d[d > 0.0]
        rho[i] = nz.min() if nz.size else 0.0
        lo, hi, mid = 0.0, np.inf, 1.0
        for _ in range(64):
            t = d[1:] - rho[i]
            psum = np.where(t > 0, np.exp(-(np.maximum(t, 0) / mid)), 1.0).sum()
            if abs(psum - target) < SMOOTH_K_TOLERANCE:
                ok[i] = True
                break
            if psum > target:
                hi = mid
                mid = (lo + hi) / 2.0
            else:
                lo = mid
                mid = mid * 2 if hi == np.inf else (lo + hi) / 2.0
        floor = MIN_K_DIST_SCALE * (d.mean() if rho[i] > 0.0 else mean_all)
        sigma[i] = max(mid, floor)
        ok[i] |= mid < floor
    return sigma, rho, ok


def membership(ids, dist, rho, sigma):
    N, k = ids.shape
    t = dist - rho[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        m = np.exp(-(t / sigma[:, None]))
    m = np.where((t <= 0.0) | (sigma[:, None] == 0.0), 1.0, m)
    m[ids == np.arange(N)[:, None]] = 0.0
    return m


def fuzzy_graph(X, n_neighbors=N_NEIGHBORS, n_epochs=None):
    """The pruned fuzzy union W (scipy CSR, f64, sorted indices), its epochs_per_sample, rho, sigma, k, n_epochs."""
    N = len(X)
    k = effective_neighbors(N, n_neighbors)
    n_epochs = default_epochs(N) if n_epochs is None else int(n_epochs)
    ids, dist = knn(X, k)
    sigma, rho, _ = smooth_knn_dist(dist, k)
    m = membership(ids, dist, rho, sigma)
    A = sp.csr_matrix((m.ravel(), ids.ravel(), np.arange(0, N * k + 1, k)), shape=(N, N))
    At = A.T.tocsr()
    W = (A + At - A.multiply(At)).tocsr()
    W.eliminate_zeros()
    if W.nnz:
        W.data[W.data < W.data.max() / float(n_epochs)] = 0.0
        W.eliminate_zeros()
    W.sort_indices()
    eps = epochs_per_sample(W.data, n_epochs)
    return dict(W=W, eps=eps, rho=rho, sigma=sigma, k=k, n_epochs=n_epochs)


def epochs_per_sample(w, n_epochs):
    if w.size == 0:
        return w.copy()
    n = n_epochs * (w / w.max())
    return float(n_epochs) / n


# ---------------------------------------------------------------- initialisation (umap's spectral_layout)


def _laplacian_vectors(G, dim):
    from scipy.sparse.linalg import eigsh
    deg = np.asarray(G.sum(axis=0)).ravel()
    D = sp.diags(1.0 / np.sqrt(deg))
    L = sp.identity(G.shape[0]) - D @ G @ D
    k = dim + 1
    ncv = max(2 * k + 1, int(np.sqrt(G.shape[0])))
    w, v = eigsh(L, k, which="SM", ncv=ncv, tol=1e-4, v0=np.ones(L.shape[0]), maxiter=G.shape[0] * 5)
    return v[:, np.argsort(w)[1:k]]


def component_layout(X, n_comp, labels, dim, rng):
    from sklearn.manifold import SpectralEmbedding
    cent = np.stack([X[labels == c].mean(0) for c in range(n_comp)])
    d2 = ((cent[:, None, :] - cent[None, :, :]) ** 2).sum(-1)
    emb = SpectralEmbedding(n_components=dim, affinity="precomputed",
                            random_state=int(rng.integers(2 ** 31))).fit_transform(np.exp(-d2))
    return emb / emb.max()


def meta_positions(X, n_comp, labels, dim, rng):
    if n_comp > 2 * dim:
        return component_layout(X, n_comp, labels, dim, rng)
    k = int(np.ceil(n_comp / 2.0))
    base = np.hstack([np.eye(k), np.zeros((k, dim - k))])
    return np.vstack([base, -base])[:n_comp]


def spectral_layout(X, W, dim, rng, vectors=_laplacian_vectors):
    """umap's spectral_layout / multi_component_layout; `vectors(G, dim)` returns the unit eigenvectors of the 2nd ..
    (dim+1)-th smallest eigenvalues of G's normalised Laplacian (the device solver in the product)."""
    from scipy.sparse.csgraph import connected_components
    N = W.shape[0]
    n_comp, labels = connected_components(W, directed=False)
    if n_comp == 1:
        return vectors(W, dim)
    meta = meta_positions(np.asarray(X, np.float64), n_comp, labels, dim, rng)
    out = np.empty((N, dim))
    for c in range(n_comp):
        rows = np.flatnonzero(labels == c)
        dm = np.sqrt(((meta - meta[c]) ** 2).sum(1))
        half = dm[dm > 0].min() / 2.0
        if len(rows) < 2 * dim or len(rows) <= dim + 1:
            out[rows] = rng.uniform(-half, half, (len(rows), dim)) + meta[c]
            continue
        G = W[rows][:, rows]
        try:
            e = vectors(G, dim)
        except Exception:
            out[rows] = rng.uniform(-half, half, (len(rows), dim)) + meta[c]
            continue
        out[rows] = e * (half / np.abs(e).max()) + meta[c]
    return out


def initial_layout(X, W, rng, dim=2, vectors=_laplacian_vectors):
    """spectral layout, scaled to max |.| = 10 plus N(0, 1e-4) noise (uniform(-10, 10) when the solver fails or
    N <= dim + 1), then every column rescaled to [0, 10]."""
    N = W.shape[0]
    emb = None
    if N > dim + 1 and W.nnz:
        try:
            emb = spectral_layout(X, W, dim, rng, vectors)
        except Exception:
            emb = None
    if emb is None:
        emb = rng.uniform(-10.0, 10.0, (N, dim))
    else:
        emb = emb * (10.0 / np.abs(emb).max()) + rng.normal(scale=1e-4, size=emb.shape)
    lo, hi = emb.min(0), emb.max(0)
    span = np.where(hi > lo, hi - lo, 1.0)
    return (10.0 * (emb - lo) / span).astype(np.float32)


# ---------------------------------------------------------------- layouts

def _sequential_kernel():
    from numba import njit

    @njit(cache=False)
    def run(Y, head, tail, eps, n_epochs, a, b, gamma, alpha0, neg_rate, seed):
        np.random.seed(seed)
        N = Y.shape[0]
        E = head.shape[0]
        epsn = eps / neg_rate
        nxt = eps.copy()
        nxn = epsn.copy()
        for n in range(n_epochs):
            alpha = alpha0 * (1.0 - n / n_epochs)
            for e in range(E):
                if nxt[e] > n:
                    continue
                i, j = head[e], tail[e]
                d2 = 0.0
                for c in range(2):
                    d2 += (Y[i, c] - Y[j, c]) ** 2
                g = 0.0
                if d2 > 0.0:
                    g = -2.0 * a * b * d2 ** (b - 1.0) / (a * d2 ** b + 1.0)
                for c in range(2):
                    gd = min(4.0, max(-4.0, g * (Y[i, c] - Y[j, c])))
                    Y[i, c] += gd * alpha
                    Y[j, c] -= gd * alpha
                nxt[e] += eps[e]
                nn = int((n - nxn[e]) / epsn[e])
                for _ in range(nn):
                    kk = np.random.randint(0, N)
                    if kk == i:
                        continue
                    q2 = 0.0
                    for c in range(2):
                        q2 += (Y[i, c] - Y[kk, c]) ** 2
                    if q2 <= 0.0:
                        continue
                    g = 2.0 * gamma * b / ((0.001 + q2) * (a * q2 ** b + 1.0))
                    for c in range(2):
                        Y[i, c] += min(4.0, max(-4.0, g * (Y[i, c] - Y[kk, c]))) * alpha
                nxn[e] += nn * epsn[e]
        return Y

    return run


_SEQ = None


def sgd_sequential(Y0, W, eps, n_epochs, a, b, seed, gamma=GAMMA, alpha0=ALPHA0, neg_rate=NEG_RATE):
    """umap's optimize_layout_euclidean order: edges in CSR order, both endpoints moved at once (float64)."""
    global _SEQ
    if _SEQ is None:
        _SEQ = _sequential_kernel()
    C = W.tocoo()
    Y = np.asarray(Y0, np.float64).copy()
    return _SEQ(Y, C.row.astype(np.int64), C.col.astype(np.int64), np.asarray(eps, np.float64), int(n_epochs),
                float(a), float(b), float(gamma), float(alpha0), float(neg_rate), int(seed))


_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def negative_ids(seed, n, e, p, N):
    """the device's negative sample p of CSR entry e in epoch n"""
    with np.errstate(over="ignore"):
        ek = splitmix64(np.uint64(seed) ^ (np.uint64(n) * np.uint64(0xD1B54A32D192ED03)))
    h = splitmix64(splitmix64(ek ^ np.asarray(e, np.uint64)) ^ np.asarray(p, np.uint64))
    return (h % np.uint64(N)).astype(np.int64)


def sgd_jacobi(Y0, W, eps, n_epochs, a, b, seed, epochs=None, gamma=GAMMA, alpha0=ALPHA0, neg_rate=NEG_RATE):
    """The device's rule in float64: the first `epochs` epochs of the n_epochs schedule, every vertex moved from the
    previous epoch's snapshot by 2x its sampled row entries' attraction plus its own negative samples; the embedding
    is rounded to float32 after every epoch, as the device stores it."""
    W = W.tocsr()
    N = W.shape[0]
    rows = np.repeat(np.arange(N), np.diff(W.indptr))
    cols = W.indices.astype(np.int64)
    eps = np.asarray(eps, np.float64)
    epsn = eps / neg_rate
    nxt, nxn = eps.copy(), epsn.copy()
    Y = np.asarray(Y0, np.float64).copy()
    for n in range(n_epochs if epochs is None else epochs):
        alpha = alpha0 * (1.0 - n / n_epochs)
        e = np.flatnonzero(nxt <= n)
        i, j = rows[e], cols[e]
        diff = Y[i] - Y[j]
        d2 = (diff ** 2).sum(1)
        with np.errstate(divide="ignore", invalid="ignore"):
            g = np.where(d2 > 0, -2.0 * a * b * d2 ** (b - 1.0) / (a * d2 ** b + 1.0), 0.0)
        step = np.zeros_like(Y)
        np.add.at(step, i, 2.0 * np.clip(g[:, None] * diff, -4, 4))
        nxt[e] += eps[e]
        nn = ((n - nxn[e]) / epsn[e]).astype(np.int64)
        ee = np.repeat(e, nn)
        pp = np.arange(nn.sum()) - np.repeat(np.cumsum(nn) - nn, nn)
        hi = rows[ee]
        kk = negative_ids(seed, n, ee, pp, N)
        diff = Y[hi] - Y[kk]
        q2 = (diff ** 2).sum(1)
        keep = (kk != hi) & (q2 > 0)
        g = 2.0 * gamma * b / ((0.001 + q2[keep]) * (a * q2[keep] ** b + 1.0))
        np.add.at(step, hi[keep], np.clip(g[:, None] * diff[keep], -4, 4))
        nxn[e] += nn * epsn[e]
        Y = (Y + alpha * step).astype(np.float32).astype(np.float64)      # the device keeps the embedding in float32
    return Y


def umap_sequential(X, seed, n_neighbors=N_NEIGHBORS, min_dist=MIN_DIST, spread=SPREAD, n_epochs=None):
    """The whole oracle pipeline: graph, initialisation, sequential SGD.  -> (f32[N, 2], graph dict)"""
    g = fuzzy_graph(X, n_neighbors, n_epochs)
    a, b = find_ab_params(spread, min_dist)
    rng = np.random.default_rng(seed)
    Y0 = initial_layout(X, g["W"], rng)
    Y = sgd_sequential(Y0, g["W"], g["eps"], g["n_epochs"], a, b, seed)
    return Y.astype(np.float32), g


def knn_recall(X, Y, k=15):
    """mean share of each row's k nearest neighbours in X that are among its k nearest in Y"""
    from sklearn.neighbors import NearestNeighbors
    a = NearestNeighbors(n_neighbors=k + 1).fit(X).kneighbors(X, return_distance=False)[:, 1:]
    b = NearestNeighbors(n_neighbors=k + 1).fit(Y).kneighbors(Y, return_distance=False)[:, 1:]
    return float(np.mean([len(np.intersect1d(a[i], b[i])) / k for i in range(len(X))]))


def quality(X, Y, labels=None, k=15):
    from sklearn.manifold import trustworthiness
    from sklearn.metrics import silhouette_score
    out = dict(trustworthiness=float(trustworthiness(X, Y, n_neighbors=k)), knn_recall=knn_recall(X, Y, k))
    if labels is not None:
        out["silhouette"] = float(silhouette_score(Y, labels))
    return out
