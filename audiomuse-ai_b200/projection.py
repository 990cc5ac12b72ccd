"""The library map's 2-D projection on the GPU: tasks/song_alchemy._project_with_umap (:272-287), which runs
umap.UMAP(n_components=2).fit_transform on the host, as

    umap_fit_transform(X, n_neighbors, min_dist, spread, n_epochs, seed)   -> f32[N, 2]
    project_with_umap(vectors, n_components=2)                             -> [(x, y), ...] in [-1, 1], the drop-in

with umap-learn 0.5's defaults (euclidean, local_connectivity 1, learning rate 1, 5 negative samples per sample,
repulsion 1, spectral initialisation).  Stages:
    graph         am_umap_plan_create (csrc/umap.cu): exact k-NN, smooth_knn_dist, fuzzy union, pruning for n_epochs
    a, b          scipy's curve fit of 1 / (1 + a x^(2b)) on the host
    init          the spectral layout of the pruned graph, from clustering_gpu.spectral_embedding_csr (the eigensolver
                  of csrc/spectral.cu), one call per connected component; components placed as umap's
                  multi_component_layout does; scaled to max |.| = 10 with N(0, 1e-4) noise, columns rescaled to [0, 10]
    layout        am_umap_plan_layout: the SGD, one Jacobi update per vertex and epoch (bit-identical for a seed)

There is no CPU fallback: a missing device raises, and the reference's callers (app_helper.py:1340-1354,
app_map.py:157-166) then take their PCA projection, _project_to_2d.
"""
from __future__ import annotations

import ctypes as C
import functools
import time

import numpy as np

from . import _lib
from .clustering_gpu import _finite_f32, spectral_embedding_csr

GAMMA, ALPHA0, NEG_RATE = 1.0, 1.0, 5.0
MAP_SEED = 0        # the library map is the same on every rebuild of the same library


@functools.lru_cache(maxsize=16)
def find_ab_params(spread=1.0, min_dist=0.1):
    """umap's fit of 1 / (1 + a x^(2b)) to 1 below min_dist and exp(-(x - min_dist) / spread) above, over
    linspace(0, 3 spread, 300).  (1.57694, 0.89506) for the defaults."""
    from scipy.optimize import curve_fit

    xv = np.linspace(0, spread * 3, 300)
    yv = np.where(xv < min_dist, 1.0, np.exp(-(xv - min_dist) / spread))
    (a, b), _ = curve_fit(lambda x, a, b: 1.0 / (1.0 + a * x ** (2 * b)), xv, yv)
    return float(a), float(b)


def default_epochs(N):
    return 500 if N <= 10000 else 200


def _unit_vectors(G, dim, seed, stats=None):
    """unit eigenvectors of the 2nd .. (dim+1)-th smallest eigenvalues of G's normalised Laplacian (not divided by
    sqrt(deg)).  stats (a dict, optional) accumulates eigensolver_ms (the device plan and the solve, host clock) and
    eigensolver_calls, and keeps the eigenvalues of the last call."""
    t0 = time.perf_counter()
    emb, ev = spectral_embedding_csr(G, dim + 1, seed=seed)
    if stats is not None:
        stats["eigensolver_ms"] = stats.get("eigensolver_ms", 0.0) + 1e3 * (time.perf_counter() - t0)
        stats["eigensolver_calls"] = stats.get("eigensolver_calls", 0) + 1
        stats["eigenvalues"] = ev
    dd = np.sqrt(np.asarray(G.sum(axis=1)).ravel())
    return emb[:, 1:dim + 1] * dd[:, None]


def _solver(G, dim, seed, stats=None):
    """_unit_vectors, or None when the eigensolver does not converge (umap falls back to a random layout then); a
    device failure still raises"""
    try:
        return _unit_vectors(G, dim, seed, stats)
    except RuntimeError as e:
        if isinstance(e, _lib.B200Error):
            raise
        return None


def _meta_positions(X, n_comp, labels, dim, rng):
    """umap's placement of the connected components: +-e_i for at most 2 dim of them, otherwise the spectral embedding
    of the centroids' affinity exp(-||c_i - c_j||^2), divided by its maximum"""
    if n_comp <= 2 * dim:
        k = int(np.ceil(n_comp / 2.0))
        base = np.hstack([np.eye(k), np.zeros((k, dim - k))])
        return np.vstack([base, -base])[:n_comp]
    from sklearn.manifold import SpectralEmbedding
    cent = np.stack([X[labels == c].mean(0) for c in range(n_comp)])
    d2 = ((cent[:, None, :] - cent[None, :, :]) ** 2).sum(-1)
    emb = SpectralEmbedding(n_components=dim, affinity="precomputed",
                            random_state=int(rng.integers(2 ** 31))).fit_transform(np.exp(-d2))
    return emb / emb.max()


def _spectral_layout(X, W, dim, rng, seed, details):
    from scipy.sparse.csgraph import connected_components
    N = W.shape[0]
    n_comp, labels = connected_components(W, directed=False)
    details["components"] = int(n_comp)
    if n_comp == 1:
        return _solver(W, dim, seed, details)
    meta = _meta_positions(X.astype(np.float64), n_comp, labels, dim, rng)
    out = np.empty((N, dim))
    for c in range(n_comp):
        rows = np.flatnonzero(labels == c)
        dm = np.sqrt(((meta - meta[c]) ** 2).sum(1))
        half = dm[dm > 0].min() / 2.0
        U = None
        if len(rows) >= 2 * dim and len(rows) > dim + 1:
            U = _solver(W[rows][:, rows], dim, seed, details)
        if U is None:
            out[rows] = rng.uniform(-half, half, (len(rows), dim)) + meta[c]
        else:
            out[rows] = U * (half / np.abs(U).max()) + meta[c]
    return out


def initial_layout(X, W, seed=0, dim=2, details=None):
    """umap's initialisation of the pruned graph W: the spectral layout scaled to max |.| = 10 plus N(0, 1e-4) noise,
    uniform(-10, 10) when the eigensolver fails or N <= dim + 1; then every column rescaled to [0, 10].  f32[N, dim]"""
    details = {} if details is None else details
    details.update(eigensolver_ms=0.0, eigensolver_calls=0)
    rng = np.random.default_rng(seed)
    N = W.shape[0]
    emb = _spectral_layout(X, W, dim, rng, seed, details) if N > dim + 1 and W.nnz else None
    details["init"] = "random" if emb is None else "spectral"
    if emb is None:
        emb = rng.uniform(-10.0, 10.0, (N, dim))
    else:
        emb = emb * (10.0 / np.abs(emb).max()) + rng.normal(scale=1e-4, size=emb.shape)
    lo, hi = emb.min(0), emb.max(0)
    span = np.where(hi > lo, hi - lo, 1.0)
    return np.ascontiguousarray(10.0 * (emb - lo) / span, dtype=np.float32)


class UmapGraph:
    """A plan of csrc/umap.cu: the pruned fuzzy graph of X on the device, and the layout over it."""

    def __init__(self, X, n_neighbors=15, n_epochs=None):
        X = _finite_f32(X)
        N, d = X.shape
        if N < 2 or d < 1:
            raise ValueError(f"Found array with shape {X.shape}: UMAP needs at least 2 samples and 1 feature")
        if int(n_neighbors) < 2:
            raise ValueError(f"n_neighbors={n_neighbors} must be at least 2")
        self.X, self.N = X, N
        self.k = N - 1 if N <= int(n_neighbors) else int(n_neighbors)
        self.n_epochs = default_epochs(N) if n_epochs is None else int(n_epochs)
        if self.n_epochs < 1:
            raise ValueError(f"n_epochs={n_epochs} must be positive")
        self.lib = _lib.load()
        self.plan = C.c_void_p()
        _lib.check(self.lib.am_umap_plan_create(_lib.ptr(X), N, d, self.k, self.n_epochs, C.byref(self.plan)))

    def close(self):
        if self.plan:
            self.lib.am_umap_plan_free(self.plan)
            self.plan = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def info(self):
        nnz, knn_ms, graph_ms, layout_ms = C.c_int64(0), C.c_float(0), C.c_float(0), C.c_float(0)
        _lib.check(self.lib.am_umap_plan_info(self.plan, C.byref(nnz), None, None, C.byref(knn_ms), C.byref(graph_ms),
                                              C.byref(layout_ms)))
        return dict(nnz=int(nnz.value), knn_ms=float(knn_ms.value), graph_ms=float(graph_ms.value),
                    layout_ms=float(layout_ms.value))

    def graph(self):
        """-> dict(W: scipy CSR f64 (sorted indices), eps: epochs_per_sample f64[nnz], rho, sigma f64[N])"""
        import scipy.sparse as sp
        N, nnz = self.N, self.info()["nnz"]
        indptr, indices = np.empty(N + 1, np.int64), np.empty(max(nnz, 1), np.int32)
        w, eps = np.empty(max(nnz, 1)), np.empty(max(nnz, 1))
        rho, sigma = np.empty(N), np.empty(N)
        _lib.check(self.lib.am_umap_plan_graph(self.plan, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(w),
                                               _lib.ptr(rho), _lib.ptr(sigma), _lib.ptr(eps)))
        W = sp.csr_matrix((w[:nnz], indices[:nnz], indptr), shape=(N, N))
        return dict(W=W, eps=eps[:nnz], rho=rho, sigma=sigma)

    def layout(self, Y0, a, b, seed=0, epochs=None, gamma=GAMMA, alpha0=ALPHA0, neg_rate=NEG_RATE):
        """the SGD from Y0 f32[N, 2]: the first `epochs` (default all) epochs of the plan's schedule -> f32[N, 2]"""
        Y = np.array(Y0, dtype=np.float32, order="C", copy=True)
        if Y.shape != (self.N, 2):
            raise ValueError(f"Y0 must be ({self.N}, 2), got {Y.shape}")
        epochs = self.n_epochs if epochs is None else int(epochs)
        _lib.check(self.lib.am_umap_plan_layout(self.plan, _lib.ptr(Y), epochs, float(a), float(b), float(gamma),
                                                float(alpha0), float(neg_rate), int(seed) & 0xFFFFFFFFFFFFFFFF))
        return Y


def umap_fit_transform(X, n_neighbors=15, min_dist=0.1, spread=1.0, n_epochs=None, seed=0, details=None):
    """umap.UMAP(n_neighbors, min_dist, spread, n_epochs, n_components=2).fit_transform(X) on the device, with a fixed
    seed: the same input and seed give bit-identical output.  -> f32[N, 2].  details (a dict, optional) receives the
    graph (W, eps, rho, sigma), a, b, the initial layout, the connected components, the eigensolver calls and the stage
    times in ms (knn, graph, init -- of which eigensolver is the device eigensolver's share --, layout, total)."""
    t0 = time.perf_counter()
    a, b = find_ab_params(float(spread), float(min_dist))
    with UmapGraph(X, n_neighbors, n_epochs) as g:
        G = g.graph()
        t1 = time.perf_counter()
        init = {}
        Y0 = initial_layout(g.X, G["W"], seed=seed, details=init)
        t2 = time.perf_counter()
        Y = g.layout(Y0, a, b, seed=seed)
        info = g.info()
    if details is not None:
        details.update(G)
        details.update(init)
        details.update(a=a, b=b, Y0=Y0, n_neighbors=g.k, n_epochs=g.n_epochs, nnz=info["nnz"], knn_ms=info["knn_ms"],
                       graph_ms=info["graph_ms"], init_ms=1e3 * (t2 - t1), layout_ms=info["layout_ms"],
                       total_ms=1e3 * (time.perf_counter() - t0))
    return Y


def project_with_umap(vectors, n_components=2):
    """tasks/song_alchemy._project_with_umap on the device: the rows' UMAP layout, centred by its mean, divided by its
    largest absolute value and clipped to [-1, 1], as a list of (x, y).  [] for no vectors.  ValueError for
    n_components != 2 and for NaN / inf, before any device work."""
    if int(n_components) != 2:
        raise ValueError(f"n_components={n_components}: the GPU projection computes 2 components only")
    if len(vectors) == 0:
        return []
    mat = np.vstack(vectors)
    if not np.isfinite(mat).all():
        raise ValueError("Input contains NaN or infinity.")
    return scale_to_unit(umap_fit_transform(mat, seed=MAP_SEED))


def scale_to_unit(embedding):
    """song_alchemy.py:280-287: centre by the mean, divide by the largest absolute value (all zeros when it is 0),
    clip to [-1, 1] -> a list of (x, y)"""
    centred = embedding - embedding.mean(axis=0)
    max_abs = np.max(np.abs(centred))
    if max_abs == 0:
        return [(0.0, 0.0) for _ in range(len(embedding))]
    scaled = np.clip(centred / max_abs, -1.0, 1.0)
    return [(float(x), float(y)) for x, y in scaled]
