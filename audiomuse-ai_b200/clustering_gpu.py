"""Mirror of ``tasks/clustering_gpu.py`` (KMeans rows of SURVEY 8(a)) on the GPU library.

    check_gpu_available()                      tasks/clustering_gpu.py:26-79
    GPUKMeans(n_clusters, init, n_init, random_state).fit_predict(X)   :82-148
        -> labels; sets cluster_centers_, labels_, using_gpu, inertia_, n_iter_
    get_clustering_model('kmeans', {'n_clusters': k}, use_gpu)          :338-404

cuML is replaced by am_kmeans_fit (k-means++ D^2 seeding, n_init restarts, Lloyd with sklearn's
tol rule).  kmeans_fit_batch fits many small problems at once (am_kmeans_fit_batch: one CTA per (problem, init), the
same definition and seeds as am_kmeans_fit), for the clustering task's batches of iterations.  The reference silently falls back to sklearn when the GPU path raises (:130-148);
here that fallback exists only when ``B200_ALLOW_SKLEARN_FALLBACK=1`` (default: fail loudly,
so a missing CUDA library can never masquerade as the GPU path).

    GPUDBSCAN(eps, min_samples).fit_predict(X)                         :151-199  -> am_dbscan (exact, sklearn's labels)
    GPUPCA(n_components).fit_transform(X) / inverse_transform(X)      :201-277  -> am_pca_moments + LAPACK eigh on the
        host + am_pca_project; sets components_, explained_variance_ratio_, n_components_ like sklearn's PCA
    get_pca_model(n_components, use_gpu)                               :407-421

    GPUSpectralClustering(n_clusters, ..., n_neighbors, random_state, n_init).fit_predict(X)   :312-335 -> the reference
        wraps sklearn.cluster.SpectralClustering; here spectral_embedding (k-NN graph + Chebyshev-filtered subspace
        iteration, csrc/spectral.cu) + kmeans_fit on the embedding.  Sets labels_, using_gpu; no cluster_centers_.

    GPUGaussianMixture(n_components, covariance_type='full', init_params='k-means++', n_init, random_state,
        reg_covar).fit_predict(X)   :284-309 -> the reference wraps sklearn.mixture.GaussianMixture; here gmm_fit
        (am_gmm_fit, csrc/gmm.cu): scikit-learn's k-means++ initialisation on the generator's own draws and float64
        EM on the tensor cores.  Sets means_, weights_, covariances_, precisions_cholesky_, lower_bound_,
        lower_bounds_, n_iter_, converged_, labels_, using_gpu.  Only covariance_type='full' runs on the device.
    GPUGaussianMixtureAnyCovariance(...): the same for all four covariance types;
        integration.apply(gaussian_mixture=..., gmm_all_covariance_types=True) installs it.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
import time
import warnings
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _lib
from .artist_gmm import draws_per_init, kpp_draws

logger = logging.getLogger("tasks.clustering_gpu")


def check_gpu_available() -> bool:
    try:
        return _lib.load().am_init(-1) == _lib.AM_OK
    except Exception as e:
        logger.info(f"GPU library unavailable: {e}")
        return False


def kmeans_fit(X, k, n_init=10, max_iter=300, tol=1e-4, seed=0, init_centers=None):
    """-> (centers f32[k,d], labels i32[N], inertia, n_iter) via am_kmeans_fit.  X and init_centers are validated as
    scikit-learn does (ValueError for another rank, NaN or inf) before any device work."""
    X = _finite_f32(X)
    N, d = X.shape
    init = None
    if init_centers is not None:
        init = _finite_f32(init_centers)
        if init.shape != (k, d):
            raise ValueError(f"init_centers must be ({k}, {d})")
    lib = _lib.load()
    centers = np.empty((k, d), dtype=np.float32)
    labels = np.empty((N,), dtype=np.int32)
    inertia, n_iter = C.c_float(0), C.c_int(0)
    _lib.check(lib.am_kmeans_fit(_lib.ptr(X), N, d, int(k), int(n_init), int(max_iter), float(tol),
                                 int(seed) & 0xFFFFFFFFFFFFFFFF, None if init is None else _lib.ptr(init),
                                 _lib.ptr(centers), _lib.ptr(labels), C.byref(inertia), C.byref(n_iter)))
    return centers, labels, float(inertia.value), int(n_iter.value)


def kmeans_batch_serves(N, d, k):
    """True when am_kmeans_fit_batch holds the shape (centres and sums in one CTA's shared memory); larger problems
    go to am_kmeans_fit"""
    return N <= _lib.KMEANS_BATCH_MAX_ROWS and max(k, 8) * (d + 1) <= _lib.KMEANS_BATCH_MAX_KD


def kmeans_fit_batch(problems, k, n_init=10, max_iter=300, tol=1e-4, seeds=0, intermediates=False):
    """Many independent k-means fits at once.  problems: a sequence of [N_p, d_p] arrays; k and seeds: one value for
    every problem or one per problem.  -> one (centers f32[k, d], labels i32[N], inertia, n_iter) per problem, each
    kmeans_fit(problem, k, n_init, max_iter, tol, seed)'s definition; with intermediates, a fifth entry: the k-means++
    rows i32[n_init, k] (None for a problem am_kmeans_fit serves).  Problems am_kmeans_fit_batch holds run together
    on the device (am_kmeans_fit_batch); the others one by one through kmeans_fit.  Every input is checked, with
    scikit-learn's ValueError wording, before any device work."""
    Xs = [_finite_f32(X) for X in problems]
    P = len(Xs)
    ks = [int(k)] * P if np.ndim(k) == 0 else [int(v) for v in k]
    sd = [int(seeds)] * P if np.ndim(seeds) == 0 else [int(v) for v in seeds]
    if len(ks) != P or len(sd) != P:
        raise ValueError(f"k and seeds need one value per problem ({P})")
    for X, kk in zip(Xs, ks):
        N, d = X.shape
        if d < 1:
            raise ValueError(f"Found array with 0 feature(s) (shape={X.shape}) while a minimum of 1 is required "
                             "by KMeans.")
        if kk < 1:
            raise ValueError(f"The 'n_clusters' parameter of KMeans must be an int in the range [1, inf). Got {kk} "
                             "instead.")
        if N < kk:
            raise ValueError(f"n_samples={N} should be >= n_clusters={kk}.")
    if n_init < 1 or max_iter < 1:
        raise ValueError("n_init and max_iter must be >= 1")
    out = [None] * P
    batch = [p for p in range(P) if kmeans_batch_serves(Xs[p].shape[0], Xs[p].shape[1], ks[p])]
    for p in range(P):
        if p not in batch:
            r = kmeans_fit(Xs[p], ks[p], n_init=n_init, max_iter=max_iter, tol=tol, seed=sd[p])
            out[p] = r + (None,) if intermediates else r
    if not batch:
        return out
    ns = np.array([Xs[p].shape[0] for p in batch], np.int64)
    ds = np.array([Xs[p].shape[1] for p in batch], np.int32)
    kb = np.array([ks[p] for p in batch], np.int32)
    row_off = np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)
    cen_off = np.concatenate([[0], np.cumsum(kb.astype(np.int64) * ds)]).astype(np.int64)
    kpp_off = np.concatenate([[0], np.cumsum(kb.astype(np.int64) * n_init)]).astype(np.int64)
    rows = np.ascontiguousarray(np.concatenate([Xs[p].ravel() for p in batch]))
    seeds_u = np.array([sd[p] & 0xFFFFFFFFFFFFFFFF for p in batch], np.uint64)
    centers = np.empty(int(cen_off[-1]), np.float32)
    labels = np.empty(int(row_off[-1]), np.int32)
    inertia = np.empty(len(batch), np.float32)
    n_iter = np.empty(len(batch), np.int32)
    kpp = np.empty(int(kpp_off[-1]), np.int32) if intermediates else None
    lib = _lib.load()
    _lib.check(lib.am_kmeans_fit_batch(_lib.ptr(rows), _lib.ptr(row_off), int(row_off[-1]), _lib.ptr(ds), _lib.ptr(kb),
                                       len(batch), int(n_init), int(max_iter), float(tol), _lib.ptr(seeds_u),
                                       _lib.ptr(centers), _lib.ptr(cen_off), _lib.ptr(labels), _lib.ptr(inertia),
                                       _lib.ptr(n_iter), None if kpp is None else _lib.ptr(kpp)))
    for i, p in enumerate(batch):
        r = (centers[cen_off[i]:cen_off[i + 1]].reshape(kb[i], ds[i]).copy(),
             labels[row_off[i]:row_off[i + 1]].copy(), float(inertia[i]), int(n_iter[i]))
        out[p] = r + (kpp[kpp_off[i]:kpp_off[i + 1]].reshape(n_init, kb[i]).copy(),) if intermediates else r
    return out


class GPUKMeans:
    def __init__(self, n_clusters, init="k-means++", n_init=10, random_state=None, max_iter=300, tol=1e-4):
        self.n_clusters = n_clusters
        self.init = init
        self.n_init = n_init
        self.random_state = random_state
        self.max_iter = max_iter
        self.tol = tol
        self.model = None
        self.cluster_centers_ = None
        self.labels_ = None
        self.inertia_ = None
        self.n_iter_ = None
        self.using_gpu = False

    def fit_predict(self, X):
        try:
            init_centers = None if isinstance(self.init, str) else np.asarray(self.init, dtype=np.float32)
            seed = 0 if self.random_state is None else int(self.random_state)
            c, l, inertia, it = kmeans_fit(X, int(self.n_clusters), n_init=int(self.n_init),
                                           max_iter=self.max_iter, tol=self.tol, seed=seed,
                                           init_centers=init_centers)
            self.cluster_centers_, self.labels_, self.inertia_, self.n_iter_ = c, l, inertia, it
            self.using_gpu = True
            logger.debug(f"GPU KMeans completed: {self.n_clusters} clusters")
            return l
        except Exception as e:
            if os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") != "1":
                raise
            logger.warning(f"GPU KMeans failed, falling back to CPU: {e}")
        from sklearn.cluster import KMeans
        self.model = KMeans(n_clusters=self.n_clusters, init=self.init, n_init=self.n_init,
                            random_state=self.random_state)
        labels = self.model.fit_predict(X)
        self.cluster_centers_ = self.model.cluster_centers_
        self.labels_ = labels
        self.using_gpu = False
        return labels

    def fit(self, X):
        self.fit_predict(X)
        return self

    def predict(self, X):
        X = np.asarray(X, dtype=np.float32)
        c = self.cluster_centers_
        d2 = (X * X).sum(1)[:, None] - 2.0 * X @ c.T + (c * c).sum(1)[None, :]
        return d2.argmin(1).astype(np.int32)


def _finite_f32(X):
    """X as C-contiguous float32 [N, d]; ValueError (scikit-learn's) for another rank or for NaN / inf, also after the
    cast to float32, before any device work.  A non-finite row is adjacent to nothing in the distance kernels, so without
    this check DBSCAN would call it noise and PCA would feed NaN to eigh."""
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError(f"Expected 2D array, got {X.ndim}D array instead")
    with np.errstate(over="ignore"):   # a float64 value beyond float32's range becomes inf here and is reported below
        X32 = np.ascontiguousarray(X, dtype=np.float32)
    if not (np.isfinite(X).all() and np.isfinite(X32).all()):
        raise ValueError("Input X contains NaN or infinity.")
    return X32


class GPUDBSCAN:
    """tasks/clustering_gpu.py:151-199.  labels_ are sklearn.cluster.DBSCAN's (same numbering), computed on the device."""

    def __init__(self, eps, min_samples):
        self.eps = eps
        self.min_samples = min_samples
        self.model = None
        self.labels_ = None
        self.n_clusters_ = None
        self.using_gpu = False

    def fit_predict(self, X):
        X = _finite_f32(X)
        try:
            labels = np.empty((X.shape[0],), dtype=np.int32)
            n = C.c_int(0)
            _lib.check(_lib.load().am_dbscan(_lib.ptr(X), X.shape[0], X.shape[1], float(self.eps), int(self.min_samples),
                                             _lib.ptr(labels), C.byref(n)))
            self.labels_, self.n_clusters_, self.using_gpu = labels, int(n.value), True
            logger.debug(f"GPU DBSCAN completed: eps={self.eps}, min_samples={self.min_samples}")
            return labels
        except Exception as e:
            if os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") != "1":
                raise
            logger.warning(f"GPU DBSCAN failed, falling back to CPU: {e}")
        from sklearn.cluster import DBSCAN
        self.model = DBSCAN(eps=self.eps, min_samples=self.min_samples)
        self.labels_ = self.model.fit_predict(X)
        self.using_gpu = False
        return self.labels_

    def fit(self, X):
        self.fit_predict(X)
        return self


def pca_fit(X, n_components):
    """-> (mean f64[d], components f64[k, d], explained_variance f64[k], total_variance) with sklearn.decomposition.PCA's
    conventions: covariance with n - 1, components sorted by variance, sign of each component chosen so that its
    largest-magnitude coordinate is positive (svd_flip(u_based_decision=False))."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    N, d = X.shape
    mean = np.empty((d,), dtype=np.float64)
    cov = np.empty((d, d), dtype=np.float64)
    _lib.check(_lib.load().am_pca_moments(_lib.ptr(X), N, d, _lib.ptr(mean), _lib.ptr(cov)))
    w, v = np.linalg.eigh(cov)                      # ascending
    order = np.argsort(w)[::-1][:n_components]
    comps = v[:, order].T.copy()
    idx = np.argmax(np.abs(comps), axis=1)
    signs = np.sign(comps[np.arange(comps.shape[0]), idx])
    signs[signs == 0] = 1.0
    comps *= signs[:, None]
    return mean, comps, np.maximum(w[order], 0.0), float(np.maximum(w, 0.0).sum())


class GPUPCA:
    """tasks/clustering_gpu.py:201-277 (cuml.decomposition.PCA -> the GPU library; float n_components in (0, 1) selects
    the smallest number of components explaining that share of the variance, as scikit-learn does)."""

    def __init__(self, n_components):
        self.n_components = n_components
        self.model = None
        self.components_ = None
        self.explained_variance_ = None
        self.explained_variance_ratio_ = None
        self.mean_ = None
        self.n_components_ = n_components
        self.using_gpu = False

    def fit_transform(self, X):
        X32 = _finite_f32(X)
        try:
            N, d = X32.shape
            kmax = min(N, d)
            if isinstance(self.n_components, float) and 0 < self.n_components < 1:
                mean, comps, ev, total = pca_fit(X32, kmax)
                k = int(np.searchsorted(np.cumsum(ev / total), self.n_components, side="right") + 1)
                k = min(k, kmax)
                comps, ev = comps[:k], ev[:k]
            else:
                k = kmax if self.n_components is None else int(self.n_components)
                if not 1 <= k <= kmax:
                    raise ValueError(f"n_components={self.n_components} must be between 1 and min(n_samples, n_features)={kmax}")
                mean, comps, ev, total = pca_fit(X32, k)
            Y = np.empty((N, k), dtype=np.float32)
            c32 = np.ascontiguousarray(comps, dtype=np.float32)
            _lib.check(_lib.load().am_pca_project(_lib.ptr(X32), N, d, _lib.ptr(mean), _lib.ptr(c32), k, _lib.ptr(Y)))
            self.mean_, self.components_ = mean, comps
            self.explained_variance_, self.explained_variance_ratio_ = ev, ev / total
            self.n_components_, self.using_gpu = k, True
            logger.debug(f"GPU PCA completed: {self.n_components_} components")
            return Y
        except Exception as e:
            if os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") != "1":
                raise
            logger.warning(f"GPU PCA failed, falling back to CPU: {e}")
        from sklearn.decomposition import PCA
        self.model = PCA(n_components=self.n_components)
        Y = self.model.fit_transform(X)
        self.components_, self.mean_ = self.model.components_, self.model.mean_
        self.explained_variance_ratio_ = self.model.explained_variance_ratio_
        self.n_components_, self.using_gpu = self.model.n_components_, False
        return Y

    def fit(self, X):
        self.fit_transform(X)
        return self

    def transform(self, X):
        if self.components_ is None:
            raise ValueError("Model must be fitted before transform")
        if not self.using_gpu:
            return self.model.transform(X)
        X32 = _finite_f32(X)
        Y = np.empty((X32.shape[0], self.n_components_), dtype=np.float32)
        m64 = np.ascontiguousarray(self.mean_, dtype=np.float64)
        c32 = np.ascontiguousarray(self.components_, dtype=np.float32)
        _lib.check(_lib.load().am_pca_project(_lib.ptr(X32), X32.shape[0], X32.shape[1], _lib.ptr(m64), _lib.ptr(c32),
                                              int(self.n_components_), _lib.ptr(Y)))
        return Y

    def inverse_transform(self, X):
        if self.components_ is None:
            raise ValueError("Model must be fitted before inverse_transform")
        if not self.using_gpu:
            return self.model.inverse_transform(X)
        return (np.asarray(X, dtype=np.float64) @ self.components_ + self.mean_).astype(np.float32)


# Chebyshev filter of the spectral eigensolver: a degree is chosen so that the filter amplifies by at most _CHEB_AMP
# (the Gram matrix of the filtered block then has a condition number of about _CHEB_AMP^2, far from float64's limit),
# and never above _CHEB_MAX_DEGREE SpMMs per outer iteration.
_CHEB_AMP = 1e4
_CHEB_MAX_DEGREE = 200


def _spectral_block(n_components, N):
    """b: the wanted vectors + a guard of half as many (at least 16), rounded up to whole 32-column warps (the padding
    is computed anyway).  The guard vectors widen the gap the filter works against: the convergence rate of the k-th
    pair is set by lambda_k against lambda_{b+1}, not lambda_{k+1}."""
    return min(N, -(-(n_components + max(16, n_components // 2)) // 32) * 32)


def _cheb_degree(cut):
    t0 = (3.0 - cut) / (1.0 + cut)                  # where x = 1 lands once [-1, cut] is mapped onto [-1, 1]
    return int(np.clip(np.floor(np.arccosh(_CHEB_AMP) / np.arccosh(t0)), 1, _CHEB_MAX_DEGREE))


def _rayleigh_ritz(G, H):
    """Ritz pairs of S in the span of V from G = V^T V and H = V^T S V: theta descending, Q with Q^T G Q = I.  G is
    Jacobi-scaled and whitened through its eigendecomposition (not one Cholesky factor), which stays accurate when a
    strong filter has left G ill-conditioned."""
    G = 0.5 * (G + G.T)
    H = 0.5 * (H + H.T)
    s = np.sqrt(np.diag(G))
    if not np.all(s > 0):
        raise RuntimeError("spectral eigensolver: a block vector vanished")
    Gs, Hs = G / np.outer(s, s), H / np.outer(s, s)
    mu, U = np.linalg.eigh(Gs)
    if mu[0] <= mu[-1] * 1e-14:
        raise RuntimeError(f"spectral eigensolver: the block lost rank (Gram eigenvalues {mu[0]:.3g} .. {mu[-1]:.3g})")
    B = U / np.sqrt(mu)
    T = B.T @ Hs @ B
    th, Z = np.linalg.eigh(0.5 * (T + T.T))
    th, Z = th[::-1], Z[:, ::-1]
    return th.copy(), np.ascontiguousarray((B @ Z) / s[:, None])


def spectral_embedding(X, n_components, n_neighbors=10, seed=0, tol=1e-8, max_iter=300, details=None):
    """-> (embedding f64[N, n_components], eigenvalues of L_sym ascending) with sklearn.manifold.spectral_embedding's
    meaning for affinity='nearest_neighbors' as SpectralClustering builds it (0.5 (C + C^T) of
    kneighbors_graph(include_self=True), normed Laplacian, drop_first=False): the eigenvectors of the smallest
    eigenvalues of L_sym = I - D^-1/2 W D^-1/2, each divided by sqrt(deg) and sign-flipped so that its largest-magnitude
    entry is positive.

    Chebyshev-filtered subspace iteration on S = I - L_sym (csrc/spectral.cu): filter the block, Rayleigh-Ritz on the
    host, rotate, repeat until every wanted Ritz pair has ||S u - theta u|| <= tol with ||u|| = 1 (measured on the
    device).  RuntimeError after max_iter outer iterations: unconverged vectors are never returned.  details (a dict,
    optional) receives the graph (affinity: W as a scipy CSR matrix without diagonal; dd = sqrt(deg)), the final
    residuals and the stage counts and times."""
    X = _check_spectral_input(X)
    N, d = X.shape
    k = int(n_components)
    if not 1 <= k <= N:
        raise ValueError(f"n_components={n_components} must be between 1 and n_samples={N}")
    if not 2 <= int(n_neighbors) <= N:
        raise ValueError(f"n_neighbors={n_neighbors} must be between 2 and n_samples={N}")
    lib = _lib.load()
    b = _spectral_block(k, N)
    plan = C.c_void_p()
    _lib.check(lib.am_spectral_plan_create(_lib.ptr(X), N, d, int(n_neighbors), b, int(seed) & 0xFFFFFFFFFFFFFFFF,
                                           C.byref(plan)))
    try:
        t0 = time.perf_counter()
        emb, thk, res, it = _solve_plan(lib, plan, N, b, k, tol, max_iter)
        eig_s = time.perf_counter() - t0
        if details is not None:
            nnz, blk, n_spmm = C.c_int64(0), C.c_int(0), C.c_int64(0)
            knn_ms, graph_ms = C.c_float(0), C.c_float(0)
            _lib.check(lib.am_spectral_plan_info(plan, C.byref(nnz), C.byref(blk), C.byref(n_spmm), C.byref(knn_ms),
                                                 C.byref(graph_ms)))
            details.update(block=int(blk.value), nnz=int(nnz.value), n_spmm=int(n_spmm.value), outer_iterations=it,
                           knn_ms=float(knn_ms.value), graph_ms=float(graph_ms.value), eigensolver_ms=1e3 * eig_s,
                           residuals=res.copy())
            details["affinity"], details["dd"] = _spectral_graph(lib, plan, N, int(nnz.value))
    finally:
        lib.am_spectral_plan_free(plan)
    return _sign_flip(emb), 1.0 - thk


def spectral_embedding_csr(W, n_components, seed=0, tol=1e-8, max_iter=300, details=None):
    """spectral_embedding's eigensolver on a given graph: W a symmetric scipy sparse matrix with positive weights and
    no empty row (float64 on the device).  -> (embedding f64[N, n_components], eigenvalues of L_sym ascending), the
    embedding divided by sqrt(deg) and sign-flipped as spectral_embedding's.  details (optional) receives the outer
    iterations, the residuals and the solver time."""
    import scipy.sparse as sp
    W = sp.csr_matrix(W, dtype=np.float64)
    W.sort_indices()
    N = W.shape[0]
    k = int(n_components)
    if W.shape != (N, N) or not 1 <= k <= N:
        raise ValueError(f"need a square graph and 1 <= n_components <= N (got {W.shape}, {n_components})")
    indptr = np.ascontiguousarray(W.indptr, dtype=np.int64)
    indices = np.ascontiguousarray(W.indices, dtype=np.int32)
    data = np.ascontiguousarray(W.data, dtype=np.float64)
    lib = _lib.load()
    b = _spectral_block(k, N)
    plan = C.c_void_p()
    _lib.check(lib.am_spectral_plan_create_csr(_lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data), N, b,
                                               int(seed) & 0xFFFFFFFFFFFFFFFF, C.byref(plan)))
    try:
        t0 = time.perf_counter()
        emb, thk, res, it = _solve_plan(lib, plan, N, b, k, tol, max_iter)
        if details is not None:
            details.update(block=b, outer_iterations=it, residuals=res.copy(),
                           eigensolver_ms=1e3 * (time.perf_counter() - t0))
    finally:
        lib.am_spectral_plan_free(plan)
    return _sign_flip(emb), 1.0 - thk


def _solve_plan(lib, plan, N, b, k, tol, max_iter):
    """The outer loop shared by both plan kinds: filter, Rayleigh-Ritz on the host, rotate, until every wanted Ritz
    pair has a residual <= tol.  -> (V Q / dd f64[N, k], theta descending f64[k], residuals, outer iterations)"""
    G, H = np.empty((b, b)), np.empty((b, b))
    res = np.full(k, np.inf)
    Q, cut, it = None, None, 0
    while True:
        if it == max_iter:
            raise RuntimeError(f"spectral eigensolver did not converge in {max_iter} iterations "
                               f"(largest residual {res.max():.3g} > tol {tol:g})")
        degree = 0 if cut is None else _cheb_degree(cut)
        _lib.check(lib.am_spectral_plan_iterate(plan, None if Q is None else _lib.ptr(Q), degree,
                                                0.0 if cut is None else cut, _lib.ptr(G), _lib.ptr(H)))
        it += 1
        theta, Q = _rayleigh_ritz(G, H)
        Qk, thk = np.ascontiguousarray(Q[:, :k]), np.ascontiguousarray(theta[:k])
        _lib.check(lib.am_spectral_plan_residuals(plan, _lib.ptr(Qk), _lib.ptr(thk), k, _lib.ptr(res), None))
        if np.all(res <= tol):
            break
        cut = float(np.clip(theta[-1], -1.0 + 1e-12, 1.0 - 1e-12))   # damp everything below the block
    emb = np.empty((N, k), dtype=np.float64)
    _lib.check(lib.am_spectral_plan_embed(plan, _lib.ptr(Qk), k, _lib.ptr(emb)))
    return emb, thk, res, it


def _sign_flip(emb):
    """sklearn.utils.extmath._deterministic_vector_sign_flip on the (n_components, N) layout"""
    top = np.argmax(np.abs(emb), axis=0)
    signs = np.sign(emb[top, np.arange(emb.shape[1])])
    signs[signs == 0] = 1.0
    emb *= signs[None, :]
    return emb


def spectral_graph(X, n_neighbors=10):
    """-> (W, dd): the affinity graph spectral_embedding works on, built on the device -- W = 0.5 (C + C^T) of
    kneighbors_graph(X, n_neighbors, include_self=True) without its diagonal, as a scipy CSR matrix (float32 values 0.5
    or 1, sorted column indices) -- and dd = sqrt(row sums of W), float64."""
    X = _check_spectral_input(X)
    N, d = X.shape
    if not 2 <= int(n_neighbors) <= N:
        raise ValueError(f"n_neighbors={n_neighbors} must be between 2 and n_samples={N}")
    lib = _lib.load()
    plan = C.c_void_p()
    _lib.check(lib.am_spectral_plan_create(_lib.ptr(X), N, d, int(n_neighbors), 1, 0, C.byref(plan)))
    try:
        nnz = C.c_int64(0)
        _lib.check(lib.am_spectral_plan_info(plan, C.byref(nnz), None, None, None, None))
        return _spectral_graph(lib, plan, N, int(nnz.value))
    finally:
        lib.am_spectral_plan_free(plan)


def _spectral_graph(lib, plan, N, nnz):
    import scipy.sparse as sp
    indptr, indices = np.empty(N + 1, np.int64), np.empty(max(nnz, 1), np.int32)
    data, dd = np.empty(max(nnz, 1), np.float32), np.empty(N, np.float64)
    _lib.check(lib.am_spectral_plan_graph(plan, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data), _lib.ptr(dd)))
    return sp.csr_matrix((data[:nnz], indices[:nnz], indptr), shape=(N, N)), dd


def _check_spectral_input(X):
    X32 = _finite_f32(X)
    if X32.shape[0] < 2 or X32.shape[1] < 1:
        raise ValueError(f"Found array with shape {X32.shape}: need at least 2 samples and 1 feature")
    return X32


class GPUSpectralClustering:
    """tasks/clustering_gpu.py:312-335 (sklearn.cluster.SpectralClustering there) on the device: the k-NN affinity
    graph and the Laplacian eigenvectors come from spectral_embedding, the labels from kmeans_fit on the embedding with
    n_init restarts.  Sets labels_ and using_gpu.  It sets no cluster_centers_ / means_, so the clustering task takes
    the per-label means of the data as the centres (clustering_helper.py:320-333), as it does for scikit-learn's
    class."""

    def __init__(self, n_clusters, assign_labels="kmeans", affinity="nearest_neighbors", n_neighbors=10,
                 random_state=None, n_init=10, verbose=False):
        self.n_clusters = n_clusters
        self.assign_labels = assign_labels
        self.affinity = affinity
        self.n_neighbors = n_neighbors
        self.random_state = random_state
        self.n_init = n_init
        self.verbose = verbose
        self.model = None
        self.labels_ = None
        self.using_gpu = False

    def _validate(self, X):
        if self.affinity != "nearest_neighbors":
            raise ValueError(f"affinity={self.affinity!r} is not supported on the GPU (only 'nearest_neighbors')")
        if self.assign_labels != "kmeans":
            raise ValueError(f"assign_labels={self.assign_labels!r} is not supported on the GPU (only 'kmeans')")
        X = _check_spectral_input(X)
        N = X.shape[0]
        if not 2 <= int(self.n_clusters) <= N - 1:
            raise ValueError(f"n_clusters={self.n_clusters} must be between 2 and n_samples - 1 = {N - 1}")
        if not 2 <= int(self.n_neighbors) <= N:
            raise ValueError(f"n_neighbors={self.n_neighbors} must be between 2 and n_samples = {N}")
        return X

    def fit_predict(self, X):
        X32 = self._validate(X)
        try:
            seed = 0 if self.random_state is None else int(self.random_state)
            emb, _ = spectral_embedding(X32, int(self.n_clusters), n_neighbors=int(self.n_neighbors), seed=seed)
            _, labels, _, _ = kmeans_fit(emb.astype(np.float32), int(self.n_clusters), n_init=int(self.n_init),
                                         seed=seed)
            self.labels_, self.using_gpu = labels, True
            logger.debug(f"GPU SpectralClustering completed: {self.n_clusters} clusters")
            return labels
        except Exception as e:
            if os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") != "1":
                raise
            logger.warning(f"GPU SpectralClustering failed, falling back to CPU: {e}")
        from sklearn.cluster import SpectralClustering
        self.model = SpectralClustering(n_clusters=self.n_clusters, assign_labels=self.assign_labels,
                                        affinity=self.affinity, n_neighbors=self.n_neighbors,
                                        random_state=self.random_state, n_init=self.n_init, verbose=self.verbose)
        self.labels_ = self.model.fit_predict(X)
        self.using_gpu = False
        return self.labels_

    def fit(self, X):
        self.fit_predict(X)
        return self


GMM_MAX_D = 256             # AM_GMM_MAX_D
GMM_MAX_K = 512             # AM_GMM_MAX_K
GMM_MAX_COMPONENTS = 65535  # AM_GMM_MAX_COMPONENTS: n_init n_components
GMM_COVARIANCE_TYPE = "full"
GMM_COVARIANCE_TYPES = {"full": 0, "diag": 1, "tied": 2, "spherical": 3}   # AM_GMM_FULL, _DIAG, _TIED, _SPHERICAL
_ILL_DEFINED = ("Fitting the mixture model failed because some components have ill-defined empirical covariance (for "
                "instance caused by singleton or collapsed samples). Try to decrease the number of components, increase "
                "reg_covar, or scale the input data.")


@dataclass
class GmmFit:
    """One GaussianMixture fit: the best init's parameters (float64), its bounds and the labels of one more E-step.
    covariances and precisions_cholesky have scikit-learn's shapes for the fit's covariance type: full [K, d, d], tied
    [d, d], diag [K, d], spherical [K].
    With intermediates=True also kpp i32[n_init, K] (the k-means++ rows) and, per init, lower_bounds
    f64[n_init, max_iter] (NaN after its n_iter), n_iter and converged."""
    weights: np.ndarray
    means: np.ndarray
    covariances: np.ndarray
    precisions_cholesky: np.ndarray
    lower_bound: float
    lower_bounds: list
    n_iter: int
    converged: bool
    best_init: int
    labels: np.ndarray
    phase_ms: dict
    kpp: Optional[np.ndarray] = None
    init_lower_bounds: Optional[np.ndarray] = None
    init_n_iter: Optional[np.ndarray] = None
    init_converged: Optional[np.ndarray] = None


def _check_gmm_input(X, n_components):
    """X as C-contiguous float64 [N, d] with scikit-learn's ValueErrors, before any device work"""
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError(f"Expected 2D array, got {X.ndim}D array instead")
    if X.shape[0] < 2:
        raise ValueError(f"Found array with {X.shape[0]} sample(s) (shape={X.shape}) while a minimum of 2 is required.")
    X64 = np.ascontiguousarray(X, dtype=np.float64)
    if not np.isfinite(X64).all():
        raise ValueError("Input X contains NaN or infinity.")
    N, d = X64.shape
    if N < n_components:
        raise ValueError(f"Expected n_samples >= n_components but got n_components = {n_components}, n_samples = {N}")
    if d > GMM_MAX_D:
        raise ValueError(f"n_features = {d} exceeds {GMM_MAX_D}, the most the GPU mixture supports")
    return X64


def _check_gmm_params(n_components, n_init, max_iter, tol, reg_covar):
    if not (isinstance(n_components, (int, np.integer)) and n_components >= 1):
        raise ValueError(f"n_components must be an int >= 1, got {n_components!r}")
    if n_components > GMM_MAX_K:
        raise ValueError(f"n_components = {n_components} exceeds {GMM_MAX_K}, the most the GPU mixture supports")
    if not (isinstance(n_init, (int, np.integer)) and n_init >= 1):
        raise ValueError(f"n_init must be an int >= 1, got {n_init!r}")
    if n_init * n_components > GMM_MAX_COMPONENTS:
        raise ValueError(f"n_init * n_components = {n_init * n_components} exceeds {GMM_MAX_COMPONENTS}, the most the "
                         "GPU mixture supports")
    if not (isinstance(max_iter, (int, np.integer)) and max_iter >= 1):
        raise ValueError(f"max_iter must be an int >= 1, got {max_iter!r}")
    if not tol >= 0:
        raise ValueError(f"tol must be >= 0, got {tol!r}")
    if not reg_covar >= 0:
        raise ValueError(f"reg_covar must be >= 0, got {reg_covar!r}")


def gmm_fit(X, n_components, n_init=10, max_iter=100, tol=1e-3, reg_covar=1e-4, random_state=None,
            intermediates=False, covariance_type="full") -> GmmFit:
    """GaussianMixture(n_components, covariance_type, init_params='k-means++', n_init, max_iter, tol, reg_covar,
    random_state).fit_predict(X) on the device (am_gmm_fit), in float64 whatever X's dtype.  The k-means++ draws come
    from check_random_state(random_state) on the host, so the generator ends where scikit-learn's fit leaves it.
    ValueError for invalid input (before any device work) and for an ill-defined covariance; B200Error when the device
    fails."""
    if covariance_type not in GMM_COVARIANCE_TYPES:
        raise ValueError(f"covariance_type must be one of 'full', 'tied', 'diag', 'spherical', got {covariance_type!r}")
    _check_gmm_params(n_components, n_init, max_iter, tol, reg_covar)
    X = _check_gmm_input(X, int(n_components))
    N, d = X.shape
    K, n_init, max_iter = int(n_components), int(n_init), int(max_iter)
    lib = _lib.load()
    draws = np.ascontiguousarray(kpp_draws(random_state, K, n_init))
    w = np.empty(K)
    m = np.empty((K, d))
    shape = {"full": (K, d, d), "tied": (d, d), "diag": (K, d), "spherical": (K,)}[covariance_type]
    cv = np.empty(shape)
    pc = np.empty(shape)
    lbs = np.empty(max_iter)
    it, conv, best, bad = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int32(0)
    labels = np.empty(N, np.int64)
    ms = np.zeros(5, np.float32)
    kpp = np.empty((n_init, K), np.int32) if intermediates else None
    ilb = np.empty((n_init, max_iter)) if intermediates else None
    iit = np.empty(n_init, np.int32) if intermediates else None
    iconv = np.empty(n_init, np.int32) if intermediates else None
    opt = lambda a: None if a is None else _lib.ptr(a)   # noqa: E731
    outputs = (_lib.ptr(w), _lib.ptr(m), _lib.ptr(cv), _lib.ptr(pc), _lib.ptr(lbs), C.byref(it), C.byref(conv),
               C.byref(best), _lib.ptr(labels), C.byref(bad), opt(kpp), opt(ilb), opt(iit), opt(iconv), _lib.ptr(ms))
    _lib.check(lib.am_gmm_fit(_lib.ptr(X), N, d, K, GMM_COVARIANCE_TYPES[covariance_type], n_init, max_iter,
                              float(tol), float(reg_covar), _lib.ptr(draws), len(draws), *outputs))
    if bad.value:
        raise ValueError(_ILL_DEFINED)
    n = int(it.value)
    return GmmFit(weights=w, means=m, covariances=cv, precisions_cholesky=pc, lower_bound=float(lbs[n - 1]),
                  lower_bounds=[float(v) for v in lbs[:n]], n_iter=n, converged=bool(conv.value),
                  best_init=int(best.value), labels=labels,
                  phase_ms=dict(zip(("seeding", "estep", "normalise", "mstep", "cholesky"), map(float, ms))),
                  kpp=kpp, init_lower_bounds=ilb, init_n_iter=iit, init_converged=None if iconv is None else iconv > 0)


class GPUGaussianMixture:
    """tasks/clustering_gpu.py:284-309 (sklearn.mixture.GaussianMixture there) on the device through gmm_fit, for
    the covariance types in DEVICE_COVARIANCE_TYPES and init_params='k-means++'; other values are refused with
    ValueError.  max_iter and tol are scikit-learn's defaults.  The clustering task reads means_ for the centres
    (clustering_helper.py:324-325)."""

    DEVICE_COVARIANCE_TYPES = ("full",)

    def __init__(self, n_components, covariance_type="full", init_params="k-means++", n_init=10, random_state=None,
                 reg_covar=1e-4, max_iter=100, tol=1e-3):
        self.n_components = n_components
        self.covariance_type = covariance_type
        self.init_params = init_params
        self.n_init = n_init
        self.random_state = random_state
        self.reg_covar = reg_covar
        self.max_iter = max_iter
        self.tol = tol
        self.model = None
        self.means_ = None
        self.weights_ = None
        self.covariances_ = None
        self.precisions_cholesky_ = None
        self.lower_bound_ = None
        self.lower_bounds_ = None
        self.n_iter_ = None
        self.converged_ = None
        self.labels_ = None
        self.using_gpu = False

    def _validate(self, X):
        if self.covariance_type not in self.DEVICE_COVARIANCE_TYPES:
            raise ValueError(f"covariance_type={self.covariance_type!r} is not supported on the GPU (only "
                             f"{', '.join(map(repr, self.DEVICE_COVARIANCE_TYPES))})")
        if self.init_params != "k-means++":
            raise ValueError(f"init_params={self.init_params!r} is not supported on the GPU (only 'k-means++')")
        _check_gmm_params(self.n_components, self.n_init, self.max_iter, self.tol, self.reg_covar)
        return _check_gmm_input(X, int(self.n_components))

    def fit_predict(self, X):
        X64 = self._validate(X)
        rs = self.random_state
        if rs is None:
            rs = np.random.mtrand._rand
        state = rs.get_state() if isinstance(rs, np.random.RandomState) else None
        try:
            f = gmm_fit(X64, int(self.n_components), n_init=int(self.n_init), max_iter=int(self.max_iter),
                        tol=self.tol, reg_covar=self.reg_covar, random_state=rs,
                        covariance_type=self.covariance_type)
            dt = X.dtype if isinstance(X, np.ndarray) and X.dtype in (np.float32, np.float64) else np.float64
            self.weights_, self.means_ = f.weights.astype(dt), f.means.astype(dt)
            self.covariances_, self.precisions_cholesky_ = f.covariances.astype(dt), f.precisions_cholesky.astype(dt)
            self.lower_bound_, self.lower_bounds_ = f.lower_bound, f.lower_bounds
            self.n_iter_, self.converged_, self.labels_ = f.n_iter, f.converged, f.labels
            self.using_gpu = True
            if not f.converged:
                from sklearn.exceptions import ConvergenceWarning
                warnings.warn("Best performing initialization did not converge. Try different init parameters, or "
                              "increase max_iter, tol, or check for degenerate data.", ConvergenceWarning)
            logger.debug(f"GPU GaussianMixture completed: {self.n_components} components, {f.n_iter} iterations")
            return f.labels
        except _lib.B200Error as e:
            if os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") != "1":
                raise
            logger.warning(f"GPU GaussianMixture failed, falling back to CPU: {e}")
        if state is not None:
            rs.set_state(state)                     # the fallback draws what the device fit would have drawn
        from sklearn.mixture import GaussianMixture
        self.model = GaussianMixture(n_components=self.n_components, covariance_type=self.covariance_type,
                                     init_params=self.init_params, n_init=self.n_init, random_state=rs,
                                     reg_covar=self.reg_covar, max_iter=self.max_iter, tol=self.tol)
        self.labels_ = self.model.fit_predict(X)
        for n in ("means_", "weights_", "covariances_", "precisions_cholesky_", "lower_bound_", "lower_bounds_",
                  "n_iter_", "converged_"):
            setattr(self, n, getattr(self.model, n))
        self.using_gpu = False
        return self.labels_

    def fit(self, X):
        self.fit_predict(X)
        return self


class GPUGaussianMixtureAnyCovariance(GPUGaussianMixture):
    """GPUGaussianMixture for every covariance type the clustering task's GMM_COVARIANCE_TYPE may name: 'full',
    'tied', 'diag' and 'spherical' all fit on the device, and covariances_ / precisions_cholesky_ have scikit-learn's
    shapes for the type, in the input's dtype.  The generator handling, the B200_ALLOW_SKLEARN_FALLBACK path (which
    fits scikit-learn with the same type) and the ConvergenceWarning are GPUGaussianMixture's."""

    DEVICE_COVARIANCE_TYPES = ("full", "tied", "diag", "spherical")


def get_clustering_model(method, params, use_gpu=False):
    if use_gpu and method == "kmeans":
        return GPUKMeans(n_clusters=params["n_clusters"], init="k-means++", n_init=10)
    if use_gpu and method == "dbscan":
        return GPUDBSCAN(eps=params["eps"], min_samples=params["min_samples"])
    if use_gpu and method == "spectral":
        return GPUSpectralClustering(n_clusters=params["n_clusters"], assign_labels="kmeans",
                                     affinity="nearest_neighbors", n_neighbors=params.get("n_neighbors", 20),
                                     random_state=params.get("random_state"), n_init=10, verbose=False)
    if use_gpu and method == "gmm":
        return GPUGaussianMixture(n_components=params["n_components"], covariance_type=GMM_COVARIANCE_TYPE,
                                  init_params="k-means++", n_init=10, random_state=None, reg_covar=1e-4)
    from sklearn.cluster import DBSCAN, KMeans, SpectralClustering
    if method == "kmeans":
        return KMeans(n_clusters=params["n_clusters"], init="k-means++", n_init=10)
    if method == "dbscan":
        return DBSCAN(eps=params["eps"], min_samples=params["min_samples"])
    if method == "spectral":
        return SpectralClustering(n_clusters=params["n_clusters"], assign_labels="kmeans", affinity="nearest_neighbors",
                                  n_neighbors=params.get("n_neighbors", 20), random_state=params.get("random_state"),
                                  n_init=10, verbose=False)
    if method == "gmm":
        from sklearn.mixture import GaussianMixture
        return GaussianMixture(n_components=params["n_components"], covariance_type=GMM_COVARIANCE_TYPE,
                               init_params="k-means++", n_init=10, random_state=None, reg_covar=1e-4)
    raise ValueError(f"Unsupported clustering method: {method}")


def get_pca_model(n_components, use_gpu=False):
    if not use_gpu:
        from sklearn.decomposition import PCA
        return PCA(n_components=n_components)
    return GPUPCA(n_components=n_components)
