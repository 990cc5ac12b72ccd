"""Mirror of ``tasks/clustering_gpu.py`` (KMeans rows of SURVEY 8(a)) on the GPU library.

    check_gpu_available()                      tasks/clustering_gpu.py:26-79
    GPUKMeans(n_clusters, init, n_init, random_state).fit_predict(X)   :82-148
        -> labels; sets cluster_centers_, labels_, using_gpu, inertia_, n_iter_
    get_clustering_model('kmeans', {'n_clusters': k}, use_gpu)          :338-404

cuML is replaced by am_kmeans_fit (k-means++ D^2 seeding, n_init restarts, Lloyd with sklearn's
tol rule).  The reference silently falls back to sklearn when the GPU path raises (:130-148);
here that fallback exists only when ``B200_ALLOW_SKLEARN_FALLBACK=1`` (default: fail loudly,
so a missing CUDA library can never masquerade as the GPU path).

    GPUDBSCAN(eps, min_samples).fit_predict(X)                         :151-199  -> am_dbscan (exact, sklearn's labels)
    GPUPCA(n_components).fit_transform(X) / inverse_transform(X)      :201-277  -> am_pca_moments + LAPACK eigh on the
        host + am_pca_project; sets components_, explained_variance_ratio_, n_components_ like sklearn's PCA
    get_pca_model(n_components, use_gpu)                               :407-421

GMM / spectral clustering have no GPU implementation in the reference either (:280-335, scikit-learn always).
"""
from __future__ import annotations

import ctypes as C
import logging
import os

import numpy as np

from . import _lib

logger = logging.getLogger("tasks.clustering_gpu")


def check_gpu_available() -> bool:
    try:
        return _lib.load().am_init(-1) == _lib.AM_OK
    except Exception as e:
        logger.info(f"GPU library unavailable: {e}")
        return False


def kmeans_fit(X, k, n_init=10, max_iter=300, tol=1e-4, seed=0, init_centers=None):
    """-> (centers f32[k,d], labels i32[N], inertia, n_iter) via am_kmeans_fit."""
    lib = _lib.load()
    X = np.ascontiguousarray(X, dtype=np.float32)
    if X.ndim != 2:
        raise ValueError("X must be [N, d]")
    N, d = X.shape
    centers = np.empty((k, d), dtype=np.float32)
    labels = np.empty((N,), dtype=np.int32)
    inertia, n_iter = C.c_float(0), C.c_int(0)
    init = None
    if init_centers is not None:
        init = np.ascontiguousarray(init_centers, dtype=np.float32)
        if init.shape != (k, d):
            raise ValueError(f"init_centers must be ({k}, {d})")
    _lib.check(lib.am_kmeans_fit(_lib.ptr(X), N, d, int(k), int(n_init), int(max_iter), float(tol),
                                 int(seed) & 0xFFFFFFFFFFFFFFFF, None if init is None else _lib.ptr(init),
                                 _lib.ptr(centers), _lib.ptr(labels), C.byref(inertia), C.byref(n_iter)))
    return centers, labels, float(inertia.value), int(n_iter.value)


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
        try:
            X = np.ascontiguousarray(X, dtype=np.float32)
            if X.ndim != 2:
                raise ValueError("X must be [N, d]")
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
        try:
            X32 = np.ascontiguousarray(X, dtype=np.float32)
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
            m32, c32 = mean.astype(np.float32), np.ascontiguousarray(comps, dtype=np.float32)
            _lib.check(_lib.load().am_pca_project(_lib.ptr(X32), N, d, _lib.ptr(m32), _lib.ptr(c32), k, _lib.ptr(Y)))
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
        X32 = np.ascontiguousarray(X, dtype=np.float32)
        Y = np.empty((X32.shape[0], self.n_components_), dtype=np.float32)
        m32, c32 = self.mean_.astype(np.float32), np.ascontiguousarray(self.components_, dtype=np.float32)
        _lib.check(_lib.load().am_pca_project(_lib.ptr(X32), X32.shape[0], X32.shape[1], _lib.ptr(m32), _lib.ptr(c32),
                                              int(self.n_components_), _lib.ptr(Y)))
        return Y

    def inverse_transform(self, X):
        if self.components_ is None:
            raise ValueError("Model must be fitted before inverse_transform")
        if not self.using_gpu:
            return self.model.inverse_transform(X)
        return (np.asarray(X, dtype=np.float64) @ self.components_ + self.mean_).astype(np.float32)


def get_clustering_model(method, params, use_gpu=False):
    if use_gpu and method == "kmeans":
        return GPUKMeans(n_clusters=params["n_clusters"], init="k-means++", n_init=10)
    if use_gpu and method == "dbscan":
        return GPUDBSCAN(eps=params["eps"], min_samples=params["min_samples"])
    from sklearn.cluster import DBSCAN, KMeans
    if method == "kmeans":
        return KMeans(n_clusters=params["n_clusters"], init="k-means++", n_init=10)
    if method == "dbscan":
        return DBSCAN(eps=params["eps"], min_samples=params["min_samples"])
    raise ValueError(f"Unsupported clustering method: {method}")


def get_pca_model(n_components, use_gpu=False):
    if not use_gpu:
        from sklearn.decomposition import PCA
        return PCA(n_components=n_components)
    return GPUPCA(n_components=n_components)
