"""The artist-similarity GMMs on the GPU: tasks/artist_gmm_manager.select_optimal_gmm_components (:63-126) and
fit_artist_gmm (:129-216), which build_and_store_artist_index (:406-721) calls once per new or changed artist.

    fit_artist_gmms(row_arrays, min_components=2, max_components=10)   -> [ArtistFit, ...], the batched sweep
    select_optimal_gmm_components(embeddings, min_components=2, max_components=10)   -> K, the drop-in
    fit_artist_gmm(artist_name, track_embeddings)                       -> gmm_params dict or None, the drop-in

For every artist and every K from 1 to max_feasible, am_artist_gmm_fit (csrc/artist_gmm.cu) runs scikit-learn's
GaussianMixture(K, covariance_type='diag', max_iter=100, n_init=3, random_state=42).fit and bic in float64 on the
float32 rows, and keeps the first K with the strictly lowest BIC.  random_state=42 is an int, so every fit draws the
same prefix of MT19937(42): draw_table builds it once on the host and no generator runs on the device.  The chosen
K's fit is the sweep's own (the reference fits it a second time with the same seed, which gives the same fit).

Both drop-ins call fit_artist_gmms.  They return what the reference returns, including its failure values: None from
fit_artist_gmm for no rows, rows of different lengths, NaN or infinity, or a failed fit; select_optimal_gmm_components
returns min(min_components, max_feasible) when every K fails.  The parameters are rounded to float32, as the
reference's float32 scikit-learn run returns them.  There is no CPU fallback: without a device fit_artist_gmm logs the
error and returns None and select_optimal_gmm_components raises, unless B200_ALLOW_SKLEARN_FALLBACK=1, in which case
both call the reference's own functions, which integration.apply captured before it replaced them.
"""
from __future__ import annotations

import ctypes as C
import functools
import logging
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from . import _lib

logger = logging.getLogger(__name__)

MAX_K = 16                  # AM_ARTIST_GMM_MAX_K
MAX_D = 1024                # AM_ARTIST_GMM_MAX_D
SMEM_BYTES = 98304          # AM_ARTIST_GMM_SMEM_BYTES: an artist's rows are staged in shared memory when n d 4 <= this
GMM_N_COMPONENTS_MIN = 2
GMM_N_COMPONENTS_MAX = 10
GMM_COVARIANCE_TYPE = "diag"
GMM_MAX_ITER = 100
GMM_N_INIT = 3
GMM_TOL = 1e-3
GMM_REG_COVAR = 1e-6
GMM_SEED = 42
MIN_TRACKS_PER_ARTIST = 1
FEW_SONGS = 5               # below this, one fixed component per song
FIXED_VARIANCE = 0.01

# the reference's own functions, captured by integration.apply before it replaces them
_originals: Dict[str, object] = {}


def n_local_trials(K: int) -> int:
    return 2 + int(np.log(K))


def draws_per_init(K: int) -> int:
    return 1 + (K - 1) * n_local_trials(K)


@functools.lru_cache(maxsize=4)
def draw_table(k_max: int = MAX_K, n_init: int = GMM_N_INIT, seed: int = GMM_SEED) -> np.ndarray:
    """every double the k-means++ inits of a GaussianMixture(K <= k_max, n_init, random_state=seed).fit draw, in order"""
    t = np.random.RandomState(seed).random_sample(n_init * draws_per_init(k_max))
    t.flags.writeable = False
    return t


def max_feasible(n: int, min_components: int = GMM_N_COMPONENTS_MIN,
                 max_components: int = GMM_N_COMPONENTS_MAX) -> int:
    """the largest K select_optimal_gmm_components tries for n rows (:84-97)"""
    if n <= 5:
        mf = min(n, max_components)
    else:
        mf = max(min_components, min(max_components, n // 5))
    if mf < min_components:
        mf = min(min_components, n)
    return mf


@dataclass
class ArtistFit:
    """One artist's sweep.  k is the reference's answer; fitted is False when every K failed (k is then the
    reference's fallback) or nothing was fitted (one row).  Per K tried: bic and failed; per (K, init): lower_bound,
    n_iter, converged.  weights / means / covariances (float32) are the chosen K's fit when fitted."""
    n: int
    d: int
    k: int
    fitted: bool
    k_range: tuple
    bic: Dict[int, float] = field(default_factory=dict)
    failed: Dict[int, bool] = field(default_factory=dict)
    lower_bound: Optional[np.ndarray] = None     # f64[16, n_init], row K - 1
    n_iter: Optional[np.ndarray] = None
    converged: Optional[np.ndarray] = None
    weights: Optional[np.ndarray] = None
    means: Optional[np.ndarray] = None
    covariances: Optional[np.ndarray] = None
    kpp: Optional[np.ndarray] = None             # i32[16, n_init, 16] with intermediates=True
    labels: Optional[np.ndarray] = None          # i32[16, n_init, n] with intermediates=True


def _sweep(X_list, k_lo, k_hi, intermediates, timings=None):
    """one am_artist_gmm_fit call over artists with rows of the same width"""
    A = len(X_list)
    d = X_list[0].shape[1]
    sizes = np.array([len(x) for x in X_list], dtype=np.int64)
    offsets = np.zeros(A + 1, np.int64)
    np.cumsum(sizes, out=offsets[1:])
    rows = np.ascontiguousarray(np.concatenate(X_list), dtype=np.float32)
    lo = np.ascontiguousarray(k_lo, dtype=np.int32)
    hi = np.ascontiguousarray(k_hi, dtype=np.int32)
    draws = draw_table()
    chosen = np.zeros(A, np.int32)
    bic = np.zeros((A, MAX_K), np.float64)
    failed = np.zeros((A, MAX_K), np.uint8)
    lb = np.zeros((A, MAX_K, GMM_N_INIT), np.float64)
    n_iter = np.zeros((A, MAX_K, GMM_N_INIT), np.int32)
    conv = np.zeros((A, MAX_K, GMM_N_INIT), np.uint8)
    w = np.zeros((A, MAX_K), np.float32)
    m = np.zeros((A, MAX_K, d), np.float32)
    cv = np.zeros((A, MAX_K, d), np.float32)
    kpp = np.zeros((A, MAX_K, GMM_N_INIT, MAX_K), np.int32) if intermediates else None
    labels = np.zeros((MAX_K, GMM_N_INIT, len(rows)), np.int32) if intermediates else None
    ms = np.zeros(2, np.float32)
    lib = _lib.load()
    _lib.check(lib.am_artist_gmm_fit(
        _lib.ptr(rows), len(rows), d, _lib.ptr(offsets), A, _lib.ptr(lo), _lib.ptr(hi), GMM_N_INIT, GMM_MAX_ITER,
        GMM_TOL, GMM_REG_COVAR, _lib.ptr(draws), len(draws), _lib.ptr(chosen), _lib.ptr(bic), _lib.ptr(failed),
        _lib.ptr(lb), _lib.ptr(n_iter), _lib.ptr(conv), _lib.ptr(w), _lib.ptr(m), _lib.ptr(cv),
        _lib.ptr(kpp) if intermediates else None, _lib.ptr(labels) if intermediates else None, _lib.ptr(ms)))
    if timings is not None:
        timings["fit_ms"] = timings.get("fit_ms", 0.0) + float(ms[0])
        timings["select_ms"] = timings.get("select_ms", 0.0) + float(ms[1])
    out = []
    for a in range(A):
        K = int(chosen[a])
        ks = range(int(lo[a]), int(hi[a]) + 1)
        f = ArtistFit(n=int(sizes[a]), d=d, k=K, fitted=K > 0, k_range=(int(lo[a]), int(hi[a])),
                      bic={k: float(bic[a, k - 1]) for k in ks}, failed={k: bool(failed[a, k - 1]) for k in ks},
                      lower_bound=lb[a], n_iter=n_iter[a], converged=conv[a].astype(bool))
        if K > 0:
            f.weights, f.means, f.covariances = w[a, :K].copy(), m[a, :K].copy(), cv[a, :K].copy()
        if intermediates:
            f.kpp = kpp[a]
            f.labels = labels[:, :, offsets[a]:offsets[a + 1]]
        out.append(f)
    return out


def fit_artist_gmms(row_arrays, min_components: int = GMM_N_COMPONENTS_MIN,
                    max_components: int = GMM_N_COMPONENTS_MAX, intermediates: bool = False,
                    timings: Optional[dict] = None) -> List[ArtistFit]:
    """The BIC sweep of select_optimal_gmm_components for many artists in one device batch (one call per row
    width).  row_arrays: one [n, d] array per artist.  Raises ValueError before any device work for an empty artist,
    a K above 16, d above 1024 or a NaN / infinity; B200Error when the device fails.  An artist's result does not
    depend on the rest of the batch or its order."""
    Xs = []
    for a, r in enumerate(row_arrays):
        X = np.asarray(r)
        if X.ndim != 2 or X.shape[0] < 1 or X.shape[1] < 1:
            raise ValueError(f"artist {a}: need a non-empty [n, d] array, got shape {X.shape}")
        if X.shape[1] > MAX_D:
            raise ValueError(f"artist {a}: d = {X.shape[1]} exceeds {MAX_D}")
        X32 = np.ascontiguousarray(X, dtype=np.float32)
        if not np.isfinite(X32).all():
            raise ValueError(f"artist {a}: the rows contain NaN or infinity")
        Xs.append(X32)
    los, his, fallback = [], [], []
    for X in Xs:
        n = len(X)
        mf = max_feasible(n, min_components, max_components)
        if n == 1 or mf < 1:
            los.append(1), his.append(0), fallback.append(1)
            continue
        if mf > MAX_K:
            raise ValueError(f"K up to {mf} requested; at most {MAX_K} components are supported")
        los.append(1), his.append(mf), fallback.append(min(min_components, mf))
    res: List[Optional[ArtistFit]] = [None] * len(Xs)
    for d in sorted({X.shape[1] for X in Xs}):
        sel = [i for i, X in enumerate(Xs) if X.shape[1] == d]
        for i, f in zip(sel, _sweep([Xs[i] for i in sel], [los[i] for i in sel], [his[i] for i in sel],
                                    intermediates, timings)):
            if not f.fitted:
                f.k = fallback[i]
            res[i] = f
    return res


def _fallback_allowed() -> bool:
    return os.environ.get("B200_ALLOW_SKLEARN_FALLBACK", "0") == "1" and bool(_originals)


def select_optimal_gmm_components(embeddings: np.ndarray, min_components: int = GMM_N_COMPONENTS_MIN,
                                  max_components: int = GMM_N_COMPONENTS_MAX) -> int:
    """The reference's select_optimal_gmm_components on the GPU: the K with the lowest BIC."""
    n = len(embeddings)
    if n == 1:
        return 1
    mf = max_feasible(n, min_components, max_components)
    if mf < 1:
        return 1
    X = np.asarray(embeddings)
    if not np.isfinite(X).all():      # every fit raises in the reference, which then keeps its starting value
        return min(min_components, mf)
    try:
        return fit_artist_gmms([X], min_components, max_components)[0].k
    except _lib.B200Error:
        if _fallback_allowed():
            return _originals["select_optimal_gmm_components"](embeddings, min_components, max_components)
        raise


def _few_songs(all_embeddings: np.ndarray, n_tracks: int) -> dict:
    n_samples, n_features = all_embeddings.shape
    return {
        "weights": [1.0 / n_samples] * n_samples,
        "means": all_embeddings.tolist(),
        "covariances": [[FIXED_VARIANCE] * n_features] * n_samples,
        "n_components": n_samples,
        "covariance_type": GMM_COVARIANCE_TYPE,
        "n_features": n_features,
        "n_tracks": n_samples,
        "is_few_songs": True,
    }


def fit_artist_gmm(artist_name: str, track_embeddings) -> Optional[dict]:
    """The reference's fit_artist_gmm on the GPU: the gmm_params dict build_and_store_artist_index stores, or None."""
    if len(track_embeddings) < MIN_TRACKS_PER_ARTIST:
        logger.warning(f"Artist '{artist_name}' has only {len(track_embeddings)} tracks, "
                       f"need at least {MIN_TRACKS_PER_ARTIST}")
        return None
    try:
        all_embeddings = np.vstack(track_embeddings)
        n_samples, n_features = all_embeddings.shape
        if n_samples < FEW_SONGS:
            return _few_songs(all_embeddings, len(track_embeddings))
        if not np.isfinite(all_embeddings).all():
            raise ValueError("Input contains NaN or infinity.")
        f = fit_artist_gmms([all_embeddings])[0]
        if not f.fitted:
            raise ValueError(f"every GaussianMixture fit failed for {n_samples} rows")
        return {
            "weights": f.weights.tolist(),
            "means": f.means.tolist(),
            "covariances": f.covariances.tolist(),
            "n_components": f.k,
            "covariance_type": GMM_COVARIANCE_TYPE,
            "n_features": n_features,
            "n_tracks": len(track_embeddings),
            "is_few_songs": False,
        }
    except _lib.B200Error as e:
        if _fallback_allowed():
            return _originals["fit_artist_gmm"](artist_name, track_embeddings)
        logger.error(f"Failed to fit GMM for artist '{artist_name}': {e}")
        return None
    except Exception as e:
        logger.error(f"Failed to fit GMM for artist '{artist_name}': {e}")
        return None


def capture_originals(module) -> None:
    """remember the reference module's own functions (once: a second apply must not capture the drop-ins)"""
    for name in ("fit_artist_gmm", "select_optimal_gmm_components"):
        fn = getattr(module, name, None)
        if fn is not None and getattr(fn, "__module__", "") != __name__:
            _originals[name] = fn
