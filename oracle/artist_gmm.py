"""Oracle: the artist-similarity GMM sweep, float64 numpy.  TEST INFRASTRUCTURE ONLY.

Restates tasks/artist_gmm_manager.select_optimal_gmm_components (:63-126): for K = 1 .. max_feasible,
GaussianMixture(K, covariance_type='diag', max_iter=100, n_init=3, random_state=42).fit(X), then gmm.bic(X); the
first K with the strictly lowest BIC wins.  Every step follows scikit-learn 1.9.0 (the reference pins 1.8.0; the
code paths used here are the same in both):

  draws        random_state=42 is an int, so every fit starts a fresh RandomState(42) and its n_init k-means++
               inits consume it in turn: 1 + (K - 1) (2 + floor(ln K)) doubles each.  One table, the first
               n_init * draws_per_init(K_max) doubles of MT19937(42), serves every artist and every K.
  k-means++    on X centred by its column mean (KMeans.fit, dense input).  The first centre is
               choice(n, p=uniform) = searchsorted(cumsum(full(n, 1/n)) / last, u, 'right'); every further centre
               samples 2 + floor(ln K) candidates at searchsorted(cumsum(closest_dist_sq), u * pot) clipped to
               n - 1, and keeps the one with the lowest potential (ties: the first).  Squared distances are
               (-2 c.x + |c|^2) + |x|^2 clipped at 0.
  Lloyd        labels = argmin_j |c_j|^2 - 2 x.c_j (ties: the lowest j); empty clusters take the point farthest
               from its centre; centres = sums * (1 / count); stop when the labels repeat (strict) or when
               sum |dc|^2 <= 1e-4 mean(var(X)); max 300 iterations; not strict: one more assignment.
  EM           one-hot labels -> first M-step (nk = sum resp + 10 eps, weights = nk / n); every M-step fails (the
               whole K) when a covariance is <= 0; the E-step's log-density
               -0.5 (d log 2 pi + sum mu^2 p - 2 x.(mu p) + x^2.p) + sum log sqrt(p) + log w and scikit-learn's
               logsumexp (the maxima split off, log1p of the rest); the lower bound is the mean log-normaliser of
               the E-step before the M-step; |change| < 1e-3 stops; at most 100 iterations.  The best init is the
               first one whose bound is strictly greater.
  BIC          -2 n score(X) + (2 K d + K - 1) ln n, score with the best init's final parameters.

Unverified against scikit-learn: which point an empty cluster takes when two or more clusters are empty at once
(scikit-learn's argpartition order); here the farthest points in decreasing distance, ties to the lowest index.
Every fit also returns the smallest margin of each discrete decision it took, so a test can show that its data are
not on a knife edge.
"""
from __future__ import annotations

import math

import numpy as np

N_INIT = 3
MAX_ITER = 100
TOL = 1e-3
REG_COVAR = 1e-6
SEED = 42
KM_MAX_ITER = 300
KM_TOL = 1e-4
EPS = float(np.finfo(np.float64).eps)
LOG_2PI = math.log(2.0 * math.pi)


def n_local_trials(K: int) -> int:
    return 2 + int(np.log(K))


def draws_per_init(K: int) -> int:
    return 1 + (K - 1) * n_local_trials(K)


def draw_table(k_max: int, n_init: int = N_INIT, seed: int = SEED) -> np.ndarray:
    """The doubles a GaussianMixture(K <= k_max, n_init, random_state=seed).fit draws, in order; init i of a K-fit
    uses table[i * draws_per_init(K):(i + 1) * draws_per_init(K)]"""
    return np.random.RandomState(seed).random_sample(n_init * draws_per_init(k_max))


def max_feasible(n: int, min_components: int = 2, max_components: int = 10) -> int:
    """the largest K the reference tries (select_optimal_gmm_components :84-97); 0 means none"""
    if n <= 5:
        mf = min(n, max_components)
    else:
        mf = max(min_components, min(max_components, n // 5))
    if mf < min_components:
        mf = min(min_components, n)
    return mf


def _logsumexp(a):
    """scikit-learn 1.9's _logsumexp over axis 1: the maxima are split off and the rest enters through log1p"""
    amax = a.max(1, keepdims=True)
    is_max = a == amax
    m = is_max.sum(1, keepdims=True).astype(np.float64)
    rest = np.where(is_max, -np.inf, a)
    shift = np.where(np.isfinite(amax), amax, 0.0)
    s = np.exp(rest - shift).sum(1, keepdims=True)
    s = np.where(s == 0, s, s / m)
    return (np.log1p(s) + np.log(m) + amax)[:, 0]


class Margins:
    """the smallest distance of each discrete decision from flipping, each scaled to its own quantity"""

    KEYS = ("first_centre", "candidate", "best_candidate", "lloyd_label", "lloyd_tol", "em_tol", "best_init",
            "relocation", "choice_of_k")

    def __init__(self):
        self.m = {k: np.inf for k in self.KEYS}

    def add(self, key, v):
        self.m[key] = min(self.m[key], float(v))

    def merge(self, other):
        for k, v in other.m.items():
            self.add(k, v)


def first_centre(n: int, u: float, mg: Margins | None = None) -> int:
    cdf = np.cumsum(np.full(n, 1.0 / n))
    cdf /= cdf[-1]
    i = int(np.searchsorted(cdf, u, side="right"))
    if mg is not None:
        mg.add("first_centre", np.abs(cdf - u).min())
    return i


def _sqdist(C, X, xsq):
    d = -2.0 * (C @ X.T)
    d += np.einsum("ij,ij->i", C, C)[:, None]
    d += xsq[None, :]
    return np.maximum(d, 0.0)


def kmeans_plusplus(Xc, xsq, K, u, mg: Margins | None = None):
    """indices of the K initial centres of centred rows Xc from one init's draws u"""
    n = len(Xc)
    L = n_local_trials(K)
    idx = [first_centre(n, u[0], mg)]
    closest = _sqdist(Xc[idx[0]][None, :], Xc, xsq)[0]
    pot = closest.sum()
    pos = 1
    for _ in range(1, K):
        rv = u[pos:pos + L] * pot
        pos += L
        cs = np.cumsum(closest)
        cand = np.minimum(np.searchsorted(cs, rv), n - 1)
        if mg is not None and pot > 0:
            mg.add("candidate", min(np.abs(cs - r).min() for r in rv) / pot)
        D = np.minimum(closest[None, :], _sqdist(Xc[cand], Xc, xsq))
        pots = D.sum(1)
        b = int(np.argmin(pots))
        if mg is not None:
            # a candidate that is a copy of the best row has the same potential to the bit: not a decision
            other = pots[np.any(Xc[cand] != Xc[cand[b]], axis=1)]
            if len(other):
                mg.add("best_candidate", (other.min() - pots[b]) / max(abs(pots[b]), 1e-300))
        pot = pots[b]
        closest = D[b]
        idx.append(int(cand[b]))
    return np.array(idx, dtype=np.int64)


def _assign(Xc, C, mg: Margins | None):
    cn = (C * C).sum(1)
    D = cn[None, :] - 2.0 * (Xc @ C.T)
    lab = D.argmin(1).astype(np.int32)
    if mg is not None and C.shape[0] > 1:
        s = np.sort(D, 1)
        gap = (s[:, 1] - s[:, 0]) / (np.abs(D).max(1) + 1e-300)
        if len(np.unique(C, axis=0)) < len(C):
            gap = gap[gap > 0]      # identical centres tie exactly, and every order of them gives the same labels
        if len(gap):
            mg.add("lloyd_label", gap.min())
    return lab


def lloyd(Xc, C0, tol, mg: Margins | None = None):
    """labels and iteration count of scikit-learn's dense Lloyd from centres C0"""
    n, K = len(Xc), len(C0)
    C = np.array(C0, dtype=np.float64)
    labels_old = np.full(n, -1, np.int32)
    strict = False
    it = 0
    for it in range(KM_MAX_ITER):
        labels = _assign(Xc, C, mg)
        sums = np.zeros_like(C)
        np.add.at(sums, labels, Xc)
        w = np.bincount(labels, minlength=K).astype(np.float64)
        empty = np.flatnonzero(w == 0)
        if len(empty):
            dist = ((Xc - C[labels]) ** 2).sum(1)
            far = np.argsort(-dist, kind="stable")[:len(empty)]
            if mg is not None and len(dist) > len(empty):
                s = np.sort(dist)[::-1]
                if s[0] > 0:
                    mg.add("relocation", (s[len(empty) - 1] - s[len(empty)]) / s[0])
            for e, f in zip(empty, far):
                old = labels[f]
                sums[old] -= Xc[f]
                sums[e] = Xc[f]
                w[e] = 1.0
                w[old] -= 1.0
        Cn = sums.copy()          # a cluster left with no weight keeps its sums, as scikit-learn's _average_centers
        nz = w > 0
        Cn[nz] *= (1.0 / w[nz])[:, None]
        shift = np.sqrt(((Cn - C) ** 2).sum(1))
        C = Cn
        if np.array_equal(labels, labels_old):
            strict = True
            break
        tot = (shift ** 2).sum()
        if mg is not None and tol > 0:
            mg.add("lloyd_tol", abs(tot - tol) / tol)
        if tot <= tol:
            break
        labels_old = labels
    if not strict:
        labels = _assign(Xc, C, mg)
    return labels, it + 1


def m_step(X, resp, reg_covar=REG_COVAR):
    nk = resp.sum(0) + 10.0 * EPS
    means = (resp.T @ X) / nk[:, None]
    cov = (resp.T @ (X * X)) / nk[:, None] - means ** 2 + reg_covar
    return nk, means, cov


def weighted_log_prob(X, weights, means, pc):
    prec = pc ** 2
    log_det = np.log(pc).sum(1)
    lp = (means ** 2 * prec).sum(1) - 2.0 * (X @ (means * prec).T) + (X ** 2) @ prec.T
    return -0.5 * (X.shape[1] * LOG_2PI + lp) + log_det + np.log(weights)


class FitFailed(ValueError):
    """a covariance <= 0 after an M-step: scikit-learn's ValueError, the reference skips the K"""


def em(X, labels, K, max_iter=MAX_ITER, tol=TOL, reg_covar=REG_COVAR, mg: Margins | None = None):
    n = len(X)
    resp = np.zeros((n, K))
    resp[np.arange(n), labels] = 1.0
    nk, means, cov = m_step(X, resp, reg_covar)
    weights = nk / n
    if np.any(cov <= 0):
        raise FitFailed("covariance <= 0 after the initial M-step")
    pc = 1.0 / np.sqrt(cov)
    lb = -np.inf
    converged = False
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        prev = lb
        wlp = weighted_log_prob(X, weights, means, pc)
        norm = _logsumexp(wlp)
        resp = np.exp(wlp - norm[:, None])
        nk, means, cov = m_step(X, resp, reg_covar)
        weights = nk / nk.sum()
        if np.any(cov <= 0):
            raise FitFailed(f"covariance <= 0 after M-step {n_iter}")
        pc = 1.0 / np.sqrt(cov)
        lb = norm.mean()
        change = lb - prev
        if mg is not None and np.isfinite(change):
            mg.add("em_tol", abs(abs(change) - tol) / tol)
        if abs(change) < tol:
            converged = True
            break
    return dict(weights=weights, means=means, covariances=cov, pc=pc, lower_bound=float(lb), n_iter=n_iter,
                converged=converged)


def score(X, weights, means, pc) -> float:
    return float(_logsumexp(weighted_log_prob(X, weights, means, pc)).mean())


def same_partition(a, b) -> bool:
    """labels a and b group the rows the same way, whatever the cluster numbers"""
    pairs = set(zip(np.asarray(a).tolist(), np.asarray(b).tolist()))
    return len(pairs) == len(set(np.asarray(a).tolist())) == len(set(np.asarray(b).tolist()))


def fit_k(X, K, draws, n_init=N_INIT, max_iter=MAX_ITER, tol=TOL, reg_covar=REG_COVAR, mg: Margins | None = None):
    """GaussianMixture(K, 'diag', max_iter, n_init, random_state=42).fit(X) and its bic(X), with the intermediates.
    Returns a dict; 'failed' is True when any init raised (the reference then skips this K)."""
    X = np.asarray(X, dtype=np.float64)
    n, d = X.shape
    out = dict(K=K, failed=False, kpp=[], labels=[], lloyd_iter=[], lower_bound=[], n_iter=[], converged=[])
    if n < K:
        out["failed"] = True
        return out
    Xc = X - X.mean(0)
    xsq = np.einsum("ij,ij->i", Xc, Xc)
    km_tol = float(np.var(X, axis=0).mean() * KM_TOL)
    D = draws_per_init(K)
    fits = []
    for i in range(n_init):
        kpp = kmeans_plusplus(Xc, xsq, K, draws[i * D:(i + 1) * D], mg)
        labels, lit = lloyd(Xc, Xc[kpp], km_tol, mg)
        out["kpp"].append(kpp)
        out["labels"].append(labels)
        out["lloyd_iter"].append(lit)
        try:
            f = em(X, labels, K, max_iter, tol, reg_covar, mg)
        except FitFailed:
            out["failed"] = True
            return out
        fits.append(f)
        out["lower_bound"].append(f["lower_bound"])
        out["n_iter"].append(f["n_iter"])
        out["converged"].append(f["converged"])
    best, best_lb = 0, -np.inf
    for i, f in enumerate(fits):
        if f["lower_bound"] > best_lb or best_lb == -np.inf:
            best, best_lb = i, f["lower_bound"]
    if mg is not None:
        # inits that start EM from the same partition (up to the order of the clusters) reach the same mixture:
        # which of them is kept is not a decision
        lbs = np.array(out["lower_bound"])
        for i in range(n_init):
            if not same_partition(out["labels"][i], out["labels"][best]):
                mg.add("best_init", abs(lbs[i] - lbs[best]) / max(abs(lbs[best]), 1e-300))
    f = fits[best]
    sc = score(X, f["weights"], f["means"], f["pc"])
    out.update(best_init=best, score=sc, bic=-2.0 * sc * n + (2 * K * d + K - 1) * np.log(n),
               weights=f["weights"], means=f["means"], covariances=f["covariances"])
    return out


def select(X, min_components=2, max_components=10, draws=None):
    """select_optimal_gmm_components(X, min_components, max_components) with every per-K fit and the margins.
    Returns dict(K=chosen, fits={K: fit_k(...)}, margins={...}, best=the chosen fit or None)."""
    X = np.asarray(X, dtype=np.float64)
    n = len(X)
    mg = Margins()
    if n == 1:
        return dict(K=1, fits={}, margins=mg.m, best=None)
    mf = max_feasible(n, min_components, max_components)
    if mf < 1:
        return dict(K=1, fits={}, margins=mg.m, best=None)
    if draws is None:
        draws = draw_table(mf)
    best_bic, best_k = np.inf, min(min_components, mf)
    fits, bics = {}, []
    finite = bool(np.isfinite(X).all())
    for K in range(1, mf + 1):
        if not finite:
            fits[K] = dict(K=K, failed=True)
            continue
        f = fit_k(X, K, draws, mg=mg)
        fits[K] = f
        if f["failed"]:
            continue
        bics.append(f["bic"])
        if f["bic"] < best_bic:
            best_bic, best_k = f["bic"], K
    if len(bics) > 1:
        s = np.sort(np.array(bics))
        mg.add("choice_of_k", (s[1] - s[0]) / max(abs(s[0]), 1e-300))
    best = fits.get(best_k)
    return dict(K=best_k, fits=fits, margins=mg.m, best=None if best is None or best["failed"] else best)
