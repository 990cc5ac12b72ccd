"""Spectral clustering on the device (csrc/spectral.cu + clustering_gpu.spectral_embedding / GPUSpectralClustering)
against scikit-learn's SpectralClustering(affinity='nearest_neighbors'), the class the reference runs
(tasks/clustering_gpu.py:312-335).  Inputs are float32 values, so scikit-learn's float64 k-NN ranking and the device's
see the same points."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components, laplacian
from scipy.sparse.linalg import eigsh

pytestmark = pytest.mark.gpu

TOL = 1e-8


def _cg():
    from audiomuse_ai_b200 import clustering_gpu
    return clustering_gpu


def _mixture(n, d, k, spread, seed):
    """k overlapping Gaussian groups, StandardScaler-ed, float32 values"""
    from sklearn.preprocessing import StandardScaler
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((k, d)) * spread
    lab = rng.integers(0, k, n)
    return StandardScaler().fit_transform(c[lab] + rng.standard_normal((n, d))).astype(np.float32), lab


def _separated(n, d, k, seed, gap=40.0):
    rng = np.random.default_rng(seed)
    lab = np.arange(n) % k
    c = rng.standard_normal((k, d)) * gap
    return (c[lab] + rng.standard_normal((n, d))).astype(np.float32), lab


def _sk_affinity(X, n_neighbors):
    from sklearn.neighbors import kneighbors_graph
    C = kneighbors_graph(X.astype(np.float64), n_neighbors, include_self=True)
    return 0.5 * (C + C.T)


def _without_diag(A):
    A = sp.csr_matrix(A, copy=True)
    A.setdiag(0)
    A.eliminate_zeros()
    A.sort_indices()
    return A


def _ari(a, b):
    from sklearn.metrics import adjusted_rand_score
    return adjusted_rand_score(a, b)


@pytest.mark.parametrize("N", [1000, 7000])
@pytest.mark.parametrize("d", [13, 200])
@pytest.mark.parametrize("n_neighbors", [2, 20])
def test_graph_equals_sklearn(N, d, n_neighbors):
    X = np.random.default_rng(N + d + n_neighbors).standard_normal((N, d)).astype(np.float32)
    W, dd = _cg().spectral_graph(X, n_neighbors)
    A = _sk_affinity(X, n_neighbors)
    ref = _without_diag(A)
    assert W.shape == (N, N) and W.nnz == ref.nnz
    np.testing.assert_array_equal(W.indptr, ref.indptr)
    np.testing.assert_array_equal(W.indices, ref.indices)
    np.testing.assert_array_equal(W.data, ref.data.astype(np.float32))
    _, dd_ref = laplacian(A, normed=True, return_diag=True)
    np.testing.assert_allclose(dd, dd_ref, rtol=1e-15, atol=0)


def test_graph_with_duplicate_rows():
    """Which of several identical rows enters a list may differ from scikit-learn; the graph stays symmetric, its rows sum
    to dd^2, and every copy of a row lands in the same cluster."""
    cg = _cg()
    base, _ = _separated(300, 8, 3, seed=2)
    X = np.concatenate([base, base[:40], base[:40]])
    W, dd = cg.spectral_graph(X, 10)
    assert abs(W - W.T).max() == 0
    np.testing.assert_allclose(np.asarray(W.sum(1)).ravel(), dd ** 2, rtol=1e-15)
    assert set(np.unique(W.data)) <= {0.5, 1.0} and W.diagonal().max() == 0
    labels = cg.GPUSpectralClustering(n_clusters=3, n_neighbors=10, random_state=1).fit_predict(X)
    np.testing.assert_array_equal(labels[300:340], labels[:40])
    np.testing.assert_array_equal(labels[340:380], labels[:40])


def _check_spectrum(X, n_clusters, n_neighbors=20, seed=0):
    cg = _cg()
    details = {}
    emb, ev = cg.spectral_embedding(X, n_clusters, n_neighbors=n_neighbors, seed=seed, tol=TOL, details=details)
    N = len(X)
    L = laplacian(_sk_affinity(X, n_neighbors), normed=True)
    if n_clusters + 1 < N - 1:
        w, U = eigsh(L, k=n_clusters + 1, sigma=-1e-5, which="LM", tol=0)
    else:
        w, U = np.linalg.eigh(L.toarray())
    order = np.argsort(w)
    w, U = w[order], U[:, order]
    np.testing.assert_allclose(ev, w[:n_clusters], rtol=0, atol=1e-8)
    assert np.all(np.diff(ev) >= -1e-12)
    # sin of the largest principal angle between the D^1/2 embedding subspaces, against residual / gap
    gap = w[n_clusters] - w[n_clusters - 1] if n_clusters < N else np.inf
    Qa, _ = np.linalg.qr(emb * details["dd"][:, None])
    Qb, _ = np.linalg.qr(U[:, :n_clusters])
    sin = np.linalg.norm(Qa - Qb @ (Qb.T @ Qa), 2)
    assert sin <= max(10 * TOL / gap, 1e-12), (sin, gap)
    assert np.all(details["residuals"] <= TOL)
    # sklearn's sign convention: the largest-magnitude entry of every vector is positive
    top = np.argmax(np.abs(emb), axis=0)
    assert np.all(emb[top, np.arange(n_clusters)] > 0)
    return details


@pytest.mark.parametrize("n_clusters", [2, 40, 100])
def test_spectrum_connected_overlapping(n_clusters):
    X, _ = _mixture(3000, 13, 60, 1.0, seed=5)
    W, _ = _cg().spectral_graph(X, 20)
    assert connected_components(W, directed=False)[0] == 1
    _check_spectrum(X, n_clusters)


def test_spectrum_disconnected():
    X, _ = _separated(1200, 10, 12, seed=3)
    W, _ = _cg().spectral_graph(X, 20)
    assert connected_components(W, directed=False)[0] == 12
    _check_spectrum(X, 20)


def test_spectrum_block_equals_n():
    X, _ = _mixture(150, 6, 5, 2.0, seed=9)
    details = _check_spectrum(X, 100)
    assert details["block"] == 150 and details["outer_iterations"] == 1


def test_labels_disconnected_components():
    X, _ = _separated(1500, 16, 9, seed=4)
    W, _ = _cg().spectral_graph(X, 20)
    n, comp = connected_components(W, directed=False)
    assert n == 9
    labels = _cg().GPUSpectralClustering(n_clusters=9, n_neighbors=20, random_state=3).fit_predict(X)
    assert _ari(labels, comp) == 1.0


def test_labels_separable_connected_match_sklearn():
    from sklearn.cluster import SpectralClustering
    X, _ = _mixture(2000, 13, 8, 2.0, seed=6)
    W, _ = _cg().spectral_graph(X, 20)
    assert connected_components(W, directed=False)[0] == 1
    ref = SpectralClustering(n_clusters=8, affinity="nearest_neighbors", n_neighbors=20, random_state=7,
                             n_init=10).fit_predict(X)
    got = _cg().GPUSpectralClustering(n_clusters=8, n_neighbors=20, random_state=7).fit_predict(X)
    assert _ari(got, ref) >= 0.99


def test_labels_overlapping_inertia_within_one_percent():
    """Overlapping groups: the labellings may differ, but as k-means solutions on scikit-learn's own embedding ours is
    within 1 % of scikit-learn's."""
    from sklearn.cluster import SpectralClustering
    from sklearn.manifold import spectral_embedding
    X, _ = _mixture(2500, 13, 30, 1.0, seed=8)
    k = 20
    sk = SpectralClustering(n_clusters=k, affinity="nearest_neighbors", n_neighbors=20, random_state=11, n_init=10)
    ref = sk.fit_predict(X)
    E = spectral_embedding(sk.affinity_matrix_, n_components=k, random_state=11, drop_first=False)
    got = _cg().GPUSpectralClustering(n_clusters=k, n_neighbors=20, random_state=11).fit_predict(X)

    def inertia(lab):
        return sum(((E[lab == c] - E[lab == c].mean(0)) ** 2).sum() for c in np.unique(lab))

    assert inertia(got) <= 1.01 * inertia(ref), (inertia(got), inertia(ref))


def test_same_random_state_same_labels_and_attributes():
    X, _ = _mixture(3000, 13, 40, 1.0, seed=10)
    a = _cg().GPUSpectralClustering(n_clusters=40, n_neighbors=20, random_state=123)
    b = _cg().GPUSpectralClustering(n_clusters=40, n_neighbors=20, random_state=123)
    la, lb = a.fit_predict(X), b.fit_predict(X)
    np.testing.assert_array_equal(la, lb)
    assert a.using_gpu and a.labels_ is la and la.dtype == np.int32 and len(np.unique(la)) == 40
    assert not hasattr(a, "cluster_centers_") and not hasattr(a, "means_")


def test_golden_replay(golden_dir):
    import ast
    g = np.load(os.path.join(golden_dir, "spectral_golden.npz"))
    kw = {str(n): ast.literal_eval(str(v)) for n, v in zip(g["ctor_names"], g["ctor_values"])}
    X = g["X"]
    labels = _cg().GPUSpectralClustering(**kw).fit_predict(X)
    assert _ari(labels, g["labels"]) >= 0.99
    # the reference's centres for a model without cluster_centers_ (clustering_helper.py:320-333), from our labels,
    # matched to the recorded ones through the label overlap
    ours = {c: X[labels == c].mean(0) for c in np.unique(labels)}
    for c in np.unique(labels):
        ref_c = np.bincount(g["labels"][labels == c]).argmax()
        np.testing.assert_allclose(ours[c], g["centers"][ref_c], rtol=0, atol=1e-6)


def test_scale_50k_residuals_checked_on_the_host():
    X, _ = _mixture(50000, 13, 60, 1.5, seed=12)
    details = {}
    emb, ev = _cg().spectral_embedding(X, 60, n_neighbors=20, seed=1, tol=TOL, details=details)
    W, dd = details["affinity"], details["dd"]
    S = sp.diags(1.0 / dd) @ W.astype(np.float64) @ sp.diags(1.0 / dd)
    U = emb * dd[:, None]
    U /= np.linalg.norm(U, axis=0)
    R = S @ U - U * (1.0 - ev)[None, :]
    res = np.linalg.norm(R, axis=0)
    assert np.all(res <= 2 * TOL), res.max()
