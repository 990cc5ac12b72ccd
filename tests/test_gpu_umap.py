"""UMAP on the device (csrc/umap.cu + projection.umap_fit_transform / project_with_umap) against the float64 oracle
(oracle/umap.py): the graph entry for entry, the spectral initialisation against scipy's eigsh, the layout rule against
the Jacobi restatement, determinism, and the layout's quality against the sequential oracle's floor
(tests/golden/umap_golden.json, made by tests/golden/make_umap_golden.py)."""
import json
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from oracle import umap as ou

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_umap_golden as mg  # noqa: E402

TOL = 1e-8


def _pj():
    from audiomuse_ai_b200 import projection
    return projection


def _device_graph(X, n_neighbors=15, n_epochs=None):
    with _pj().UmapGraph(X, n_neighbors, n_epochs) as g:
        return g.graph(), g.k, g.n_epochs


def _check_graph(X, n_neighbors=15, n_epochs=None):
    got, k, ne = _device_graph(X, n_neighbors, n_epochs)
    ref = ou.fuzzy_graph(X, n_neighbors, n_epochs)
    assert (k, ne) == (ref["k"], ref["n_epochs"])
    W, R = got["W"], ref["W"]
    assert W.nnz == R.nnz
    np.testing.assert_array_equal(W.indptr, R.indptr)
    np.testing.assert_array_equal(W.indices, R.indices)
    np.testing.assert_allclose(W.data, R.data, rtol=1e-9, atol=0)
    np.testing.assert_allclose(got["eps"], ref["eps"], rtol=1e-9, atol=0)
    np.testing.assert_allclose(got["rho"], ref["rho"], rtol=1e-9, atol=0)
    np.testing.assert_allclose(got["sigma"], ref["sigma"], rtol=1e-9, atol=0)
    assert abs(W - W.T).max() == 0 if W.nnz else True
    return got, ref


@pytest.mark.parametrize("name", ["blobs", "mixture", "curve", "clique"])
def test_graph_equals_oracle(name):
    X, _ = mg.DATASETS[name]()
    _check_graph(X)


@pytest.mark.parametrize("N", [2, 3, 10, 16, 255, 256, 257, 1025])
def test_graph_small_and_tile_edges(N):
    X = np.random.default_rng(N).standard_normal((N, 13)).astype(np.float32)
    got, _ = _check_graph(X)
    Y = _pj().umap_fit_transform(X, n_epochs=50)
    assert Y.shape == (N, 2) and Y.dtype == np.float32 and np.isfinite(Y).all()


@pytest.mark.parametrize("d", [13, 200, 512])
def test_graph_dims(d):
    X = np.random.default_rng(d).standard_normal((1200, d)).astype(np.float32)
    _check_graph(X, n_epochs=200)


def test_epoch_switch_rows():
    for n in (10000, 10001):
        X, _ = mg.mixture200(n)
        got, ref = _check_graph(X)
        assert ref["n_epochs"] == (500 if n == 10000 else 200)


def test_spectral_initialisation_against_eigsh():
    from scipy.sparse.linalg import eigsh
    X, _ = mg.mixture()
    details = {}
    _pj().umap_fit_transform(X, details=details)
    W = details["W"]
    assert details["components"] == 1 and details["init"] == "spectral"
    deg = np.asarray(W.sum(1)).ravel()
    D = sp.diags(1.0 / np.sqrt(deg))
    L = sp.identity(W.shape[0]) - D @ W @ D
    w, U = eigsh(L, k=4, sigma=-1e-5, which="LM", tol=0)
    o = np.argsort(w)
    w, U = w[o], U[:, o]
    ev = details["eigenvalues"]
    np.testing.assert_allclose(ev, w[:3], rtol=0, atol=1e-8)
    # the raw unit vectors of the 2nd and 3rd eigenvalues span the same plane as eigsh's
    got = _pj()._unit_vectors(W, 2, 0)
    gap = w[3] - w[2]
    Qa, _ = np.linalg.qr(got)
    Qb, _ = np.linalg.qr(U[:, 1:3])
    sin = np.linalg.norm(Qa - Qb @ (Qb.T @ Qa), 2)
    assert sin <= max(10 * TOL / gap, 1e-12), (sin, gap)
    np.testing.assert_allclose(np.linalg.norm(got, axis=0), 1.0, rtol=1e-10)


def test_clique_component_eigenspace_and_placement():
    from audiomuse_ai_b200 import clustering_gpu as cg
    X, _ = mg.clique()
    details = {}
    Y = _pj().umap_fit_transform(X, details=details)
    W = details["W"]
    n, lab = connected_components(W, directed=False)
    assert n == 2 and details["components"] == 2
    assert len(set(lab[-40:])) == 1 and lab[-1] != lab[0]
    for c in range(2):
        rows = np.flatnonzero(lab == c)
        G = W[rows][:, rows]
        det = {}
        emb, ev = cg.spectral_embedding_csr(G, 3, tol=TOL, details=det)
        dd = np.sqrt(np.asarray(G.sum(1)).ravel())
        S = sp.diags(1.0 / dd) @ G @ sp.diags(1.0 / dd)
        U = emb * dd[:, None]
        U /= np.linalg.norm(U, axis=0)
        res = np.linalg.norm(S @ U - U * (1.0 - ev)[None, :], axis=0)
        assert np.all(res <= 2 * TOL), res
    # two components start at -e_1 and +e_1: the copies' x range and the other rows' do not overlap
    Y0 = details["Y0"]
    a, b = Y0[-40:, 0], Y0[:-40, 0]
    assert a.min() > b.max() or a.max() < b.min()
    assert np.isfinite(Y).all()


@pytest.mark.parametrize("epochs", [1, 2, 5])
def test_layout_rule_equals_jacobi_oracle(epochs):
    X, _ = mg.mixture(2000, 13, 10, 7)
    a, b = _pj().find_ab_params()
    with _pj().UmapGraph(X) as g:
        G = g.graph()
        Y0 = _pj().initial_layout(g.X, G["W"], seed=3)
        got = g.layout(Y0, a, b, seed=11, epochs=epochs)
    ref = ou.sgd_jacobi(Y0, G["W"], G["eps"], g.n_epochs, a, b, seed=11, epochs=epochs)
    if epochs == 1:         # every epochs_per_sample is >= 1: no entry is due in epoch 0
        np.testing.assert_array_equal(got, Y0)
    else:
        assert np.abs(got - Y0).max() > 1e-3
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-4)


def test_same_seed_bit_identical_other_seed_differs():
    X, _ = mg.mixture(3000, 13, 20, 9)
    a = _pj().umap_fit_transform(X, seed=0)
    b = _pj().umap_fit_transform(X, seed=0)
    c = _pj().umap_fit_transform(X, seed=1)
    assert a.tobytes() == b.tobytes()
    assert np.abs(a - c).max() > 1e-3


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "umap_golden.json")) as f:
        return json.load(f)


MARGIN = {"trustworthiness": 0.01, "knn_recall": 0.02, "silhouette": 0.05}


@pytest.mark.parametrize("name", list(mg.DATASETS))
def test_quality_not_below_the_sequential_oracle(name, golden):
    X, lab = mg.DATASETS[name]()
    ref = golden["sets"][name]
    assert ref["N"] == len(X)
    Y = _pj().umap_fit_transform(X, seed=0)
    q = ou.quality(X, Y, lab)
    print(name, {m: round(v, 4) for m, v in q.items()}, "oracle min", ref["min"])
    for m, v in q.items():
        assert v >= ref["min"][m] - MARGIN[m], (m, v, ref["min"][m])


def test_project_with_umap_end_to_end(golden_dir):
    """the drop-in on the matrix app_helper.build_and_store_map_projection handed to _project_with_umap
    (tests/golden/map_golden.npz)"""
    M = np.load(os.path.join(golden_dir, "map_golden.npz"))["matrix"]
    out = _pj().project_with_umap([v for v in M])
    P = np.asarray(out)
    assert isinstance(out, list) and len(out) == len(M) and all(isinstance(t, tuple) and len(t) == 2 for t in out)
    assert np.abs(P).max() == pytest.approx(1.0, abs=1e-12) and np.all(np.abs(P) <= 1.0)
    np.testing.assert_allclose(P.mean(0), 0.0, atol=1e-6)
    assert np.array(out, dtype=np.float32).tobytes().__len__() == 8 * len(M)
    assert out == _pj().project_with_umap(list(M))       # the same library gives the same map
