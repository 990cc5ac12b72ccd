"""Silhouette, Davies-Bouldin and Calinski-Harabasz on the device (csrc/cluster_metrics.cu) against scikit-learn on the
same float64 arrays -- the functions tasks/clustering_helper.py:462-470 calls -- and a replay of the reference's own
fitness scoring (tests/golden/cluster_metrics_golden.npz)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIL_TOL, SAMPLE_TOL, RTOL = 1e-5, 5e-4, 1e-6


def _blobs(n, d, k, seed, n_dup=20):
    """scaled blobs with n_dup near-duplicate rows (the precision-sensitive case for the split-bf16 distances)"""
    from sklearn.preprocessing import StandardScaler
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((k, d)) * 1.5
    lab = rng.integers(0, k, n)
    x = centres[lab] + rng.standard_normal((n, d))
    src = rng.choice(n, n_dup, replace=False)
    dst = rng.choice(np.setdiff1d(np.arange(n), src), n_dup, replace=False)
    x[dst] = x[src] + 1e-4 * rng.standard_normal((n_dup, d))
    return StandardScaler().fit_transform(x), lab


def _compare(x, labels, check_samples=True):
    from sklearn import metrics
    from audiomuse_ai_b200 import cluster_metrics as cm
    got = {n: getattr(cm, n)(x, labels) for n in ("silhouette_score", "davies_bouldin_score", "calinski_harabasz_score")}
    want = {n: getattr(metrics, n)(x, labels) for n in got}
    print({n: (got[n], want[n]) for n in got})
    assert all(type(v) is float for v in got.values())
    assert abs(got["silhouette_score"] - want["silhouette_score"]) <= SIL_TOL
    np.testing.assert_allclose(got["davies_bouldin_score"], want["davies_bouldin_score"], rtol=RTOL)
    np.testing.assert_allclose(got["calinski_harabasz_score"], want["calinski_harabasz_score"], rtol=RTOL)
    s = None
    if check_samples:
        s = cm.silhouette_samples(x, labels)
        ref = metrics.silhouette_samples(x, labels)
        assert s.dtype == np.float64 and s.shape == ref.shape
        err = np.abs(s - ref).max()
        print(f"max |ds| = {err:.3g}")
        assert err <= SAMPLE_TOL
    return got, s


@pytest.mark.parametrize("n,d,k", [(3000, 200, 40), (5000, 58, 10), (2000, 512, 64), (4099, 37, 7)])
def test_blobs_match_sklearn(n, d, k):
    x, lab = _blobs(n, d, k, n + d)
    _compare(x, lab)


def test_exactly_two_clusters():
    x, lab = _blobs(1500, 20, 2, 7)
    _compare(x, lab)


def test_dbscan_labels_with_noise():
    """DBSCAN's -1 is an ordinary label to scikit-learn's metrics, and here"""
    from sklearn.cluster import DBSCAN
    rng = np.random.default_rng(4)
    centres = rng.standard_normal((6, 8)) * 4
    x = np.concatenate([centres[rng.integers(0, 6, 2400)] + 0.4 * rng.standard_normal((2400, 8)),
                        rng.uniform(-9, 9, (100, 8))])
    lab = DBSCAN(eps=1.2, min_samples=6).fit_predict(x)
    assert (lab == -1).sum() > 0 and len(set(lab.tolist()) - {-1}) >= 3
    _compare(x, lab)


def test_singleton_clusters_score_zero():
    x, lab = _blobs(1000, 16, 5, 9)
    single = np.array([3, 100, 517, 998])
    lab = lab.copy()
    lab[single] = 10 + np.arange(len(single))                  # four clusters of one point each
    _, s = _compare(x, lab)
    assert np.all(s[single] == 0.0)


def test_identical_points_in_different_clusters():
    """rows whose own cluster and nearest other cluster are all the same point: a = b = 0, scikit-learn's 0 / 0 -> 0"""
    from audiomuse_ai_b200 import cluster_metrics as cm
    x, lab = _blobs(800, 12, 4, 12)
    p = np.round(x[0] * 4)                                     # integer coordinates: scikit-learn's distances are exact
    x = np.concatenate([x, np.repeat(p[None], 5, axis=0)])
    lab = np.concatenate([lab, [7, 7, 7, 8, 8]])
    _, s = _compare(x, lab)
    assert np.all(s[-5:] == 0.0)
    # the same with a point that is not exactly representable in bf16: D_ii from the tensor cores cancels D_ij exactly
    q = x[1] + 1.0 / 3.0
    y = np.concatenate([x[:-5], np.repeat(q[None], 5, axis=0)])
    assert np.all(cm.silhouette_samples(y, lab)[-5:] == 0.0)


def test_degenerate_davies_bouldin_and_calinski_harabasz():
    from sklearn import metrics
    from audiomuse_ai_b200 import cluster_metrics as cm
    # every cluster a single repeated point (4 copies: the means are exact): CH = 1.0, DB = 0.0, silhouette 1
    pts = np.array([[0.0, 1.0, 2.0], [5.0, -3.0, 1.0], [-4.0, 4.0, 8.0]])
    x = np.repeat(pts, 4, axis=0)
    lab = np.repeat([0, 1, 2], 4)
    assert metrics.calinski_harabasz_score(x, lab) == 1.0 and metrics.davies_bouldin_score(x, lab) == 0.0
    assert cm.calinski_harabasz_score(x, lab) == 1.0
    assert cm.davies_bouldin_score(x, lab) == 0.0
    assert cm.silhouette_score(x, lab) == metrics.silhouette_score(x, lab) == 1.0
    # two clusters with the same centroid: their distance of 0 counts as infinite (DB = (0.2 + 0.4 + 0.4) / 3)
    x = np.array([[-1.0, 0.0], [1.0, 0.0], [0.0, -3.0], [0.0, 3.0], [9.0, 0.0], [11.0, 0.0]])
    lab = np.array([0, 0, 1, 1, 2, 2])
    want = metrics.davies_bouldin_score(x, lab)
    assert abs(want - 1.0 / 3.0) < 1e-15
    np.testing.assert_allclose(cm.davies_bouldin_score(x, lab), want, rtol=RTOL)
    np.testing.assert_allclose(cm.calinski_harabasz_score(x, lab), metrics.calinski_harabasz_score(x, lab), rtol=RTOL)


def test_large_case_against_float64_restatement():
    """N = 50 000, d = 200, L = 100 against a float64 chunked torch.cdist restatement on the same GPU (scikit-learn
    takes minutes here), on the float32 values the device sees"""
    import torch
    from audiomuse_ai_b200 import cluster_metrics as cm
    x, lab = _blobs(50000, 200, 100, 21, n_dup=200)
    x32 = x.astype(np.float32)
    s = cm.silhouette_samples(x32, lab)
    score = cm.silhouette_score(x32, lab)
    dev = torch.device("cuda")
    xt = torch.from_numpy(x32.astype(np.float64)).to(dev)
    lt = torch.from_numpy(lab).to(dev)
    onehot = torch.nn.functional.one_hot(lt, 100).to(torch.float64)
    counts = onehot.sum(0)
    S = torch.cat([torch.cdist(xt[i:i + 2048], xt) @ onehot
                   for i in range(0, len(xt), 2048)])
    own = S.gather(1, lt[:, None])[:, 0]
    a = own / (counts[lt] - 1)
    b = (S / counts[None, :]).scatter(1, lt[:, None], float("inf")).min(1).values
    ref = torch.nan_to_num((b - a) / torch.maximum(a, b)).cpu().numpy()
    err = np.abs(s - ref).max()
    print(f"N=50000: score {score} vs {ref.mean()}, max |ds| = {err:.3g}")
    assert abs(score - ref.mean()) <= SIL_TOL and err <= SAMPLE_TOL


def test_golden_replay_of_the_reference_scoring(golden_dir):
    """the reference's _format_and_score_iteration_result (k-means and DBSCAN labellings, all three weights on): the
    metric values, their transforms at clustering_helper.py:463-469, and the fitness score with them"""
    from audiomuse_ai_b200 import cluster_metrics as cm
    g = np.load(os.path.join(golden_dir, "cluster_metrics_golden.npz"))
    w = dict(zip([str(n) for n in g["weight_names"]], g["weights"]))
    for case in ("kmeans", "dbscan"):
        X, labels = g[f"{case}_X"], g[f"{case}_labels"]
        sil = cm.silhouette_score(X, labels)
        db = cm.davies_bouldin_score(X, labels)
        ch = cm.calinski_harabasz_score(X, labels)
        assert abs(sil - g[f"{case}_silhouette_score"]) <= SIL_TOL
        np.testing.assert_allclose(db, g[f"{case}_davies_bouldin_score"], rtol=RTOL)
        np.testing.assert_allclose(ch, g[f"{case}_calinski_harabasz_score"], rtol=RTOL)

        def transformed(s, d, c):
            return {"silhouette": (s + 1) / 2.0, "davies_bouldin": 1.0 / (1.0 + d),
                    "calinski_harabasz": 1.0 - np.exp(-c / 500.0)}

        t_got = transformed(sil, db, ch)
        t_ref = transformed(float(g[f"{case}_silhouette_score"]), float(g[f"{case}_davies_bouldin_score"]),
                            float(g[f"{case}_calinski_harabasz_score"]))
        assert abs(t_got["silhouette"] - t_ref["silhouette"]) <= SIL_TOL / 2
        for k in ("davies_bouldin", "calinski_harabasz"):
            np.testing.assert_allclose(t_got[k], t_ref[k], rtol=RTOL)
        fitness = float(g[f"{case}_fitness"]) + sum(w[k] * (t_got[k] - t_ref[k]) for k in t_got)
        assert abs(fitness - float(g[f"{case}_fitness"])) <= sum(w[k] for k in t_got) * SIL_TOL
