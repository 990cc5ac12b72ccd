"""Host checks of the k-means one-step oracle (oracle/kmeans.py): the generators have the properties the GPU tests
rely on, a float32 restatement of the fp32 step passes the acceptance rule, and the rule rejects planted faults."""
import numpy as np
import pytest

from oracle import kmeans as okm


@pytest.mark.parametrize("N,d,k", [(64, 1, 16), (64, 3, 17), (40, 64, 33), (24, 513, 100), (8, 4097, 5)])
def test_lattice_is_exact_in_fp32(N, d, k):
    """every partial sum of every dot product, norm, v, dist and column sum is an integer below 2^24, and the
    bf16 split of every entry has lo = 0: both steps compute the lattice cases without a rounding"""
    X, C = okm.lattice(N, d, k, seed=d)
    X64, C64 = X.astype(np.float64), C.astype(np.float64)
    assert (X64 == np.rint(X64)).all() and (C64 == np.rint(C64)).all()
    bf16_hi = lambda a: (a.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)  # noqa: E731 (exact: |a| <= 256)
    assert (bf16_hi(X) == X).all() and (bf16_hi(C) == C).all()
    lim = 2.0 ** 24
    # the largest partial sum of x.c, c.c, x.x in any order is at most sum |x c|
    assert (np.abs(X64) @ np.abs(C64).T).max() < lim / 4
    assert (X64 * X64).sum(1).max() < lim / 4 and (C64 * C64).sum(1).max() < lim / 4
    D = okm.distances(X, C)
    assert (D == np.rint(D)).all() and D.max() < lim
    S, _ = okm.sums_exact(np.abs(X), np.zeros(N, np.int64), 1)
    assert S.max() < lim


def test_lattice_has_exact_ties():
    X, C = okm.lattice(400, 5, 16, seed=1)
    D = okm.distances(X, C)
    m = D.min(1, keepdims=True)
    tied = (D == m).sum(1) > 1
    assert (C[0] == C[1]).all()
    assert tied.mean() > 0.2                       # duplicated centres and the planted equidistant rows
    lab = okm.oracle_labels(D)
    assert (lab != 1).all()                        # centre 1 duplicates centre 0: never the lowest tied index
    np.testing.assert_array_equal(lab[tied], np.argmax(D[tied] == m[tied], 1))


def test_probes_hit_every_level():
    for signed in (False, True):
        X, C, lev = okm.probes(64, per_level=16, signed=signed, seed=3)
        if not signed:
            assert (X >= 0).all()
        D = okm.distances(X, C)
        gap, _ = okm.margins(D, okm.fp32_errors(X, C))
        scale = np.sqrt((X.astype(np.float64) ** 2).sum(1)) * np.sqrt((C.astype(np.float64) ** 2).sum(1).max())
        rel = gap / scale
        for lv in (4, 10, 16, 20):
            r = rel[lev == lv]
            assert np.median(np.abs(np.log2(r) + lv)) < 0.5, (signed, lv)


CASES = {
    "lattice": lambda: okm.lattice(300, 65, 33, seed=5)[:2],
    "lattice_d1": lambda: okm.lattice(200, 1, 16, seed=6)[:2],
    "probes_pos": lambda: okm.probes(512, per_level=8, seed=7)[:2],
    "probes_signed": lambda: okm.probes(200, per_level=8, signed=True, seed=8)[:2],
    "blobs": lambda: okm.blobs(600, 58, 40, seed=9)[:2],
    "offset_blobs": lambda: okm.blobs(400, 64, 16, seed=10, offset=1000.0)[:2],
    "uniform": lambda: okm.uniform(300, 1024, 16, seed=11),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_fp32_step_passes_the_rule(case):
    """the float32 restatement of exact_argmin passes the acceptance rule on every generator, and its dist is within
    dist_bound"""
    X, C = CASES[case]()
    lab, v, dist = okm.fp32_step(X, C)
    D = okm.distances(X, C)
    assert okm.accept(X, C, lab, D=D).all()
    err = np.abs(dist.astype(np.float64) - D[np.arange(len(X)), lab])
    assert (err <= okm.dist_bound(X, C, lab, tensor_cores=False)).all()
    if case.startswith("lattice"):
        np.testing.assert_array_equal(lab, okm.oracle_labels(D))
        np.testing.assert_array_equal(dist.astype(np.float64), D[np.arange(len(X)), lab])


def test_rule_rejects_runner_up_outside_the_slack():
    X, C = okm.blobs(2000, 58, 40, seed=12)[:2]
    D, E = okm.distances(X, C), okm.fp32_errors(X, C)
    gap, slack = okm.margins(D, E)
    second = np.argsort(D, axis=1, kind="stable")[:, 1]
    lab = okm.oracle_labels(D)
    out = gap > slack
    assert out.sum() > 1000
    bad = lab.copy()
    bad[out] = second[out]
    ok = okm.accept(X, C, bad, D=D, E=E)
    assert not ok[out].any() and ok[~out].all()


@pytest.mark.parametrize("signed", [False, True])
def test_rule_rejects_v_perturbed_on_probes(signed):
    """v of every centre but the float64 winner lowered by 2^-10 ||x|| cmax: probes closer than that flip, and the
    rule catches every flip that lies outside the fp32 slack -- a tensor-core error of that size could not pass"""
    X, C, lev = okm.probes(256, per_level=8, levels=range(4, 25), signed=signed, seed=13)
    lab, v, _ = okm.fp32_step(X, C)
    D, E = okm.distances(X, C), okm.fp32_errors(X, C)
    js = okm.oracle_labels(D)
    X64 = X.astype(np.float64)
    delta = 2.0 ** -10 * np.sqrt((X64 ** 2).sum(1)) * np.sqrt((C.astype(np.float64) ** 2).sum(1).max())
    vp = v.astype(np.float64) - delta[:, None]
    vp[np.arange(len(X)), js] += delta
    bad = vp.argmin(1)
    ok = okm.accept(X, C, bad, D=D, E=E)
    gap, slack = okm.margins(D, E)
    flipped = bad != js
    assert flipped.sum() > 50
    assert not ok[flipped & (gap > slack)].any()
    assert (flipped & (gap > slack)).sum() > 30


def test_rule_rejects_tie_to_higher_index():
    X, C = okm.lattice(200, 8, 16, seed=14)
    D = okm.distances(X, C)
    lab = okm.oracle_labels(D)
    m = D.min(1, keepdims=True)
    tied = np.nonzero((D == m).sum(1) > 1)[0]
    assert len(tied) > 20
    assert okm.accept(X, C, lab, D=D).all()
    bad = lab.copy()
    bad[tied] = (D[tied] == m[tied]).shape[1] - 1 - np.argmax((D[tied] == m[tied])[:, ::-1], 1)  # highest tied
    assert (bad[tied] != lab[tied]).all()
    assert not okm.accept(X, C, bad, D=D)[tied].any()


def test_lloyd_step_relocates_as_sklearn():
    """the oracle's relocation is scikit-learn's: the empty cluster takes the row farthest from its centre"""
    X, C, _ = okm.separated(300, 8, 6, seed=15)
    X = X.copy()
    X[17] += 100.0                                  # the farthest row from its centre
    init = C.copy()
    init[4] = init[1]                               # cluster 4 is empty after the E-step
    lab, newC, n0 = okm.lloyd_step(X, init)
    assert n0[4] == 0
    np.testing.assert_array_equal(newC[4], X[17].astype(np.float64))
    # sklearn's own Lloyd, one iteration from the same centres
    from sklearn.cluster import KMeans
    km = KMeans(6, init=init, n_init=1, max_iter=1, tol=0).fit(X.astype(np.float64))
    np.testing.assert_allclose(km.cluster_centers_, newC, rtol=0, atol=1e-9)


def test_lloyd_step_keeps_empty_clusters_when_every_row_is_on_its_centre():
    """more clusters than distinct rows: scikit-learn's relocation returns early and the empty cluster moves to the
    centre of the first largest cluster"""
    X = np.repeat(np.array([[1.0, 2.0], [4.0, 0.0], [-3.0, 5.0]], np.float32), 4, axis=0)
    init = np.array([[1, 2], [4, 0], [-3, 5], [1, 2]], np.float32)
    lab, newC, n0 = okm.lloyd_step(X, init)
    assert n0[3] == 0
    np.testing.assert_array_equal(newC[:3], init[:3])
    np.testing.assert_array_equal(newC[3], init[0])
    from sklearn.cluster import KMeans
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        km = KMeans(4, init=init, n_init=1, max_iter=1, tol=0).fit(X)
    np.testing.assert_allclose(km.cluster_centers_, newC, atol=1e-6)
    np.testing.assert_array_equal(km.labels_, lab)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 1e39])
def test_kmeans_fit_rejects_non_finite_input_before_device_work(bad, monkeypatch):
    """kmeans_fit and GPUKMeans raise scikit-learn's ValueError for NaN / inf rows (also a float64 value beyond
    float32's range) and initial centres, without loading the native library"""
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg

    def no_device():
        raise AssertionError("device work before input validation")
    monkeypatch.setattr(_lib, "load", no_device)
    X = np.random.default_rng(0).standard_normal((50, 4))
    init = X[:3].copy()
    Xb = X.copy()
    Xb[7, 2] = bad
    with pytest.raises(ValueError, match="NaN or infinity"):
        cg.kmeans_fit(Xb, 3)
    with pytest.raises(ValueError, match="NaN or infinity"):
        cg.GPUKMeans(3).fit_predict(Xb)
    init[1, 0] = bad
    with pytest.raises(ValueError, match="NaN or infinity"):
        cg.kmeans_fit(X, 3, init_centers=init)
    from sklearn.cluster import KMeans
    with pytest.raises(ValueError):
        KMeans(3, n_init=1).fit(Xb.astype(np.float32))
