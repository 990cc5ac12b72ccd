"""The DBSCAN oracle (oracle/dbscan.py) against scikit-learn, and the generated cases of test_gpu_cluster_extra_exact.py
checked for the property each is meant to test.  No GPU needed."""
import numpy as np
import pytest

from oracle import dbscan as od


def _sklearn(x, eps, min_samples):
    from sklearn.cluster import DBSCAN
    return DBSCAN(eps=eps, min_samples=min_samples, algorithm="brute").fit_predict(x.astype(np.float64)).astype(np.int32)


def _relation_to_csr(rel):
    r, c = np.nonzero(rel)
    indptr = np.zeros(rel.shape[0] + 1, np.int64)
    np.cumsum(np.bincount(r, minlength=rel.shape[0]), out=indptr[1:])
    return indptr, c


def _margins(x, eps):
    """|s - eps^2| / eps^2 over all pairs whose squared distance s is not exactly eps^2 (exact ties are decided alike
    by every exact evaluation)"""
    s = od.sq_dist(x[:, None, :], x[None, :, :])
    rel = np.abs(s - eps * eps) / (eps * eps)
    return rel[rel != 0]


@pytest.mark.parametrize("d", od.RAGGED_D)
def test_ragged_cases_oracle_equals_sklearn(d):
    for n in od.RAGGED_N:
        x, eps, ms = od.ragged(n, d)
        lab, nc = od.dbscan(x, eps, ms)
        assert np.array_equal(lab, _sklearn(x, eps, ms)), (n, d)
        assert nc == len(set(lab.tolist()) - {-1})
        if n > 1:
            assert _margins(x, eps).min() > 1e-6, (n, d)   # eps sits between two pair distances, far from both
    x, eps, ms = od.ragged(129, d)
    lab, _ = od.dbscan(x, eps, ms)
    assert (lab >= 0).any() and (lab == -1).any(), "the largest ragged case must have clusters and noise"


def test_degenerate_cases_oracle_equals_sklearn():
    got = {}
    for name, x, eps, ms in od.degenerate():
        lab, nc = od.dbscan(x, eps, ms)
        assert np.array_equal(lab, _sklearn(x, eps, ms)), name
        got[name] = (lab, nc)
    assert (got["min_samples_1"][0] >= 0).all()                    # every point core
    assert (got["min_samples_above_n"][0] == -1).all() and got["min_samples_above_n"][1] == 0
    assert (got["identical_rows"][0] == 0).all()
    assert (got["identical_rows_all_noise"][0] == -1).all()
    lab, nc = got["duplicate_blocks"]
    assert nc == 7 and (lab == -1).sum() == sum(range(1, 6))      # blocks of 6 .. 12 copies are clusters, 1 .. 5 noise


@pytest.mark.parametrize("d", [2, 64, 512])
def test_near_eps_probes_sit_at_their_margins(d):
    for k in range(8, 24):
        for sign in (1, -1):
            x, eps, ms, inside = od.probe(d, k, sign)
            s = od.sq_dist(x[4], x[0])
            rel = (s - eps * eps) / (eps * eps)
            want = (1.0 + sign * 2.0 ** -k) ** 2 - 1.0
            assert (rel < 0) == inside and abs(rel) >= 1e-12
            assert abs(rel - want) <= 1e-6 * abs(want), (d, k, sign, rel)
            lab, _ = od.dbscan(x, eps, ms)
            expect = np.array([0, 0, -1, 0, 0 if inside else -1, 0], np.int32)
            assert np.array_equal(lab, expect) and np.array_equal(_sklearn(x, eps, ms), expect), (d, k, sign)


@pytest.mark.parametrize("dim,side,eps,ms", od.LATTICE_CASES)
def test_lattice_cases_flip_under_float32_eps_squared(dim, side, eps, ms):
    """The float32 square of eps (what the kernel compared against when eps was passed as float) moves lattice pairs
    across the boundary for eps 0.1 / 0.2 / 0.3, enough to change the labels; 0.23 and 0.5 are controls."""
    x = od.lattice(dim, side)
    s = od.sq_dist(x[:, None, :], x[None, :, :])
    exact = s <= eps * eps
    rounded = s <= float(np.float32(np.float32(eps) * np.float32(eps)))
    flips = int((exact != rounded)[np.triu_indices(len(x), 1)].sum())
    lab, _ = od.dbscan(x, eps, ms)
    assert np.array_equal(lab, _sklearn(x, eps, ms))
    assert np.array_equal(lab, od.expand(*_relation_to_csr(exact), ms)[0])
    # the squares of these 24-bit differences are exact in float64 and their sum is rounded at most dim - 1 times, so
    # any margin above dim ulps is decided alike by every float64 evaluation (some pairs sit 1.4e-14 from 0.5^2)
    assert _margins(x, eps).min() >= 4 * dim * 2.0 ** -53
    old, _ = od.expand(*_relation_to_csr(rounded), ms)
    if eps in (0.23, 0.5):
        assert flips == 0
    else:
        assert flips > 0 and (old != lab).sum() > 0, (flips, int((old != lab).sum()))
    if (dim, side) == (2, 20):
        assert flips == {0.1: 80, 0.2: 80, 0.3: 40}.get(eps, 0)


def test_border_point_touches_two_clusters():
    x, eps, ms, expect = od.border_between_clusters()
    s = od.sq_dist(x[10], x)
    indptr, _ = od.neighbourhoods(x, eps)
    count = np.diff(indptr)
    core = count >= ms
    assert not core[10] and core[:10].all()
    near = np.nonzero((s <= eps * eps) & core)[0]
    assert set(near.tolist()) == {4, 5}                              # one core row of each cluster
    assert s[5] < s[4]                                               # the nearer one is in cluster 1
    assert np.abs(s - eps * eps).min() > 1e-3
    lab, nc = od.dbscan(x, eps, ms)
    assert nc == 2 and np.array_equal(lab, expect) and np.array_equal(_sklearn(x, eps, ms), expect)


@pytest.mark.parametrize("n,order", [(20_000, "random"), (20_000, "ascending"), (20_000, "descending"),
                                     (60_000, "random"), (60_000, "ascending"), (60_000, "descending")])
def test_chains_are_one_component_with_border_ends(n, order):
    x, eps, ms = od.chain(n, order)
    lab, nc = od.dbscan(x, eps, ms)
    assert nc == 1 and (lab == 0).all()
    counts = np.diff(od.neighbourhoods(x, eps)[0])
    ends = np.argsort(x[:, 0])[[0, -1]]
    assert (counts[ends] == 2).all() and np.sort(counts)[2] == 3    # the two ends are border points, the rest core
    if n == 20_000:
        assert np.array_equal(_sklearn(x, eps, ms), lab)


def test_band_is_one_component():
    x, eps, ms = od.band(7_000)
    lab, nc = od.dbscan(x, eps, ms)
    assert nc == 1 and (lab == 0).all() and len(x) == 21_000
    assert np.array_equal(_sklearn(x, eps, ms), lab)


@pytest.mark.parametrize("d,eps,ms", od.TASK_CASES)
def test_task_shaped_cases_oracle_equals_sklearn(d, eps, ms):
    x = od.task_blobs(20_003, d)
    indptr, _ = od.neighbourhoods(x, eps)
    lab, nc = od.dbscan(x, eps, ms)
    assert np.array_equal(lab, _sklearn(x, eps, ms))
    core = np.diff(indptr) >= ms
    border = (~core) & (lab >= 0)
    print(f"d={d} eps={eps} min_samples={ms}: {nc} clusters, {(lab == -1).sum()} noise, {border.sum()} border, "
          f"mean neighbourhood {np.diff(indptr).mean():.1f}")
    assert nc >= 10 and (lab == -1).sum() > 0 and border.sum() > 0
    assert np.diff(indptr).mean() < 200


def test_nonfinite_input_is_rejected_before_device_work():
    """ValueError whether or not a device or the library is present: the check runs before the GPU path (and before
    the optional scikit-learn fallback, which would raise its own ValueError)"""
    from audiomuse_ai_b200 import clustering_gpu as cg
    x = np.random.default_rng(0).standard_normal((50, 4)).astype(np.float32)
    for bad in (np.nan, np.inf, -np.inf):
        y = x.copy()
        y[7, 2] = bad
        with pytest.raises(ValueError, match="NaN or infinity"):
            cg.GPUDBSCAN(0.5, 3).fit_predict(y)
        with pytest.raises(ValueError, match="NaN or infinity"):
            cg.GPUPCA(2).fit_transform(y)
    with pytest.raises(ValueError, match="NaN or infinity"):
        cg.GPUDBSCAN(0.5, 3).fit_predict(np.full((4, 2), 1e39))      # finite in float64, inf in float32
    pca = cg.GPUPCA(2)
    pca.mean_, pca.components_, pca.n_components_, pca.using_gpu = np.zeros(4), np.eye(2, 4), 2, True
    with pytest.raises(ValueError, match="NaN or infinity"):
        pca.transform(np.array([[0.0, np.nan, 0.0, 0.0]]))
