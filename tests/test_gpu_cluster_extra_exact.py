"""DBSCAN and PCA on the device (csrc/cluster_extra.cu) against exact float64 references, at the shapes, settings and
inputs where the kernels can go wrong: ragged tiles, degenerate settings, pairs at eps to within 2^-23, quantised
coordinates, border points between clusters, components that span the whole index range, and PCA data far from the
origin.  DBSCAN labels and n_clusters_ must equal oracle/dbscan.py exactly; the cases themselves are checked in
test_cluster_extra_host.py."""
import numpy as np
import pytest

from oracle import dbscan as od

pytestmark = pytest.mark.gpu


def _dbscan_equals(x, eps, ms, want=None, what=""):
    from audiomuse_ai_b200 import clustering_gpu as cg
    if want is None:
        want, n_want = od.dbscan(x, eps, ms)
    else:
        n_want = len(set(want.tolist()) - {-1})
    model = cg.GPUDBSCAN(eps, ms)
    got = model.fit_predict(x)
    assert model.using_gpu
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{what}: {bad.size} labels differ, first at {bad[:5]}: got {got[bad[:5]]}, want {want[bad[:5]]}"
    assert model.n_clusters_ == n_want, (what, model.n_clusters_, n_want)


@pytest.mark.parametrize("d", od.RAGGED_D)
@pytest.mark.parametrize("n", od.RAGGED_N)
def test_dbscan_ragged_sizes(n, d):
    x, eps, ms = od.ragged(n, d)
    _dbscan_equals(x, eps, ms, what=f"n={n} d={d}")


@pytest.mark.parametrize("case", [c[0] for c in od.degenerate()])
def test_dbscan_degenerate_settings(case):
    (name, x, eps, ms), = [c for c in od.degenerate() if c[0] == case]
    _dbscan_equals(x, eps, ms, what=name)


@pytest.mark.parametrize("d", [2, 64, 512])
def test_dbscan_near_eps_probes(d):
    """a probe at eps (1 +- 2^-k) from a core blob, k = 8 .. 23: from well outside the fp32 band to its float64 recheck"""
    for k in range(8, 24):
        for sign in (1, -1):
            x, eps, ms, inside = od.probe(d, k, sign)
            want = np.array([0, 0, -1, 0, 0 if inside else -1, 0], np.int32)
            _dbscan_equals(x, eps, ms, want, what=f"d={d} k={k} sign={sign}")


@pytest.mark.parametrize("dim,side,eps,ms", od.LATTICE_CASES)
def test_dbscan_quantised_coordinates(dim, side, eps, ms):
    """spacing float32(0.1): eps 0.1 / 0.2 / 0.3 are decided by the float64 square of eps, not by its float32 one"""
    _dbscan_equals(od.lattice(dim, side), eps, ms, what=f"{dim}-D lattice eps={eps}")


def test_dbscan_border_point_joins_first_cluster_not_nearest():
    x, eps, ms, want = od.border_between_clusters()
    _dbscan_equals(x, eps, ms, want, what="border")


@pytest.mark.parametrize("order", ["random", "ascending", "descending"])
@pytest.mark.parametrize("n", [20_000, 60_000])
def test_dbscan_long_chain_is_one_cluster(n, order):
    """a component whose diameter is the whole data set, in any index order: one cluster, ends included"""
    x, eps, ms = od.chain(n, order)
    _dbscan_equals(x, eps, ms, np.zeros(n, np.int32), what=f"{n} {order}")


def test_dbscan_band_is_one_cluster():
    x, eps, ms = od.band(7_000)
    _dbscan_equals(x, eps, ms, np.zeros(len(x), np.int32), what="band")


@pytest.mark.parametrize("d,eps,ms", od.TASK_CASES)
def test_dbscan_task_shaped(d, eps, ms):
    _dbscan_equals(od.task_blobs(20_003, d), eps, ms, what=f"d={d} eps={eps} min_samples={ms}")


def test_nonfinite_input_raises_before_device_work():
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    x = np.random.default_rng(0).standard_normal((200, 6)).astype(np.float32)
    pca = cg.GPUPCA(3)
    pca.fit_transform(x)
    assert pca.using_gpu
    before = _lib.launch_count()
    for bad in (np.nan, np.inf):
        y = x.copy()
        y[13] = bad
        with pytest.raises(ValueError):
            cg.GPUDBSCAN(0.5, 3).fit_predict(y)
        with pytest.raises(ValueError):
            cg.GPUPCA(3).fit_transform(y)
        with pytest.raises(ValueError):
            pca.transform(y[10:20])
    assert _lib.launch_count() == before


# ---------------------------------------------------------------- PCA
def _moment_cases():
    out = []
    for d in (1, 2, 63, 64, 65, 129, 1000):
        for n in sorted({2, 3, d - 1, 100_003}):
            if n >= 2:
                out.append((d, n))
    return out


@pytest.mark.parametrize("d,n", _moment_cases())
def test_pca_moments_against_float64(d, n):
    from audiomuse_ai_b200 import _lib
    rng = np.random.default_rng(d * 7 + n)
    x = (rng.standard_normal((n, d)) * rng.uniform(0.5, 2.0, d) + 3.0).astype(np.float32)
    mean, cov = np.empty(d), np.empty((d, d))
    _lib.check(_lib.load().am_pca_moments(_lib.ptr(x), n, d, _lib.ptr(mean), _lib.ptr(cov)))
    x64 = x.astype(np.float64)
    m_ref = x64.mean(0)
    xc = x64 - m_ref
    c_ref = xc.T @ xc / (n - 1)
    sd = np.sqrt(np.diag(c_ref))
    assert np.all(np.abs(mean - m_ref) <= 1e-10 * sd), np.abs(mean - m_ref).max()
    err = np.abs(cov - c_ref) / np.outer(sd, sd)
    assert err.max() <= 1e-10, err.max()


def _offset_data(offset, n, d=64, seed=0):
    """spread about 1 (principal scales 1.5 .. 0.3, randomly rotated) around a centre of about `offset` per coordinate"""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    z = rng.standard_normal((n, d)) * np.linspace(1.5, 0.3, d)
    return (z @ q.T + offset * (1 + 0.5 * rng.random(d))).astype(np.float32)


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e4])
def test_pca_projection_far_from_origin(offset):
    """the projection centres against the float64 mean: a float32 mean is off by |mean| 2^-24 per coordinate"""
    from sklearn.decomposition import PCA
    from audiomuse_ai_b200 import clustering_gpu as cg
    x = _offset_data(offset, 4000)
    ref = PCA(n_components=8, svd_solver="full")
    y_ref = ref.fit_transform(x.astype(np.float64))
    got = cg.GPUPCA(8)
    y = got.fit_transform(x)
    assert got.using_gpu
    sign = np.sign(np.sum(got.components_ * ref.components_, axis=1))
    err = np.abs(y * sign[None, :] - y_ref).max() / np.abs(y_ref).max()
    assert err <= 2e-6, err


@pytest.mark.parametrize("offset", [0.0, 1e3])
def test_pca_transform_unseen_rows(offset):
    from sklearn.decomposition import PCA
    from audiomuse_ai_b200 import clustering_gpu as cg
    x = _offset_data(offset, 3500, seed=1)
    fit, new = x[:3000], x[3000:]
    ref = PCA(n_components=8, svd_solver="full").fit(fit.astype(np.float64))
    got = cg.GPUPCA(8)
    got.fit_transform(fit)
    for rows in (new, new[:1], new[-1:]):
        y_ref = ref.transform(rows.astype(np.float64))
        y = got.transform(rows)
        assert y.shape == y_ref.shape
        sign = np.sign(np.sum(got.components_ * ref.components_, axis=1))
        err = np.abs(y * sign[None, :] - y_ref).max() / np.abs(ref.transform(new.astype(np.float64))).max()
        assert err <= 2e-6, (len(rows), err)
