"""One Lloyd step of both k-means paths against the float64 oracle (oracle/kmeans.py), and am_kmeans_fit's trajectory.

Every case runs through am_debug_kmeans_step path 0 (the tensor-core step: split-bf16 wgmma GEMM, fused argmin,
exact recheck of near-ties, accumulate_sorted_kernel) and path 1 (the CUDA-core step: assign_kernel +
accumulate_kernel) on the same operands.  The lattice cases are exact in fp32, so every output must equal the oracle
bit for bit; the other cases hold every label to the acceptance rule and every other output to its bound.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import kmeans as okm

pytestmark = pytest.mark.gpu

TC_MAX_K, TC_MAX_D = 128, 4096


def _tc_ok(d, k):
    return k <= TC_MAX_K and d <= TC_MAX_D


def _bufs(n, d, k):
    import torch
    return (torch.full((n,), -1, dtype=torch.int32, device="cuda"), torch.full((k, d), np.nan, device="cuda"),
            torch.full((k,), np.nan, device="cuda"), torch.zeros(1, device="cuda"), torch.full((n,), np.nan, device="cuda"))


def _host(bufs):
    lab, sums, cnt, inert, dist = bufs
    return dict(labels=lab.cpu().numpy(), sums=sums.cpu().numpy(), counts=cnt.cpu().numpy(),
                inertia=np.float32(inert.item()), dist=dist.cpu().numpy())


def debug_step(path, X, Cn):
    """am_debug_kmeans_step on the named path: labels, sums, counts, inertia (f32), dist"""
    import torch
    from audiomuse_ai_b200 import _lib
    n, d = X.shape
    k = Cn.shape[0]
    xd, cd = torch.from_numpy(X).cuda(), torch.from_numpy(Cn).cuda()
    b = _bufs(n, d, k)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check_debug(_lib.load_debug().am_debug_kmeans_step(
        path, p(xd), n, d, k, p(cd), *[p(t) for t in b], C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return _host(b)


def plan_step(X, Cn):
    """KMeansPlan.step (the path kmeans_use_tensor_cores picks for a plan) -> (outputs, uses_tensor_cores, rechecked)"""
    import torch
    from audiomuse_ai_b200 import dist as amdist
    n, d = X.shape
    k = Cn.shape[0]
    xd, cd = torch.from_numpy(X).cuda(), torch.from_numpy(Cn).cuda()
    b = _bufs(n, d, k)
    plan = amdist.KMeansPlan(xd, k)
    try:
        plan.step(cd, *b)
        torch.cuda.synchronize()
        return _host(b), plan.uses_tensor_cores, plan.last_recheck()
    finally:
        plan.close()


def assign_dev(X, Cn):
    """am_kmeans_assign_dev: labels, sums, counts, inertia"""
    import torch
    from audiomuse_ai_b200 import _lib
    n, d = X.shape
    k = Cn.shape[0]
    xd, cd = torch.from_numpy(X).cuda(), torch.from_numpy(Cn).cuda()
    lab, sums, cnt, inert, _ = _bufs(n, d, k)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(_lib.load().am_kmeans_assign_dev(p(xd), n, d, p(cd), k, p(lab), p(sums), p(cnt), p(inert),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return dict(labels=lab.cpu().numpy(), sums=sums.cpu().numpy(), counts=cnt.cpu().numpy(),
                inertia=np.float32(inert.item()))


# ---------------------------------------------------------------- (a) lattice: bit-exact on both paths
# (N, d, k): every assign_tc_kernel<KP> instance (KP = 16 ... 128), partial and ragged tiles, both
# accumulate_sorted_kernel widths (float4 when d % 4 == 0) with 1 - 8 column passes, and the CUDA-core
# accumulate_kernel slabs W = 128, 64 (k <= 256) and 32 (k > 256); d = 4097 and k > 128 run on CUDA cores only.
LATTICE = [
    (1, 1, 1), (2, 3, 16), (127, 58, 17), (128, 63, 33), (129, 64, 64), (4095, 65, 65), (4097, 200, 96),
    (100_003, 64, 100), (4095, 512, 113), (1000, 513, 128), (300, 1024, 16), (200, 4096, 33), (4095, 4096, 128),
    (500, 4097, 129), (3000, 58, 300), (2000, 3, 1000),
]
_REACHED = {}


def _lattice_check(X, Cn, out, with_dist=True):
    D = okm.distances(X, Cn)
    want = okm.oracle_labels(D)
    np.testing.assert_array_equal(out["labels"], want)
    S, n = okm.sums_exact(X, want, Cn.shape[0])
    np.testing.assert_array_equal(out["counts"], n.astype(np.float32))
    np.testing.assert_array_equal(out["sums"], S.astype(np.float32))
    tot = D[np.arange(len(X)), want].sum()
    assert out["inertia"] == np.float32(tot), (out["inertia"], tot)
    if with_dist:
        np.testing.assert_array_equal(out["dist"].astype(np.float64), D[np.arange(len(X)), want])


@pytest.mark.parametrize("N,d,k", LATTICE)
def test_lattice_step_is_exact(N, d, k):
    X, Cn = okm.lattice(N, d, k, seed=N + d + k)
    paths = (0, 1) if _tc_ok(d, k) else (1,)
    for path in paths:
        _lattice_check(X, Cn, debug_step(path, X, Cn))
    out, tc, _ = plan_step(X, Cn)
    assert tc == _tc_ok(d, k)
    _lattice_check(X, Cn, out)
    _lattice_check(X, Cn, assign_dev(X, Cn), with_dist=False)
    _REACHED[(N, d, k)] = paths


def test_every_branch_is_reached():
    """the lattice cases together reach every value of each axis the kernels branch on"""
    for case in LATTICE:
        if case not in _REACHED:
            test_lattice_step_is_exact(*case)
    tc = [(N, d, k) for (N, d, k), paths in _REACHED.items() if 0 in paths]
    assert {-(-k // 16) * 16 for _, _, k in tc} == {16, 32, 48, 64, 80, 96, 112, 128}
    assert {k for _, _, k in tc} >= {1, 16, 17, 33, 64, 65, 96, 100, 113, 128}
    assert {k for _, _, k in LATTICE if k > TC_MAX_K} == {129, 300, 1000}        # CUDA-core slabs W = 64, 32
    assert {d for _, d, _ in tc} == {1, 3, 58, 63, 64, 65, 200, 512, 513, 1024, 4096}
    assert 4097 in {d for _, d, _ in LATTICE}
    assert {N for N, _, _ in LATTICE} >= {1, 2, 127, 128, 129, 4095, 4097, 100_003}
    # accumulate_sorted_kernel: float4 and scalar loads, one and several 512 / 128-column passes
    passes = {(d % 4 == 0, -(-d // (512 if d % 4 == 0 else 128))) for _, d, _ in tc}
    assert {(True, 1), (True, 2), (True, 8), (False, 1), (False, 5)} <= passes
    # am_kmeans_assign_dev on both paths (tensor cores from N k d >= 2e9)
    assert any(N * d * k >= 2e9 for N, d, k in tc) and any(N * d * k < 2e9 for N, d, k in tc)


# ---------------------------------------------------------------- (b) realistic operands
REALISTIC = {
    "blobs_d58_k40": lambda: okm.blobs(20000, 58, 40, seed=1)[:2],
    "blobs_d200_k100": lambda: okm.blobs(20000, 200, 100, seed=2)[:2],
    "blobs_d512_k128": lambda: okm.blobs(20000, 512, 128, seed=3)[:2],
    "uniform_d1024_k64": lambda: okm.uniform(8000, 1024, 64, seed=4),
    "uniform_d4096_k16": lambda: okm.uniform(4000, 4096, 16, seed=5),
    "uniform_d4097_k200": lambda: okm.uniform(3000, 4097, 200, seed=6),
}


def _bounded_check(X, Cn, out, tensor_cores, D=None, E=None, what=""):
    D = okm.distances(X, Cn) if D is None else D
    E = okm.fp32_errors(X, Cn) if E is None else E
    lab = out["labels"]
    ok = okm.accept(X, Cn, lab, D=D, E=E)
    assert ok.all(), f"{what}: {int((~ok).sum())} rows fail the acceptance rule, e.g. {np.nonzero(~ok)[0][:8]}"
    k = Cn.shape[0]
    S, n = okm.sums_exact(X, lab, k)
    np.testing.assert_array_equal(out["counts"], n.astype(np.float32))
    assert (np.abs(out["sums"].astype(np.float64) - S) <= okm.sums_bound(X, lab, k)).all(), what
    tot, bound = okm.inertia_bound(X, Cn, lab, tensor_cores, D=D)
    assert abs(float(out["inertia"]) - tot) <= bound, (what, float(out["inertia"]), tot, bound)
    if "dist" in out:
        err = np.abs(out["dist"].astype(np.float64) - D[np.arange(len(X)), lab])
        assert (err <= okm.dist_bound(X, Cn, lab, tensor_cores)).all(), what
        return err
    return None


@pytest.mark.parametrize("case", sorted(REALISTIC))
def test_realistic_step_within_bounds(case):
    X, Cn = REALISTIC[case]()
    D, E = okm.distances(X, Cn), okm.fp32_errors(X, Cn)
    d, k = X.shape[1], Cn.shape[0]
    for path in ((0, 1) if _tc_ok(d, k) else (1,)):
        _bounded_check(X, Cn, debug_step(path, X, Cn), path == 0, D, E, f"{case} path {path}")


# ---------------------------------------------------------------- (c) near-tie probes, (d) the error claim measured
PROBE_D = (64, 512, 1024, 4096)


@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("d", PROBE_D)
def test_near_tie_probes_pass_the_rule(d, signed):
    """rows at float64 gaps of 2^-4 ... 2^-24 ||x|| max||c|| between two centres: every label must be as good as the
    fp32 step's.  On the tensor-core path this is the test of the recheck band"""
    X, Cn, _ = okm.probes(d, k=16, per_level=48, signed=signed, seed=d + signed)
    D, E = okm.distances(X, Cn), okm.fp32_errors(X, Cn)
    out = [debug_step(path, X, Cn) for path in (0, 1)]
    for path in (0, 1):
        _bounded_check(X, Cn, out[path], path == 0, D, E, f"d={d} signed={signed} path {path}")
    # a row outside the band is one whose tensor-core label is the exact one; inside, the recheck takes the fp32
    # label: either way the two steps agree on every probe
    np.testing.assert_array_equal(out[0]["labels"], out[1]["labels"])


@pytest.mark.parametrize("d", PROBE_D)
def test_tensor_core_error_claim(d, capsys):
    """|dist - D_label| on the tensor-core step within the documented claim |v~ - v| <= 2^-12 ||x|| max||c|| plus the
    rounding of cn, xn and dist; prints the largest measured error in units of 2^-12 ||x|| max||c||"""
    cases = {"uniform": okm.uniform(6000, d, 64, seed=d), "probes": okm.probes(d, k=16, per_level=32, seed=3 * d)[:2]}
    for name, (X, Cn) in cases.items():
        out, tc, rechecked = plan_step(X, Cn)
        assert tc
        err = _bounded_check(X, Cn, out, True, what=f"{name} d={d}")
        X64 = X.astype(np.float64)
        scale = np.sqrt((X64 ** 2).sum(1)) * np.sqrt((Cn.astype(np.float64) ** 2).sum(1).max())
        with capsys.disabled():
            print(f"\n[kmeans tc error] {name} d={d}: max |dist - D| = {float((err / scale).max()) / 2 ** -12:.4f} "
                  f"x 2^-12 ||x|| cmax, {rechecked}/{len(X)} rows rechecked")


# ---------------------------------------------------------------- (e) scale invariance
@pytest.mark.parametrize("e", [20, -20])
def test_scale_by_power_of_two(e):
    X, Cn = okm.blobs(6000, 200, 100, seed=7)[:2]
    s = np.float32(2.0 ** e)
    Xs, Cs = X * s, Cn * s
    for path in (0, 1):
        a, b = debug_step(path, X, Cn), debug_step(path, Xs, Cs)
        np.testing.assert_array_equal(a["labels"], b["labels"])
        np.testing.assert_array_equal(b["dist"], a["dist"] * np.float32(2.0 ** (2 * e)))
        _bounded_check(Xs, Cs, b, path == 0, what=f"scaled 2^{e} path {path}")


# ---------------------------------------------------------------- (f) Lloyd trajectory of am_kmeans_fit
def _centre_bound(X, lab, k, ref):
    """|c_gpu - c_oracle| for centres of the same rows (`lab`: the E-step labels before any relocation): the fp32 sums
    of the centred rows (n_j terms), the division, and the centring and un-centring roundings (the only error of a
    relocated centre, a copy of one row)"""
    X64 = X.astype(np.float64)
    mu = np.abs(X64.mean(0))
    A, n = okm.sums_exact(np.abs(X64) + mu, lab, k)
    A /= np.maximum(n, 1)[:, None]
    return 2.0 * ((n[:, None] + 4.0) * okm.U * A + okm.U * np.abs(ref)) + 4.0 * okm.U * (np.abs(ref) + mu)


@pytest.mark.parametrize("N,d,k", [(2000, 16, 8), (40000, 64, 32)])   # N k d below / above 5e7: both paths
def test_lloyd_trajectory_matches_float64(N, d, k):
    from audiomuse_ai_b200 import clustering_gpu as cg
    X, cen, _ = okm.separated(N, d, k, seed=N)
    init = (cen + np.random.default_rng(1).normal(0, 3.0, cen.shape)).astype(np.float32)
    traj = okm.lloyd_trajectory(X, init, 11)
    for lab_t, _, _, gap in traj:
        assert gap.min() > 50.0          # no row near a boundary anywhere on the oracle trajectory
    for it in (1, 2, 3, 5, 10):
        c, lab, inertia, n_iter = cg.kmeans_fit(X, k, init_centers=init, max_iter=it, tol=0.0)
        ref_c = traj[it - 1][1]
        np.testing.assert_array_equal(lab, traj[it][0])
        assert (np.abs(c - ref_c) <= _centre_bound(X, traj[it - 1][0], k, ref_c)).all(), it
        tot = okm.distances(X, c)[np.arange(N), lab].sum()
        assert abs(inertia - tot) <= 1e-5 * tot


def _with_outliers(N, d, k, seed):
    X, cen, _ = okm.separated(N, d, k, seed=seed)
    X = X.copy()
    rng = np.random.default_rng(seed)
    for i, r in ((17, 300.0), (99, 220.0)):          # the two rows farthest from their centres, at distinct distances
        u = rng.standard_normal(d)
        X[i] += (r * u / np.linalg.norm(u)).astype(np.float32)
    return X, cen


@pytest.mark.parametrize("n_empty", [1, 2])
@pytest.mark.parametrize("N,d,k", [(2000, 16, 8), (40000, 64, 32)])
def test_relocation_matches_sklearn(N, d, k, n_empty):
    """duplicated initial centres leave 1 or 2 clusters empty after step 1; each takes the farthest row, as
    scikit-learn's _relocate_empty_clusters_dense does (the oracle calls it), in am_kmeans_fit and in
    kmeans_lloyd_sharded at world size 1"""
    import torch
    from audiomuse_ai_b200 import clustering_gpu as cg, dist as amdist
    X, cen = _with_outliers(N, d, k, seed=N + n_empty)
    init = cen.copy()
    init[5] = init[2]
    if n_empty == 2:
        init[6] = init[3]
    traj = okm.lloyd_trajectory(X, init, 4)
    assert (traj[0][2] == 0).sum() == n_empty
    for it in (1, 2, 3):
        c, lab, _, _ = cg.kmeans_fit(X, k, init_centers=init, max_iter=it, tol=0.0)
        np.testing.assert_array_equal(lab, traj[it][0])
        ref_c = traj[it - 1][1]
        assert (np.abs(c - ref_c) <= _centre_bound(X, traj[it - 1][0], k, ref_c)).all(), it
        c2, lab2, _, _ = amdist.kmeans_lloyd_sharded(torch.from_numpy(X).cuda(), torch.from_numpy(init).cuda(),
                                                     max_iter=it, tol=0.0)
        np.testing.assert_array_equal(lab2.cpu().numpy(), traj[it][0])
        assert (np.abs(c2.cpu().numpy() - ref_c) <= _centre_bound(X, traj[it - 1][0], k, ref_c)).all(), it


def test_more_clusters_than_distinct_rows():
    """every row on its centre: no relocation, the empty cluster moves to the first largest cluster (scikit-learn)"""
    from audiomuse_ai_b200 import clustering_gpu as cg
    from sklearn.cluster import KMeans
    import warnings
    X = np.repeat(np.array([[1.0, 2.0], [4.0, 0.0], [-3.0, 5.0]], np.float32), 4, axis=0)
    init = np.array([[1, 2], [4, 0], [-3, 5], [1, 2]], np.float32)
    for it in (1, 2):
        lab_ref, c_ref, _ = okm.lloyd_step(X, init)
        c, lab, inertia, _ = cg.kmeans_fit(X, 4, init_centers=init, max_iter=it, tol=0.0)
        np.testing.assert_array_equal(lab, lab_ref)
        np.testing.assert_allclose(c, c_ref, rtol=0, atol=1e-5)
        assert inertia <= 1e-9
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            km = KMeans(4, init=init, n_init=1, max_iter=it, tol=0).fit(X)
        np.testing.assert_allclose(c, km.cluster_centers_, rtol=0, atol=1e-5)


# ---------------------------------------------------------------- (g) data far from the origin
@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3, 1e4])
@pytest.mark.parametrize("N", [20000, 60000])     # N k d = 2e7 (CUDA cores) and 6.1e7 (tensor cores)
def test_offset_data_matches_sklearn(N, offset):
    """am_kmeans_fit centres the rows as sklearn's KMeans.fit does: the labels are scikit-learn's apart from the rows
    the oracle names as boundary rows, and the inertia is the float64 one of the returned labels and centres"""
    from sklearn.cluster import KMeans
    from audiomuse_ai_b200 import clustering_gpu as cg
    k, d = 16, 64
    X, cen, _ = okm.blobs(N, d, k, seed=21, offset=offset, spread=2.0)
    init = (cen + np.random.default_rng(2).normal(0, 0.5, cen.shape)).astype(np.float32)
    km = KMeans(k, init=init, n_init=1, tol=0.0).fit(X)   # tol = 0: both sides run to the fixed point
    D_ref = okm.distances(X, km.cluster_centers_.astype(np.float32))
    srt = np.sort(D_ref, axis=1)
    boundary = srt[:, 1] - srt[:, 0] <= 1e-3
    assert boundary.mean() < 1e-3
    fits = [cg.kmeans_fit(X, k, init_centers=init, tol=0.0)]
    m = cg.GPUKMeans(k, init=init, n_init=1, tol=0.0)
    m.fit_predict(X)
    fits.append((m.cluster_centers_, m.labels_, m.inertia_, m.n_iter_))
    for c, lab, inertia, _ in fits:
        diff = (lab != km.labels_) & ~boundary
        assert not diff.any(), f"offset {offset}: {int(diff.sum())} rows differ from scikit-learn"
        tot = okm.distances(X, c)[np.arange(N), lab].sum()
        assert abs(inertia - tot) <= 1e-4 * tot, (offset, inertia, tot)
