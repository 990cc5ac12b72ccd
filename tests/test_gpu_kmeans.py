"""K5 parity vs the reference's CPU branch (sklearn KMeans) from an identical initialisation."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import kmeans as okm


def _data(n=20000, d=64, k=16, seed=7):
    from audiomuse_ai_b200 import corpus
    return corpus.kmeans_library(n, d, k, seed)


def test_lloyd_matches_sklearn_from_same_init():
    from sklearn.metrics import adjusted_rand_score
    from audiomuse_ai_b200 import clustering_gpu as cg
    x, true_lab, _ = _data()
    rng = np.random.default_rng(0)
    init = x[rng.choice(len(x), 16, replace=False)]
    c, lab, inertia, it = cg.kmeans_fit(x, 16, init_centers=init, max_iter=300, tol=1e-4)
    c_ref, lab_ref, inertia_ref, _ = okm.sklearn_fit(x, 16, init)
    assert abs(inertia - inertia_ref) <= 0.01 * inertia_ref
    assert adjusted_rand_score(lab, lab_ref) >= 0.99
    assert lab.dtype == np.int32 and c.shape == (16, 64)
    _, inertia_chk = okm.assign(x, c)
    assert abs(inertia - inertia_chk) <= 1e-3 * inertia_chk      # inertia is consistent with labels/centres


def test_empty_cluster_relocation_matches_sklearn():
    """Two identical initial centres leave one cluster empty after the first E-step (ties go to the lower
    index).  sklearn's Lloyd hands it the point farthest from its own centre (_relocate_empty_clusters_dense);
    am_kmeans_fit and the sharded loop do the same, so the whole trajectory matches."""
    import torch
    from audiomuse_ai_b200 import clustering_gpu as cg, dist as amdist
    x, _, _ = _data(20000, 32, 12, 11)
    init = x[np.random.default_rng(4).choice(len(x), 12, replace=False)].copy()
    init[7] = init[2]
    c, lab, inertia, it = cg.kmeans_fit(x, 12, init_centers=init, max_iter=300, tol=1e-4)
    c_ref, lab_ref, inertia_ref, _ = okm.sklearn_fit(x, 12, init)
    assert np.bincount(lab, minlength=12).min() > 0
    assert abs(inertia - inertia_ref) <= 1e-4 * inertia_ref
    assert (lab == lab_ref).mean() > 0.999
    np.testing.assert_allclose(c, c_ref, atol=1e-4)
    c2, lab2, inertia2, _ = amdist.kmeans_lloyd_sharded(torch.from_numpy(x).cuda(), torch.from_numpy(init).cuda())
    assert abs(inertia2 - inertia_ref) <= 1e-3 * inertia_ref
    assert (lab2.cpu().numpy() == lab_ref).mean() > 0.999


def test_gpukmeans_interface_and_kmeanspp():
    from sklearn.metrics import adjusted_rand_score
    from audiomuse_ai_b200 import clustering_gpu as cg
    x, true_lab, _ = _data(30000, 200, 40, 3)
    m = cg.get_clustering_model("kmeans", {"n_clusters": 40}, use_gpu=True)
    assert isinstance(m, cg.GPUKMeans) and m.n_init == 10
    m.n_init = 3
    m.random_state = 1
    labels = m.fit_predict(x)
    assert m.using_gpu and m.cluster_centers_.shape == (40, 200) and labels.shape == (30000,)
    assert (m.labels_ == labels).all()
    # k-means++ restarts land in (different) local optima: compare the objective with the reference's
    # CPU branch (sklearn, same n_init) rather than the labels
    from sklearn.cluster import KMeans
    ref = KMeans(n_clusters=40, init="k-means++", n_init=3, random_state=1).fit(x)
    assert m.inertia_ <= 1.05 * ref.inertia_
    assert adjusted_rand_score(labels, true_lab) >= 0.85
    assert cg.check_gpu_available()


def test_assign_dev_partial_sums_match_numpy():
    import ctypes as C
    import torch
    from audiomuse_ai_b200 import _lib
    lib = _lib.load()
    x, _, centers = _data(5000, 96, 8, 11)
    xd = torch.from_numpy(x).cuda(); cd = torch.from_numpy(centers).cuda()
    lab = torch.empty(5000, dtype=torch.int32, device="cuda")
    sums = torch.empty(8, 96, device="cuda"); cnt = torch.empty(8, device="cuda"); inert = torch.empty(1, device="cuda")
    _lib.check(lib.am_kmeans_assign_dev(xd.data_ptr(), 5000, 96, cd.data_ptr(), 8, lab.data_ptr(), sums.data_ptr(),
                                        cnt.data_ptr(), inert.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    got = lab.cpu().numpy()
    assert okm.accept(x, centers, got).all()
    S, n = okm.sums_exact(x, got, 8)
    np.testing.assert_array_equal(cnt.cpu().numpy(), n.astype(np.float32))
    assert (np.abs(sums.cpu().numpy() - S) <= okm.sums_bound(x, got, 8)).all()
    tot, bound = okm.inertia_bound(x, centers, got, tensor_cores=False)
    assert abs(float(inert.item()) - tot) <= bound


def test_sharded_lloyd_single_rank_matches_fit():
    """dist.kmeans_lloyd_sharded (the multi-GPU Lloyd loop; world size 1 here: the all-reduces are no-ops)
    reaches the same fixed point as am_kmeans_fit from the same initial centres."""
    import torch
    from audiomuse_ai_b200 import clustering_gpu as cg, dist as amdist
    x, _, _ = _data(40000, 128, 24, 5)
    init = x[np.random.default_rng(1).choice(len(x), 24, replace=False)]
    xd, initd = torch.from_numpy(x).cuda(), torch.from_numpy(init).cuda()
    # (a) the same number of Lloyd iterations on both sides (tol = 0: no early stop): centres agree to rounding
    #     (the partial sums are added in another order; a near-tie row may flip and moves a centre by ~|x - c| / count)
    c_ref, lab_ref, inertia_ref, _ = cg.kmeans_fit(x, 24, init_centers=init, max_iter=12, tol=0.0)
    c, lab, inertia, it = amdist.kmeans_lloyd_sharded(xd, initd, max_iter=12, tol=0.0)
    assert abs(inertia - inertia_ref) <= 1e-4 * inertia_ref
    assert (lab.cpu().numpy() == lab_ref).mean() > 0.9995
    np.testing.assert_allclose(c.cpu().numpy(), c_ref, atol=5e-4)
    # (b) with the default tolerance the stopping test (shift^2 <= tol * var) may fire a few iterations apart (late iterations move one or two near-tie rows, shift^2 hovers at tol * var), so the
    #     centres agree to the tolerance's scale only
    c_ref, lab_ref, inertia_ref, it_ref = cg.kmeans_fit(x, 24, init_centers=init)
    c, lab, inertia, it = amdist.kmeans_lloyd_sharded(xd, initd)
    assert it < 300 and it_ref < 300, (it, it_ref)   # both converged
    assert abs(inertia - inertia_ref) <= 1e-3 * inertia_ref
    assert (lab.cpu().numpy() == lab_ref).mean() > 0.999
    assert np.abs(c.cpu().numpy() - c_ref).max() <= 2e-3


def test_config4_scale_properties():
    """BASELINE.json configs[3] shape (d = 512, k = 128) at 200 k rows: size-independent properties --
    labels are the argmin over the returned centres, inertia matches, every Lloyd step lowers inertia."""
    from audiomuse_ai_b200 import clustering_gpu as cg
    x, _, centers = _data(200_000, 512, 128, 7)
    rng = np.random.default_rng(2)
    init = x[rng.choice(len(x), 128, replace=False)]
    c1, l1, i1, _ = cg.kmeans_fit(x, 128, init_centers=init, max_iter=1)
    c5, l5, i5, it = cg.kmeans_fit(x, 128, init_centers=init, max_iter=5)
    assert i5 <= i1 * (1 + 1e-6) and it <= 5
    sub = rng.choice(len(x), 4000, replace=False)
    assert okm.accept(x[sub], c5, l5[sub]).all()
    _, inertia_chk = okm.assign(x[sub], c5)
    d2 = ((x[sub].astype(np.float64) - c5[l5[sub]].astype(np.float64)) ** 2).sum()
    assert abs(d2 - inertia_chk) <= 1e-3 * inertia_chk


@pytest.mark.parametrize("n,d,k,kind", [(60000, 512, 128, "clustered"), (40000, 200, 100, "clustered"),
                                        (30000, 58, 40, "uniform"), (20000, 96, 7, "uniform")])
def test_tensor_core_step_equals_debug_exact_step(n, d, k, kind):
    """am_kmeans_plan_step (split-bf16 wgmma GEMM + fused argmin + exact recheck of near-ties) returns the SAME
    labels as the exact fp32 CUDA-core step that am_debug_kmeans_step path 1 runs on the same shape -- on clustered
    data and on structureless data, where a large share of the points is a near-tie -- and matching counts / sums /
    inertia.  d = 58, 200 and k in [40, 100] are the reference's shapes (clustering_helper.py), 512 / 128 is
    config 4."""
    import ctypes as C
    import json
    import torch
    from audiomuse_ai_b200 import _lib, dist as amdist
    if kind == "clustered":
        x, _, cen = _data(n, d, k, 5)
        centers = cen + 0.02 * np.random.default_rng(0).standard_normal(cen.shape).astype(np.float32)
    else:
        x = np.random.default_rng(1).random((n, d), dtype=np.float32)
        centers = x[np.random.default_rng(2).choice(n, k, replace=False)].copy()
    xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(centers).cuda()
    out = {}
    for mode in ("tc", "simt"):
        lab = torch.empty(n, dtype=torch.int32, device="cuda")
        sums = torch.empty(k, d, device="cuda"); cnt = torch.empty(k, device="cuda"); inert = torch.zeros(1, device="cuda")
        dist = torch.empty(n, device="cuda")
        if mode == "tc":
            plan = amdist.KMeansPlan(xd, k)
            assert plan.uses_tensor_cores
            plan.step(cd, lab, sums, cnt, inert, dist)
            torch.cuda.synchronize()
            plan.close()
        else:
            p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
            dbg = _lib.load_debug()
            dbg.am_profile_enable(1)
            _lib.check_debug(dbg.am_debug_kmeans_step(
                1, p(xd), n, d, k, p(cd), p(lab), p(sums), p(cnt), p(inert), p(dist),
                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            size = dbg.am_profile_report(None, 0)
            buf = C.create_string_buffer(size + 16)
            dbg.am_profile_report(buf, size + 16)
            dbg.am_profile_enable(0)
            kernels = json.loads(buf.value.decode() or "{}")
            # the exact side ran on CUDA cores: assign_kernel, no tensor-core assignment
            assert "assign_kernel" in kernels and not any(kk.startswith("assign_tc_kernel") for kk in kernels), kernels
        out[mode] = (lab.cpu().numpy(), sums.cpu().numpy(), cnt.cpu().numpy(), float(inert.item()), dist.cpu().numpy())
    np.testing.assert_array_equal(out["tc"][0], out["simt"][0])
    np.testing.assert_array_equal(out["tc"][2], out["simt"][2])
    np.testing.assert_allclose(out["tc"][1], out["simt"][1], rtol=2e-5, atol=2e-3)
    assert abs(out["tc"][3] - out["simt"][3]) <= 1e-5 * out["simt"][3]
    np.testing.assert_allclose(out["tc"][4], out["simt"][4], rtol=0, atol=2e-3 * max(1.0, float(out["simt"][4].max())))
    assert okm.accept(x, centers, out["tc"][0]).all()              # float64 oracle, every row


def test_plan_path_follows_the_shape():
    """A plan takes the tensor-core step for every shape it can serve (k <= 128, d <= 4096) and the CUDA-core step
    beyond either limit (kmeans_use_tensor_cores in kmeans.cu)."""
    import torch
    from audiomuse_ai_b200 import dist as amdist
    x = torch.zeros(300, 4097, device="cuda")
    for k, d, want in ((128, 512, True), (129, 512, False), (40, 4097, False)):
        plan = amdist.KMeansPlan(x[:, :d].contiguous(), k)
        assert plan.uses_tensor_cores == want, (k, d)
        plan.close()
