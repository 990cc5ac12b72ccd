"""am_kmeans_fit_batch (csrc/kmeans_batch.cu) through clustering_gpu.kmeans_fit_batch: the k-means++ rows against a
numpy restatement of the greedy seeding on the same SplitMix draws, Lloyd steps against the float64 oracle
(oracle/kmeans.py), whole fits against am_kmeans_fit on the same problem and seed, determinism and independence from
the rest of the batch, and the input checks."""
import math

import numpy as np
import pytest

from oracle import kmeans as okm
from tests.test_gpu_kmeans_exact import _centre_bound

pytestmark = pytest.mark.gpu

MASK = (1 << 64) - 1


def splitmix_uniforms(seed, n):
    """the n first uniforms of am_kmeans_fit's seeding generator (kmeans_common.cuh)"""
    s = (seed ^ 0x5851f42d4c957f2d) & MASK
    out = np.empty(n)
    for i in range(n):
        s = (s + 0x9e3779b97f4a7c15) & MASK
        z = s
        z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & MASK
        z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & MASK
        z ^= z >> 31
        out[i] = (z >> 11) * (1.0 / 9007199254740992.0)
    return out


def trials(k):
    return min(8, 2 + int(math.log(k)))


def restated_seeding(X, k, u, gpu_rows, rel=1e-6):
    """greedy k-means++ in float64 on the float32 rows shifted by their float32 column means, drawing from u.  A step
    is clear when every cumulative-sum boundary is more than rel of the total from its draw and the best trial's
    potential leads by more than 2 rel (the fp32 D^2 chains are within (ceil(d / 32) + 5) 2^-24 of each term); after
    a step that is not, the restatement follows the device's row.  -> (restated rows, clear flags)"""
    Xs = (X - X.astype(np.float64).mean(0).astype(np.float32)).astype(np.float32).astype(np.float64)
    N = len(Xs)
    L = trials(k)
    rows = [min(int(u[0] * N), N - 1)]
    clear = [True]
    m2 = ((Xs - Xs[rows[0]]) ** 2).sum(1)
    for j in range(1, k):
        tot = m2.sum()
        cum = np.cumsum(m2)
        cands, ok = [], tot > 0
        for l in range(L):
            r = u[1 + (j - 1) * L + l] * tot
            i = min(int(np.searchsorted(cum, r, side="right")), N - 1)
            lo = cum[i - 1] if i else 0.0
            ok &= min(r - lo, cum[i] - r) > rel * tot
            cands.append(i)
        pot = {c: np.minimum(m2, ((Xs - Xs[c]) ** 2).sum(1)).sum() for c in cands}
        srt = np.sort(list(pot.values()))  # a row drawn twice ties with itself, which decides nothing
        ok &= len(srt) < 2 or srt[1] - srt[0] > 2 * rel * srt[0]
        best = cands[int(np.argmin([pot[c] for c in cands]))]
        rows.append(best)
        clear.append(bool(ok))
        m2 = np.minimum(m2, ((Xs - Xs[best if ok else gpu_rows[j]]) ** 2).sum(1))
    return np.array(rows), np.array(clear)


@pytest.mark.parametrize("k", [1, 2, 40, 100])
def test_seeding_matches_the_restatement(k):
    from audiomuse_ai_b200 import clustering_gpu as cg
    probs = [okm.blobs(k, 31, max(1, k // 3), seed=k)[0], okm.blobs(700, 31, 12, seed=k + 1, offset=5.0)[0]]
    n_init = 3
    res = cg.kmeans_fit_batch(probs, k, n_init=n_init, seeds=[7, 11], intermediates=True)
    per = 1 + (k - 1) * trials(k)
    for X, seed, (_, _, _, _, kpp) in zip(probs, (7, 11), res):
        u = splitmix_uniforms(seed, n_init * per)
        for r in range(n_init):
            want, clear = restated_seeding(X, k, u[r * per:(r + 1) * per], kpp[r])
            if not clear.all():
                print(f"k={k} N={len(X)} init {r}: {int((~clear).sum())} of {k} steps below the restatement's margin")
            assert clear.mean() >= 0.8, f"k={k} init {r}: only {int(clear.sum())} of {k} steps clear the margin"
            np.testing.assert_array_equal(kpp[r][clear], want[clear])
            if len(X) == k:  # distinct rows: D^2 sampling never repeats a row while another has weight
                assert sorted(kpp[r].tolist()) == list(range(k))


@pytest.mark.parametrize("N,d,k", [(2000, 16, 8), (6000, 50, 40)])
def test_lloyd_steps_follow_the_float64_trajectory(N, d, k):
    """with n_init = 1 the k-means++ rows are the initial centres; after max_iter steps the labels pass the acceptance
    rule at the returned centres and the centres are within the sums bound of the float64 trajectory"""
    from audiomuse_ai_b200 import clustering_gpu as cg
    X, _, _ = okm.separated(N, d, k, seed=N + d)
    for it in (1, 2, 3):
        c, lab, inertia, n_iter, kpp = cg.kmeans_fit_batch([X], k, n_init=1, max_iter=it, tol=0.0,
                                                           intermediates=True)[0]
        assert 1 <= n_iter <= it  # with tol = 0 a fit stops early only where the centres stopped moving
        assert okm.accept(X, c, lab).all()
        traj = okm.lloyd_trajectory(X, X[kpp[0]], n_iter)
        if min(g.min() for *_, g in traj) <= 1e-3:
            print(f"N={N} k={k} max_iter={it}: a row within 1e-3 of a boundary on the oracle trajectory")
            continue
        ref = traj[-1][1]
        assert (np.abs(c - ref) <= _centre_bound(X, traj[-1][0], k, ref)).all(), it
        tot = okm.distances(X, c)[np.arange(N), lab].sum()
        assert abs(inertia - tot) <= 1e-5 * tot


def test_more_clusters_than_distinct_rows_matches_kmeans_fit():
    """every row on its centre: the empty clusters move to the first largest cluster, as am_kmeans_fit does it
    (test_gpu_kmeans_exact.py holds am_kmeans_fit to scikit-learn on this case)"""
    from audiomuse_ai_b200 import clustering_gpu as cg
    X = np.repeat(np.array([[1.0, 2.0], [4.0, 0.0], [-3.0, 5.0]], np.float32), 4, axis=0)
    c, lab, inertia, _ = cg.kmeans_fit_batch([X], 4, n_init=2)[0]
    c_ref, lab_ref, inertia_ref, _ = cg.kmeans_fit(X, 4, n_init=2)
    np.testing.assert_array_equal(lab, lab_ref)
    np.testing.assert_allclose(c, c_ref, rtol=0, atol=1e-5)
    assert inertia <= 1e-9


def _ragged_batch():
    """>= 20 problems: N from k to 40 000, d in {1, 31, 32, 33, 50, 199, 200}, k from 2 to 100 with k = N, rows far
    from the origin and duplicated rows"""
    rng = np.random.default_rng(5)
    shapes = [(40000, 200, 100), (10000, 50, 70), (2000, 1, 2), (3000, 31, 40), (2500, 32, 41), (2600, 33, 42),
              (5000, 199, 60), (4000, 200, 100), (100, 50, 100), (60, 31, 60), (2, 33, 2), (800, 1, 5),
              (12000, 50, 40), (2000, 200, 99), (1500, 32, 3), (3000, 33, 64), (900, 199, 10), (20000, 31, 50),
              (700, 50, 45), (5000, 1, 30), (300, 200, 2)]
    probs = []
    for i, (N, d, k) in enumerate(shapes):
        X = okm.blobs(N, d, max(2, k // 2), seed=100 + i, spread=3.0, offset=(1e3 if i % 5 == 1 else 0.0))[0]
        if i % 4 == 3:  # duplicated rows
            X[N // 2:] = X[rng.integers(0, N // 2, N - N // 2)]
        probs.append((X, k, 1000 + i))
    X = np.repeat(okm.blobs(10, 33, 3, seed=9)[0], 5, axis=0)  # 10 distinct rows, k = 12 > 10
    probs.append((X, 12, 77))
    return probs


def unexplained_label_differences(X, c, c_ref, lab, lab_ref):
    """rows whose labels differ between the two drivers although no near tie explains it: a row can change its label
    between centre sets c and c_ref only when the gap between its two nearest c_ref centres is at most the fp32
    rule's slack plus what moving the centres by |c - c_ref| can change, 2 ||x - c_j|| ||c_j - c_ref_j|| +
    ||c_j - c_ref_j||^2 for each of the two centres.  -> (rows that differ, of them those not near a tie)"""
    diff = np.flatnonzero(lab != lab_ref)
    if not len(diff):
        return diff, diff
    D = okm.distances(X[diff], c_ref)
    gap, slack = okm.margins(D, okm.fp32_errors(X[diff], c_ref))
    move = np.sqrt(((c.astype(np.float64) - c_ref.astype(np.float64)) ** 2).sum(1)).max()
    shift = 2.0 * (2.0 * np.sqrt(np.sort(D, axis=1)[:, :2]).sum(1) * move + 2.0 * move * move)
    return diff, diff[gap > 4.0 * slack + shift]


def test_whole_fits_match_kmeans_fit():
    """labels and n_iter as am_kmeans_fit's on the same problem and seed, inertia within 1e-6 relative (1e-4 where
    am_kmeans_fit's tensor-core step computes it), centres within the sums bound.  A problem whose final centres
    differs from am_kmeans_fit only at rows that the two drivers' centres (am_kmeans_fit sums with float atomics)
    leave within a near tie is reported; a label difference anywhere else fails."""
    from audiomuse_ai_b200 import clustering_gpu as cg
    probs = _ragged_batch()
    res = cg.kmeans_fit_batch([p[0] for p in probs], [p[1] for p in probs], seeds=[p[2] for p in probs])
    held = 0
    for (X, k, seed), (c, lab, inertia, n_iter) in zip(probs, res):
        N, d = X.shape
        c_ref, lab_ref, inertia_ref, n_iter_ref = cg.kmeans_fit(X, k, seed=seed)
        assert okm.accept(X, c, lab).all(), (N, d, k)
        diff, wrong = unexplained_label_differences(X, c, c_ref, lab, lab_ref)
        assert not len(wrong), f"N={N} d={d} k={k}: {len(wrong)} of {len(diff)} differing rows are not near a tie"
        if len(diff):
            print(f"N={N} d={d} k={k}: {len(diff)} labels differ, every one at a near tie")
            continue
        held += 1
        np.testing.assert_array_equal(lab, lab_ref, err_msg=f"N={N} d={d} k={k}")
        assert n_iter == n_iter_ref, (N, d, k, n_iter, n_iter_ref)
        # both are fp32 distances summed in float64: 1e-6 relative, or the oracle's inertia bound where the
        # expansion's cancellation (small d, rows far from their centres' scale) is larger
        rel = 1e-6 if N * k * d < 5e7 else 1e-4
        tol = max(rel * inertia_ref, okm.inertia_bound(X, c, lab, False)[1] +
                  okm.inertia_bound(X, c_ref, lab_ref, N * k * d >= 5e7)[1])
        assert abs(inertia - inertia_ref) <= tol, (N, d, k, inertia, inertia_ref, tol)
        assert (np.abs(c - c_ref) <= 2.0 * _centre_bound(X, lab, k, c_ref.astype(np.float64))).all(), (N, d, k)
    assert held >= len(probs) - 3, f"only {held} of {len(probs)} problems clear the margins"


def test_deterministic_and_independent_of_the_batch():
    from audiomuse_ai_b200 import clustering_gpu as cg
    probs = _ragged_batch()[1:9]
    Xs, ks, seeds = [p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs]
    a = cg.kmeans_fit_batch(Xs, ks, seeds=seeds, intermediates=True)
    b = cg.kmeans_fit_batch(Xs, ks, seeds=seeds, intermediates=True)
    rev = cg.kmeans_fit_batch(Xs[::-1], ks[::-1], seeds=seeds[::-1], intermediates=True)[::-1]
    alone = cg.kmeans_fit_batch([Xs[3]], ks[3], seeds=seeds[3], intermediates=True)
    for x, y, z in zip(a, b, rev):
        for u, v, w in zip(x, y, z):
            assert np.array_equal(np.asarray(u), np.asarray(v)) and np.array_equal(np.asarray(u), np.asarray(w))
    for u, v in zip(a[3], alone[0]):
        assert np.array_equal(np.asarray(u), np.asarray(v))


def test_input_checks_before_device_work():
    from audiomuse_ai_b200 import _lib, clustering_gpu as cg
    X = np.random.default_rng(0).random((50, 4), dtype=np.float32)
    for bad in (np.nan, np.inf):
        Y = X.copy()
        Y[7, 2] = bad
        with pytest.raises(ValueError, match="NaN or infinity"):
            cg.kmeans_fit_batch([X, Y], 3)
    with pytest.raises(ValueError, match="should be >= n_clusters"):
        cg.kmeans_fit_batch([X], 51)
    with pytest.raises(ValueError, match="n_clusters"):
        cg.kmeans_fit_batch([X], 0)
    with pytest.raises(ValueError, match="minimum of 1"):
        cg.kmeans_fit_batch([np.zeros((5, 0), np.float32)], 1)
    lib = _lib.load()
    ro = np.array([0, 50], np.int64)
    dims, ks, co = np.array([4], np.int32), np.array([3], np.int32), np.array([0, 12], np.int64)
    seeds = np.zeros(1, np.uint64)
    out_c, out_l = np.empty(12, np.float32), np.empty(50, np.int32)
    out_i, out_n = np.empty(1, np.float32), np.empty(1, np.int32)
    p = _lib.ptr
    args = [p(X), p(ro), 50, p(dims), p(ks), 1, 10, 300, 1e-4, p(seeds), p(out_c), p(co), p(out_l), p(out_i), p(out_n),
            None]
    for i in (0, 1, 3, 4, 9, 10, 11, 12, 13, 14):
        a = list(args)
        a[i] = None
        assert lib.am_kmeans_fit_batch(*a) == _lib.AM_ERR_INVALID
        assert "NULL" in _lib.last_error()
    big = list(args)
    ks_big, dims_big = np.array([3], np.int32), np.array([4], np.int32)
    Xb = np.zeros((50, 3100), np.float32)  # max(3, 8) * 3101 > AM_KMEANS_BATCH_MAX_KD
    dims_big[0] = 3100
    co_big = np.array([0, 9300], np.int64)
    big[0], big[3], big[4], big[11] = p(Xb), p(dims_big), p(ks_big), p(co_big)
    big[10] = p(np.empty(9300, np.float32))
    assert lib.am_kmeans_fit_batch(*big) == _lib.AM_ERR_INVALID
    assert "AM_KMEANS_BATCH_MAX_KD" in _lib.last_error()
    # a shape beyond the kernel goes to am_kmeans_fit
    assert not cg.kmeans_batch_serves(50, 3100, 3)
    c, lab, inertia, n_iter = cg.kmeans_fit_batch([Xb + np.arange(50, dtype=np.float32)[:, None]], 3, n_init=1)[0]
    assert c.shape == (3, 3100) and lab.shape == (50,)
