"""The memory and stream of the one-shot host entry points (csrc/host_call.cuh): the fits and scores hand their scratch
back to the device when they return, and calls from several threads, which share a stream per thread, return what
the same calls return one after another."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MiB = 1 << 20


def _blobs(n, d, k, seed, spread=0.35):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((k, d)).astype(np.float32) * 3
    return (centres[rng.integers(0, k, n)] + spread * rng.standard_normal((n, d))).astype(np.float32)


def _trim_default_pool():
    """Hands back whatever the device's default stream-ordered pool has cached from earlier calls in this process, so
    that an allocation from it shows in the device's free memory."""
    import torch
    cuda = C.CDLL("libcuda.so.1")
    pool = C.c_void_p()
    assert cuda.cuDeviceGetDefaultMemPool(C.byref(pool), C.c_int(torch.cuda.current_device())) == 0
    assert cuda.cuMemPoolTrimTo(pool, C.c_size_t(0)) == 0


def test_fits_return_their_scratch():
    """am_init keeps whatever the stream-ordered pool has reserved, so scratch of hundreds of MB taken from it would
    stay out of reach of everything else in the worker.  Each large call below needs about 300 MB (the GMM's rows,
    responsibilities and seeding distances; the silhouette's f64[N, L] sums and split rows; DBSCAN's N x N adjacency
    bits) and must leave the device's free memory where it found it.  The warm-up calls are small, so that a pooled
    large call could not reuse memory they left in the pool."""
    import torch
    from audiomuse_ai_b200 import _lib, cluster_metrics as cm, clustering_gpu as cg

    _lib.check(_lib.load().am_init(0))
    torch.cuda.init()
    rng = np.random.default_rng(3)
    xg = rng.standard_normal((80, 60))[rng.integers(0, 80, 200_000)] + rng.standard_normal((200_000, 60))
    xs = _blobs(100_000, 256, 100, 4)
    ls = rng.integers(0, 100, len(xs))
    xd = _blobs(40_000, 32, 20, 5)
    calls = {
        "am_gmm_fit": lambda n: cg.gmm_fit(xg[:n], 20, n_init=3, max_iter=5, random_state=0),
        "am_cluster_scores": lambda n: (cm.silhouette_score(xs[:n], ls[:n]), cm.davies_bouldin_score(xs[:n], ls[:n])),
        "am_dbscan": lambda n: cg.GPUDBSCAN(1.0, 5).fit_predict(xd[:n]),
    }
    for name, call in calls.items():
        call(2000)  # loads the kernels and creates the thread's stream
        torch.cuda.synchronize()
        _trim_default_pool()
        before = torch.cuda.mem_get_info()[0]
        call(None)
        torch.cuda.synchronize()
        after = torch.cuda.mem_get_info()[0]
        assert before - after <= 2 * MiB, f"{name}: {(before - after) / MiB:.1f} MiB still held after the call"


def _pca_project(X, mean, comps):
    from audiomuse_ai_b200 import _lib
    Y = np.empty((X.shape[0], comps.shape[0]), np.float32)
    _lib.check(_lib.load().am_pca_project(_lib.ptr(X), X.shape[0], X.shape[1], _lib.ptr(mean), _lib.ptr(comps),
                                          comps.shape[0], _lib.ptr(Y)))
    return Y


def _dbscan(X, eps, min_samples):
    from audiomuse_ai_b200 import _lib
    labels = np.empty(X.shape[0], np.int32)
    n = C.c_int(0)
    _lib.check(_lib.load().am_dbscan(_lib.ptr(X), X.shape[0], X.shape[1], float(eps), int(min_samples),
                                     _lib.ptr(labels), C.byref(n)))
    return labels, n.value


def test_calls_from_four_threads_match_serial_calls():
    """The clustering task runs its fits from worker threads; each thread's calls share that thread's stream.
    Four threads calling am_pca_project, am_dbscan and am_kmeans_fit at once get what the same calls return one after
    another: the same bytes, except am_kmeans_fit's centres and inertia, whose sums are float atomics and so agree
    to rounding (its labels and iteration count are exact)."""
    from audiomuse_ai_b200 import clustering_gpu as cg

    jobs = []
    for t in range(4):
        rng = np.random.default_rng(10 + t)
        X = _blobs(20_000 + 1000 * t, 64, 12, 20 + t)
        mean = X.mean(axis=0).astype(np.float64)
        comps = np.linalg.qr(rng.standard_normal((64, 16)))[0].T.astype(np.float32).copy()
        jobs.append((X, mean, comps))

    def run(job, seed):
        X, mean, comps = job
        centers, labels, inertia, n_iter = cg.kmeans_fit(X, 12, n_init=1, seed=seed)
        return [_pca_project(X, mean, comps), *_dbscan(X, 4.2, 8), labels, n_iter], (centers, inertia)

    want = [run(job, t) for t, job in enumerate(jobs)]
    got, errs = [None] * 4, []

    def worker(t):
        try:
            for _ in range(3):
                got[t] = run(jobs[t], t)
                for w, g in zip(want[t][0], got[t][0]):
                    assert np.asarray(w).tobytes() == np.asarray(g).tobytes()
                for w, g in zip(want[t][1], got[t][1]):
                    np.testing.assert_allclose(g, w, rtol=1e-5, atol=1e-5)
        except Exception as e:  # pragma: no cover
            errs.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errs, errs
