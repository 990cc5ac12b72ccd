"""K4 parity: exact GPU index vs the float64 oracle -- identical ids (bit-exact index work)."""
import functools
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import knn as oknn


def _lib_data(n, d, seed):
    from audiomuse_ai_b200 import corpus
    x = corpus.knn_library(n, d, seed)
    q = corpus.knn_queries(x, 200, 56, seed + 1)
    return x, q


def _index(x, space=None):
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Cosine if space is None else space, num_dimensions=x.shape[1], M=64, ef_construction=1024)
    idx.add_items(x, ids=np.arange(len(x)))
    idx.ef = 1024
    return idx


@pytest.mark.parametrize("d,mode", [(512, 1), (512, 2), (200, 1), (200, 2), (512, 0)])
def test_topk_ids_identical_to_oracle(d, mode):
    x, q = _lib_data(20000, d, 1234)
    idx = _index(x)
    ids, dist = idx.query(q, 50, mode=mode)
    want_ids, want_dist = oknn.topk(x, q, 50)
    np.testing.assert_array_equal(ids.astype(np.int64), want_ids)
    np.testing.assert_allclose(dist, want_dist, atol=2e-7)
    assert (np.diff(dist, axis=1) >= 0).all()


def test_single_vector_query_and_get_vector():
    x, q = _lib_data(5000, 512, 7)
    idx = _index(x)
    ids, dist = idx.query(q[0], 10)
    assert ids.shape == (10,) and dist.shape == (10,)
    np.testing.assert_array_equal(ids.astype(np.int64), oknn.topk(x, q[:1], 10)[0][0])
    np.testing.assert_allclose(idx.get_vector(17), x[17], atol=1e-7)
    assert len(idx) == idx.num_elements == 5000
    i2, d2 = idx.query(idx.get_vector(123), 1)   # a stored vector is its own nearest neighbour
    assert int(i2[0]) == 123 and abs(float(d2[0])) < 1e-6


def test_unnormalised_rows_are_stored_normalised():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((3000, 200)).astype(np.float32) * rng.uniform(0.1, 10, (3000, 1)).astype(np.float32)
    idx = _index(x)
    np.testing.assert_allclose(idx.get_vector(5), oknn.normalize_rows(x)[5], atol=1e-7)
    q = rng.standard_normal((16, 200)).astype(np.float32) * 7
    ids, _ = idx.query(q, 25)
    np.testing.assert_array_equal(ids.astype(np.int64), oknn.topk(oknn.normalize_rows(x), q, 25)[0])


def test_k_equals_len_full_scan_and_recall_error():
    """voyager_manager.py:1681 asks k = len(index); k > len raises RecallError (:1448)."""
    from audiomuse_ai_b200 import voyager_compat as vc
    x, q = _lib_data(6000, 64, 9)
    idx = _index(x)
    ids, dist = idx.query(q[0], len(idx))
    want_ids, want_dist = oknn.topk(x, q[:1], len(idx))
    np.testing.assert_array_equal(ids.astype(np.int64), want_ids[0])
    np.testing.assert_allclose(dist, want_dist[0], atol=2e-7)
    with pytest.raises(vc.RecallError):
        idx.query(q[0], len(idx) + 1)


def test_duplicates_break_ties_by_lower_id():
    rng = np.random.default_rng(5)
    base = oknn.normalize_rows(rng.standard_normal((50, 128)))
    x = np.concatenate([base] * 40)          # every vector appears 40 times
    idx = _index(x)
    ids, _ = idx.query(base[:8], 60, mode=1)
    np.testing.assert_array_equal(ids.astype(np.int64), oknn.topk(x, base[:8], 60)[0])
    ids2, _ = idx.query(base[:8].repeat(4, axis=0), 60, mode=2)
    np.testing.assert_array_equal(ids2.astype(np.int64), oknn.topk(x, base[:8].repeat(4, axis=0), 60)[0])


def test_matches_reference_dummy_voyager_index_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "dummy_index_golden.npz"))
    rng = np.random.default_rng(int(g["seed"]))
    E = rng.standard_normal((500, 512)).astype(np.float32)
    E /= np.linalg.norm(E, axis=1, keepdims=True)
    Q = rng.standard_normal((8, 512)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    idx = _index(E)
    ids, dist = idx.query(Q, 50)
    np.testing.assert_array_equal(ids.astype(np.int64), g["ids"])
    np.testing.assert_allclose(dist, g["dists"], atol=3e-7)


@pytest.mark.parametrize("space_name", ["Euclidean", "InnerProduct"])
def test_other_spaces(space_name):
    from audiomuse_ai_b200 import voyager_compat as vc
    rng = np.random.default_rng(21)
    x = rng.standard_normal((4000, 96)).astype(np.float32)
    q = rng.standard_normal((20, 96)).astype(np.float32)
    space = getattr(vc.Space, space_name)
    idx = _index(x, space)
    ids, dist = idx.query(q, 30)
    metric = oknn.EUCLIDEAN if space_name == "Euclidean" else oknn.INNER_PRODUCT
    want_ids, want_dist = oknn.topk(x, q, 30, metric)
    np.testing.assert_array_equal(ids.astype(np.int64), want_ids)
    np.testing.assert_allclose(dist, want_dist, rtol=1e-6, atol=1e-5)


def test_full_size_library_properties():
    """BASELINE config 3 size (100k x 512): size-independent properties + a sampled oracle check."""
    x, q = _lib_data(100_000, 512, 1234)
    idx = _index(x)
    ids, dist = idx.query(q, 50)
    assert ids.shape == (256, 50) and (np.diff(dist, axis=1) >= 0).all()
    assert all(len(set(r.tolist())) == 50 for r in ids)
    sel = [0, 100, 255]
    np.testing.assert_array_equal(ids[sel].astype(np.int64), oknn.topk(x, q[sel], 50)[0])
    ids1, _ = idx.query(q, 50, mode=1)
    np.testing.assert_array_equal(ids, ids1)     # tensor-core filter == fp32 filter


def test_filter_by_distance_matches_reference_golden(golden_dir):
    """am_knn_filter_by_distance (the device walk of voyager_manager._filter_by_distance) keeps exactly the items
    the reference kept (tests/golden/filter_golden.npz, produced by the reference's own function), for both
    branches and look-backs, one list at a time and all lists of a length in one call."""
    import os
    g = np.load(os.path.join(golden_dir, "filter_golden.npz"))
    F, thr, B = g["vectors"], float(g["threshold"]), int(g["batch"])
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Cosine, num_dimensions=F.shape[1])
    idx.add_items(F)
    for ci in range(int(g["n_cases"])):
        order = g[f"order_{ci}"]
        for lb in (1, 3):
            keep = idx.filter_by_distance(order, thr, lookback=lb, batch=B)
            assert keep.dtype == bool and keep.shape == order.shape
            assert order[keep].tolist() == g[f"kept_{ci}_lb{lb}"].tolist(), (ci, lb)
    assert idx.filter_by_distance(np.array([3, 1, 2]), thr, lookback=0).all()
    both = np.stack([g["order_0"], g["order_0"][::-1]])
    keep2 = idx.filter_by_distance(both, thr, lookback=1, batch=B)
    assert both[0][keep2[0]].tolist() == g["kept_0_lb1"].tolist()
    want_rev = oknn.filter_by_distance(F, [int(i) for i in both[1]], thr, 1, oknn.COSINE, B)
    assert both[1][keep2[1]].tolist() == want_rev


def test_filter_by_distance_euclidean_large_list():
    """Euclidean space (distance = ||a - b||, threshold 0.15) on a 1000-item list with planted duplicates."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((3000, 64)).astype(np.float32)
    x[1500:] = x[:1500] + 0.01 * rng.standard_normal((1500, 64)).astype(np.float32)
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Euclidean, num_dimensions=64)
    idx.add_items(x)
    q = rng.standard_normal(64).astype(np.float32)
    order = np.argsort(((x - q) ** 2).sum(1), kind="stable")[:1000]
    keep = idx.filter_by_distance(order, 0.15, lookback=2)
    want = oknn.filter_by_distance(x, [int(i) for i in order], 0.15, 2, oknn.EUCLIDEAN, 50)
    assert order[keep].tolist() == want
    assert 0 < keep.sum() < len(order)


@pytest.mark.parametrize("space_name", ["Cosine", "Euclidean"])
def test_get_vectors_of_many_rows_and_of_one(space_name):
    """am_knn_get_vectors, of many rows and of one, = the stored rows."""
    from audiomuse_ai_b200 import voyager_compat as vc
    rng = np.random.default_rng(9)
    x = rng.standard_normal((500, 200)).astype(np.float32)
    idx = vc.Index(getattr(vc.Space, space_name), num_dimensions=200)
    idx.add_items(x)
    ids = [int(i) for i in rng.choice(500, 37, replace=False)]
    stored = idx.get_vectors(ids)
    np.testing.assert_array_equal(stored, np.stack([idx.get_vector(i) for i in ids]))
    from audiomuse_ai_b200 import _lib
    one = np.empty(200, np.float32)
    for j, i in enumerate(ids):   # one row per call
        row = np.array([idx._row_of(i)], np.int64)
        _lib.check(_lib.load().am_knn_get_vectors(idx._ensure_built(), _lib.ptr(row), 1, _lib.ptr(one)))
        np.testing.assert_array_equal(one, stored[j])


def test_queries_are_reentrant_across_threads():
    """The reference serves k-NN from a Flask gthread worker with 4 threads (deployment/supervisord.conf:19):
    concurrent am_knn_query / get_vectors / filter calls on ONE index (ctypes drops the GIL) must return what
    the same calls return alone."""
    import threading
    x, q = _lib_data(20000, 512, 77)
    idx = _index(x)
    want = [idx.query(q[i * 16:(i + 1) * 16], 50) for i in range(8)]
    want_single = [idx.query(q[i], 25) for i in range(8)]
    errs, got, got_single = [], [None] * 8, [None] * 8

    def worker(t):
        try:
            for rep in range(3):
                for i in range(t, 8, 4):
                    got[i] = idx.query(q[i * 16:(i + 1) * 16], 50)
                    got_single[i] = idx.query(q[i], 25)
                    v = idx.get_vectors([int(j) for j in got_single[i][0][:5]])
                    assert v.shape == (5, 512)
                    idx.filter_by_distance(got_single[i][0].astype(np.int64), 0.01)
        except Exception as e:  # pragma: no cover
            errs.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errs, errs
    for i in range(8):
        np.testing.assert_array_equal(got[i][0], want[i][0])
        np.testing.assert_array_equal(got[i][1], want[i][1])
        np.testing.assert_array_equal(got_single[i][0], want_single[i][0])


CHUNK_MAX_KS = (1, 50, 500, 600)


@functools.lru_cache(maxsize=None)
def _config3_ragged(space_name):
    """Config-3 size with a ragged N (100 003 x 512, 640 queries): the index and the oracle's top max(CHUNK_MAX_KS) of
    the rows as stored (cosine: unit-normalised), whose prefixes are the top k for every smaller k (the order is total:
    distance, then id)."""
    from audiomuse_ai_b200 import corpus, voyager_compat as vc
    x, _ = _lib_data(100_003, 512, 1234)
    q = corpus.knn_queries(x, 600, 40, 99)
    if space_name == "Euclidean":
        x = x * np.random.default_rng(3).uniform(0.5, 2.0, (len(x), 1)).astype(np.float32)
    metric = oknn.EUCLIDEAN if space_name == "Euclidean" else oknn.COSINE
    idx = _index(x, getattr(vc.Space, space_name))
    return idx, q, oknn.topk(idx.get_vectors(range(len(x))), q, max(CHUNK_MAX_KS), metric)


@pytest.mark.parametrize("k", CHUNK_MAX_KS)
@pytest.mark.parametrize("space_name", ["Cosine", "Euclidean"])
def test_chunk_max_selection_equals_row_streaming_selection(k, space_name):
    """Batches on the tensor-core path: for k <= 512 the GEMM epilogue also writes the maximum of every 32 scores, and
    the selection kernel works from those maxima (threshold + the few chunks that can hold answers) instead of
    streaming each query's whole row of scores twice; k = 600 streams the rows.  Every query's answer is the float64
    oracle's, id for id, at config-3 size with a ragged N, incl. k = 500 (the reference's n + 4n expansion), for
    cosine and euclidean spaces; and identical, id for id and distance for distance, to the fp32 scoring pass."""
    idx, q, (want_ids, want_dist) = _config3_ragged(space_name)
    ids, dist = idx.query(q, k, mode=2)
    np.testing.assert_array_equal(ids.astype(np.int64), want_ids[:, :k])
    np.testing.assert_allclose(dist, want_dist[:, :k], rtol=1e-6, atol=2e-7)
    ids1, dist1 = idx.query(q, k, mode=1)
    np.testing.assert_array_equal(ids1, ids)
    np.testing.assert_array_equal(dist1, dist)


@pytest.mark.parametrize("space_name", ["Euclidean", "InnerProduct"])
@pytest.mark.parametrize("mode", [1, 2])
def test_queries_much_larger_than_the_stored_rows(space_name, mode):
    """ADVICE r1: the fp32-accumulation part of the filter bound assumed ||q|| <= ~2 max||x||.  It now scales with each
    query's own norm, so queries 1000x larger than the library (and tiny ones) still return the oracle's ids."""
    from audiomuse_ai_b200 import voyager_compat as vc
    rng = np.random.default_rng(33)
    x = rng.standard_normal((8192, 128)).astype(np.float32)
    q = rng.standard_normal((48, 128)).astype(np.float32)
    q[:16] *= 1000.0
    q[16:32] *= 1e-3
    idx = _index(x, getattr(vc.Space, space_name))
    ids, dist = idx.query(q, 40, mode=mode)
    metric = oknn.EUCLIDEAN if space_name == "Euclidean" else oknn.INNER_PRODUCT
    want_ids, want_dist = oknn.topk(x, q, 40, metric)
    np.testing.assert_array_equal(ids.astype(np.int64), want_ids)
    np.testing.assert_allclose(dist, want_dist, rtol=1e-6, atol=1e-5)
