"""Bit-identity of the k-NN index across two builds of the library.

    python tools/knn_equiv.py dump FILE.npz       # on the build to compare against
    python tools/knn_equiv.py compare FILE.npz    # on the build under test: every array np.array_equal

Seeded inputs only, chosen so that every pair of scoring pass (fp32 rows, bf16 small batch, tensor-core GEMM) and
selection (chunk maxima, row streaming, full sort) runs: cosine / euclidean / inner product; N of 500 to 100 003; d of
64, 96, 200, 512 and 1000 (bf16 row pitch 64 to 1024); 1 to 4096 queries (the host API on both sides of its 2 MiB
staging limit); k of 1, 50, 500, 600 and len(index); modes 0, 1 and 2.  Per call: ids, distances, and the kernels
launched with their counts (am_profile_report, template arguments stripped).  Also am_knn_query_dev on a 20 000 x 200
euclidean self-query as the spectral and UMAP graphs issue it, and the duplicate filter, get_vectors and get_vector,
the radius walk under both metrics and artist rules, and the song path on seeded jobs (_song_paths).  A query with
k > 4032 is answered by the full sort alone: its kernel list may differ
from the other build's by the scoring kernels only; get_vector's launches are not compared (it used to copy from a
host mirror of the rows, and gathers its row on the device now).  Needs an H100."""
import ctypes as C
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiomuse_ai_b200 import _lib, voyager_compat as vc  # noqa: E402

SPACES = {"cos": vc.Space.Cosine, "l2": vc.Space.Euclidean, "ip": vc.Space.InnerProduct}
SHAPES = ((500, 64), (2000, 96), (2000, 200), (20_000, 200), (20_000, 1000), (100_003, 512))
BATCHES = (1, 3, 5, 16, 256, 4096)
SCORERS = ("score_f32_kernel", "chunk_max_rows_kernel", "score_bf16_small_kernel", "gemm_wgmma_kernel")
FULL_SORT_K = 4096 - 64


def _kernels():
    """Kernels launched since the last call: 'name:count', template arguments and parentheses stripped."""
    agg = {}
    for name, v in _lib.profile_report().items():
        while re.search(r"<[^<>]*>", name):
            name = re.sub(r"<[^<>]*>", "", name)
        name = name.strip("() ")
        agg[name] = agg.get(name, 0) + int(v["count"])
    return np.array(sorted(f"{k}:{c}" for k, c in agg.items()))


def _data(N, d, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((N, d)) * rng.uniform(0.5, 2.0, (N, 1))).astype(np.float32)
    near = x[rng.integers(0, N, max(BATCHES) // 2)] + 0.3 * rng.standard_normal((max(BATCHES) // 2, d)).astype(np.float32)
    q = np.concatenate([near, 1.5 * rng.standard_normal((max(BATCHES) // 2, d)).astype(np.float32)])
    return x, q[rng.permutation(len(q))].astype(np.float32)


def _song_paths(idx, x, lists, key):
    """Index.song_path over seeded jobs on the k-NN lists `lists` (rows = ids): lists shorter and longer than the
    filter batch, filter lookback 0 and 3, both caps off and on, stop_on_failure 0 and 1, both metrics.  The last job
    asks for more songs than its list can give, so it fails and gives back what it took.  Every output is recorded,
    with the in / out state arrays after the call."""
    out = {}
    rng = np.random.default_rng(len(x))
    sizes = (30, 300, 12, 200, 45, 250)  # filter_batch 50: lists on both sides of it
    cand = np.concatenate([lists[j % len(lists)][:m] for j, m in enumerate(sizes)]).astype(np.int64)
    cand[rng.integers(0, len(cand), 5)] = len(x) + 3  # ids without a vector
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    job_n = np.array([m - m // 5 for m in sizes], np.int32)
    need = np.array([3, 8, 2, 6, 4, 10_000], np.int32)
    sig = np.where(cand % 53 == 0, -1, cand % 97).astype(np.int32)
    author = (cand % 11).astype(np.int32)
    raw = (cand % 13 - 1).astype(np.int32)
    a, b = x[lists[0][:-1]].astype(np.float64), x[lists[0][1:]].astype(np.float64)
    cos = (a * b).sum(1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1)
    thr = {0: (np.quantile(1 - cos, 0.3), np.quantile(np.arccos(np.clip(cos, -1, 1)) / np.pi, 0.3)),
           1: (np.quantile(np.linalg.norm(a - b, axis=1), 0.3),) * 2}
    for metric in (0, 1):
        for lookback in (0, 3):
            for cap in (0, 2):
                for stop in (0, 1):
                    cfg = _lib.SongPathCfg(voyager_metric=metric, path_metric=metric, filter_lookback=lookback,
                                           filter_batch=50, path_lookback=2, voyager_cap=cap, path_cap=cap,
                                           stop_on_failure=stop, filter_threshold=float(thr[metric][0]),
                                           path_threshold=float(thr[metric][1]))
                    used_sig = np.zeros(97, np.uint8)
                    used_sig[[5, 17]] = 1
                    author_count = np.zeros(11, np.int32)
                    author_count[3] = 2
                    found, pos, failed, used, path, dist = idx.song_path(
                        cfg, off, job_n, need, cand, sig, author, raw, [int(lists[1][0]), int(lists[2][1])], used_sig,
                        author_count, [int(lists[0][0])], int(lists[3][-1]))
                    k = f"{key}/song_path/m{metric}/lb{lookback}/cap{cap}/stop{stop}"
                    out.update({k + "/found": found, k + "/pos": pos, k + "/failed": np.array([-1 if failed is None
                                                                                                else failed]),
                                k + "/used": np.array(used), k + "/path": np.array(path), k + "/dist": dist,
                                k + "/used_sig": used_sig, k + "/author_count": author_count})
    return out


def _collect():
    out = {}
    _lib.profile_enable(True)
    for si, (sname, space) in enumerate(SPACES.items()):
        for N, d in SHAPES:
            x, q = _data(N, d, 100 * si + d + N)
            idx = vc.Index(space, num_dimensions=d)
            idx.add_items(x)
            for nq in BATCHES:
                for k in sorted({1, 50, 500, 600, N}):
                    if k > N or (nq == 4096 and k > 50) or (k == N and nq > (16 if N <= FULL_SORT_K else 3)):
                        continue
                    for mode in (0, 1, 2):
                        key = f"{sname}/N{N}/d{d}/nq{nq}/k{k}/mode{mode}"
                        _kernels()
                        out[key + "/ids"], out[key + "/dist"] = idx.query(q[:nq], k, mode=mode)
                        out[key + "/kernels"] = _kernels()
            lists = out[f"{sname}/N{N}/d{d}/nq16/k50/mode0/ids"].astype(np.int64)
            a, b = x[lists[:, :-1]].astype(np.float64), x[lists[:, 1:]].astype(np.float64)
            thr = float(np.median(np.linalg.norm(a - b, axis=2) if sname == "l2" else
                                  1 - (a * b).sum(2) / np.linalg.norm(a, axis=2) / np.linalg.norm(b, axis=2)))
            for batch in (20, 50):
                out[f"{sname}/N{N}/d{d}/filter/batch{batch}"] = idx.filter_by_distance(lists, thr, lookback=3, batch=batch)
            ids = [int(i) for i in lists[0][:40]]
            out[f"{sname}/N{N}/d{d}/get_vectors"] = idx.get_vectors(ids)
            pool = [int(i) for i in out[f"{sname}/N{N}/d{d}/nq16/k500/mode0/ids"][0]] if N >= 500 else ids
            artists = [i % 7 - 1 for i in range(len(pool))]
            for metric in ("angular", "euclidean"):
                for ed, cap in ((True, 1), (True, 3), (False, 3)):
                    pos, dist = idx.radius_walk(q[0], pool, artists, 200, ed, cap, metric)
                    out[f"{sname}/N{N}/d{d}/radius_walk/{metric}/ed{int(ed)}/cap{cap}/pos"] = pos
                    out[f"{sname}/N{N}/d{d}/radius_walk/{metric}/ed{int(ed)}/cap{cap}/dist"] = dist
            if (N, d) == (2000, 200):
                out.update(_song_paths(idx, x, out[f"{sname}/N{N}/d{d}/nq16/k500/mode0/ids"].astype(np.int64),
                                       f"{sname}/N{N}/d{d}"))
            out[f"{sname}/N{N}/d{d}/other_kernels"] = _kernels()
            one = np.empty((5, d), np.float32)
            for j, i in enumerate(ids[:5]):
                row = np.array([i], np.int64)
                _lib.check(_lib.load().am_knn_get_vectors(idx._ensure_built(), _lib.ptr(row), 1, _lib.ptr(one[j])))
            out[f"{sname}/N{N}/d{d}/get_vector"] = one
            _kernels()
    # the spectral / UMAP graph: euclidean self-query of device rows, mode 0, on the caller's stream
    import torch
    x, _ = _data(20_000, 200, 7)
    xd = torch.from_numpy(x).cuda()
    st = torch.cuda.current_stream()
    ids = torch.empty((len(x), 15), dtype=torch.int64, device="cuda")
    dist = torch.empty((len(x), 15), dtype=torch.float32, device="cuda")
    h = C.c_void_p()
    lib = _lib.load()
    _lib.check(lib.am_knn_build_dev(C.c_void_p(xd.data_ptr()), len(x), 200, 1, C.c_void_p(st.cuda_stream), C.byref(h)))
    _lib.check(lib.am_knn_query_dev(h, C.c_void_p(xd.data_ptr()), len(x), 15, 0, C.c_void_p(ids.data_ptr()),
                                    C.c_void_p(dist.data_ptr()), C.c_void_p(st.cuda_stream)))
    st.synchronize()
    lib.am_knn_free(h)
    out["dev_self_query/ids"], out["dev_self_query/dist"] = ids.cpu().numpy(), dist.cpu().numpy()
    out["dev_self_query/kernels"] = _kernels()
    _lib.profile_enable(False)
    return out


def _full_sort_kernels_match(want, got):
    """k > 4032: the build under test runs the full sort without a scoring pass before it."""
    strip = lambda a: [s for s in a.tolist() if s.split(":")[0] not in SCORERS]  # noqa: E731
    return strip(want) == strip(got) == got.tolist()


def main():
    mode, path = sys.argv[1], sys.argv[2]
    got = _collect()
    if mode == "dump":
        np.savez(path, **got)
        print(f"wrote {len(got)} arrays to {path}")
        return 0
    want = np.load(path)
    bad, expected = [], []
    for k in sorted(set(want.files) | set(got)):
        if k in got and k in want.files and np.array_equal(want[k], got[k]):
            continue
        m = re.search(r"/k(\d+)/mode\d/kernels$", k)
        if m and int(m.group(1)) > FULL_SORT_K and k in got and k in want.files and _full_sort_kernels_match(want[k], got[k]):
            expected.append(k)
            print(f"scorer dropped: {k}: {' '.join(want[k])} -> {' '.join(got[k])}")
            continue
        bad.append(k)
        print(f"DIFFERENT: {k}" + (f": {' '.join(want[k])} -> {' '.join(got[k])}" if k.endswith("kernels") and k in got
                                   and k in want.files else ""))
    print(f"{len(got) - len(bad) - len(expected)} of {len(got)} arrays equal, {len(expected)} full-sort kernel lists "
          f"without the scoring pass, {len(bad)} different")
    return 1 if bad or len(got) != len(want.files) else 0


if __name__ == "__main__":
    sys.exit(main())
