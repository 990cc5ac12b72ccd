"""The two k-means drivers on each side of their line: one clustering-task RQ batch of fits (20 problems, n_init 10,
the task's k-means++ / max_iter 300 / tol 1e-4) through am_kmeans_fit_batch against 20 sequential am_kmeans_fit
calls, for N in {2 000, 10 000, 40 000}, d in {200, 50}, k in {40, 100}; and one large single problem through both.
Each call ends in a device synchronise, so the host clock times the whole fit; median and p99 over the repeats after
one warm-up.  'same' counts the problems whose labels and n_iter equal am_kmeans_fit's.  Prints the card, its power
limit and SM clock, then one JSON line per row.
    python tools/clustering_batch_bench.py [--repeats 3] [--problems 20] [--quick]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import _lib, clustering_gpu as cg  # noqa: E402
from oracle import kmeans as okm  # noqa: E402
from tests.test_gpu_kmeans_batch import unexplained_label_differences  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--repeats", type=int, default=3)
ap.add_argument("--problems", type=int, default=20)
ap.add_argument("--n", type=int, nargs="+", default=[2000, 10000, 40000], help="subset sizes to run")
ap.add_argument("--skip-single", action="store_true")
ap.add_argument("--quick", action="store_true", help="one small shape (rehearsal)")
a = ap.parse_args()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts)) * 1e3, float(np.percentile(ts, 99)) * 1e3


def problems(N, d, k, P):
    """task-shaped subsets: standard-scaled blobs, N within +-10 % across the batch"""
    rng = np.random.default_rng(N + d + k)
    return [okm.blobs(int(N * rng.uniform(0.9, 1.1)), d, k, seed=i, spread=1.5)[0] for i in range(P)]


_lib.check(_lib.load().am_init(0))
print(json.dumps({"card": card()}), flush=True)
shapes = [(2000, 50, 40)] if a.quick else [(N, d, k) for N in a.n for d in (200, 50) for k in (40, 100)]
for N, d, k in shapes:
    Xs = problems(N, d, k, a.problems)
    batch, tb, tb99 = timed(lambda: cg.kmeans_fit_batch(Xs, k, seeds=list(range(len(Xs)))), a.repeats)
    seq, ts, ts99 = timed(lambda: [cg.kmeans_fit(X, k, seed=i) for i, X in enumerate(Xs)], a.repeats)
    same = sum(np.array_equal(b[1], s[1]) and b[3] == s[3] for b, s in zip(batch, seq))
    # a problem whose labels differ is a near tie when every differing row is within the margin that the two
    # drivers' centres explain (am_kmeans_fit sums with float atomics), otherwise a real difference
    near = other = 0
    for X, b, s in zip(Xs, batch, seq):
        diff, wrong = unexplained_label_differences(X, b[0], s[0], b[1], s[1])
        near += bool(len(diff)) and not len(wrong)
        other += bool(len(wrong))
    print(json.dumps({"row": "batch", "N": N, "d": d, "k": k, "problems": len(Xs), "n_init": 10,
                      "batch_ms_median": round(tb, 2), "batch_ms_p99": round(tb99, 2),
                      "sequential_ms_median": round(ts, 2), "sequential_ms_p99": round(ts99, 2),
                      "speedup": round(ts / tb, 2), "same": f"{same}/{len(Xs)}", "near_tie": near,
                      "other": other}), flush=True)

if a.skip_single:
    sys.exit(0)
# one large problem: am_kmeans_fit spreads it over the whole GPU, the batch kernel runs each init on one CTA
N, d, k = (20000, 32, 16) if a.quick else (200000, 64, 64)
X = okm.blobs(N, d, k, seed=3, spread=1.5)[0]
(b,), tb, tb99 = timed(lambda: cg.kmeans_fit_batch([X], k, n_init=1), 1)
s, ts, ts99 = timed(lambda: cg.kmeans_fit(X, k, n_init=1), 1)
print(json.dumps({"row": "single", "N": N, "d": d, "k": k, "n_init": 1, "batch_ms": round(tb, 2),
                  "kmeans_fit_ms": round(ts, 2), "speedup": round(ts / tb, 2),
                  "same": int(np.array_equal(b[1], s[1]) and b[3] == s[3])}), flush=True)
print(json.dumps({"card": card()}), flush=True)
