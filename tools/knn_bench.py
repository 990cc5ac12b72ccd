"""Config 3 (100 k x 512, k = 50): per-kernel device time and host-API QPS of the k-NN query path at batch 4096 / 256 /
1.  One JSON line.  python tools/knn_bench.py"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import _lib, corpus, voyager_compat as vc  # noqa: E402

x = corpus.knn_library(100_000, 512, 1234)
q = corpus.knn_queries(x, 10_000, 1_000, 4321)
idx = vc.Index(vc.Space.Cosine, num_dimensions=512)
idx.add_items(x)
out = {}
for nq, reps in ((4096, 10), (256, 30), (1, 300)):
    qq = q[:nq] if nq > 1 else q[0]
    idx.query(qq, 50)
    t0 = time.perf_counter()
    for r in range(reps):
        idx.query(qq, 50)
    dt = (time.perf_counter() - t0) / reps
    _lib.profile_enable(True)
    for r in range(3):
        idx.query(qq, 50)
    prof = _lib.profile_report()
    _lib.profile_enable(False)
    out[f"batch{nq}"] = {"qps_host_api": round(nq / dt, 1), "ms_per_call": round(dt * 1e3, 4),
                         "kernel_ms": {k: round(v["ms"] / 3, 4) for k, v in prof.items()}}
print(json.dumps(out))
