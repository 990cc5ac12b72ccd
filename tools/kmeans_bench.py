"""Config 4 (BASELINE.json configs[3]): Lloyd iterations on 1 M x 512 f32 rows, k = 128, one GPU.
Times `iters` am_kmeans_plan_step calls (assignment GEMM with fused argmin + recheck + partial sums) with CUDA events,
checks the labels of the tensor-core path against the exact CUDA-core path (am_debug_kmeans_step in the debug
library), and prints one JSON line.
    python tools/kmeans_bench.py [--n 1000000] [--iters 20]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import _lib, corpus, dist as amdist  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=1_000_000)
ap.add_argument("--d", type=int, default=512)
ap.add_argument("--k", type=int, default=128)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--check", type=int, default=1)
a = ap.parse_args()

_lib.check(_lib.load().am_init(0))
x, _, _ = corpus.kmeans_library(a.n, a.d, a.k, 7)
xd = torch.from_numpy(x).cuda()
init = xd[torch.from_numpy(np.random.default_rng(2).choice(a.n, a.k, replace=False)).cuda()].contiguous()
k, d = a.k, a.d
labels = torch.empty(a.n, dtype=torch.int32, device="cuda")
sums = torch.empty(k, d, device="cuda"); counts = torch.empty(k, device="cuda"); inertia = torch.zeros(1, device="cuda")
plan = amdist.KMeansPlan(xd, k)
centers = init.clone()
plan.step(centers, labels, sums, counts, inertia)
torch.cuda.synchronize()
rechecks = [plan.last_recheck()]
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
c0 = centers.clone()
e0.record()
for _ in range(a.iters):
    plan.step(centers, labels, sums, counts)
    centers = torch.where(counts[:, None] > 0, sums / counts.clamp(min=1.0)[:, None], centers).contiguous()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / a.iters
# plan.step alone (no centre update between the steps): what the library costs without the caller's torch ops
e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e2.record()
for _ in range(a.iters):
    plan.step(centers, labels, sums, counts)
e3.record()
torch.cuda.synchronize()
ms_step_only = e2.elapsed_time(e3) / a.iters
# same trajectory again with the per-launch profiler on (its events cost host time: not part of `ms`)
centers = c0
_lib.profile_enable(True)
for _ in range(a.iters):
    plan.step(centers, labels, sums, counts)
    rechecks.append(plan.last_recheck())
    centers = torch.where(counts[:, None] > 0, sums / counts.clamp(min=1.0)[:, None], centers).contiguous()
torch.cuda.synchronize()
prof = _lib.profile_report()
_lib.profile_enable(False)
out = {"config": f"{a.n} x {d} f32, k={k}", "tensor_cores": plan.uses_tensor_cores, "ms_per_lloyd_iteration": round(ms, 4), "ms_per_plan_step_only": round(ms_step_only, 4),
       "kernel_ms_per_iteration": {kk: round(v["ms"] / a.iters, 4) for kk, v in prof.items()},
       "hbm_bound_ms": round(2 * a.n * d * 4 / 6586.7e9 * 1e3, 4), "recheck_rows_per_iteration": rechecks}
if a.check:
    plan.step(centers, labels, sums, counts, inertia)
    torch.cuda.synchronize()
    l2 = torch.empty_like(labels); s2 = torch.empty_like(sums); c2 = torch.empty_like(counts); i2 = torch.zeros(1, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check_debug(_lib.load_debug().am_debug_kmeans_step(1, p(xd), a.n, d, k, p(centers), p(l2), p(s2), p(c2), p(i2),
                                                            None, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    out["labels_equal_exact_path"] = bool((labels == l2).all().item())
    out["label_mismatches"] = int((labels != l2).sum().item())
    out["counts_equal"] = bool((counts == c2).all().item())
    out["sums_max_rel_diff"] = float(((sums - s2).abs().max() / s2.abs().max()).item())
    out["inertia_rel_diff"] = float(abs(inertia.item() - i2.item()) / i2.item())
print(json.dumps(out))
