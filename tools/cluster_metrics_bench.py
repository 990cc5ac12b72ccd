"""Clustering scores on the GPU (csrc/cluster_metrics.cu) at clustering-task sizes, next to scikit-learn's
silhouette_score on the box's CPU cores.  One JSON line.  python tools/cluster_metrics_bench.py

Per (N, d) with L = 100 labels (blobs, float32):
  silhouette host-API wall time (validation, label encoding and copies included; median of 3 after a warm-up call),
  kernel device times from CUDA events (am_profile_enable) of one call after the warm-up,
  TFLOP/s of the distance kernel: issued = 8 N^2 dp (four split-bf16 products, dp = d rounded up to 64),
  algorithmic = 2 N^2 d (one N x N x d dot-product GEMM); Davies-Bouldin and Calinski-Harabasz host-API wall times.
The card's name and power limit are read in the same run."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import _lib, cluster_metrics as cm  # noqa: E402

L = 100


def card():
    import torch
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception as e:  # not every driver reports it: record what nvidia-smi says instead
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,enforced.power.limit,power.max_limit",
                            "--format=csv,noheader"], capture_output=True, text=True)
        out["power_limit_w"] = None
        out["power_limit_nvidia_smi"] = r.stdout.strip() or f"unavailable ({e})"
    return out


def blobs(n, d, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((L, d)).astype(np.float32) * 1.5
    lab = rng.integers(0, L, n)
    return centres[lab] + rng.standard_normal((n, d), dtype=np.float32), lab


def wall(fn, reps=3):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        v = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), v


def main():
    out = {"metric": "cluster_scores", **card(), "cpu_cores": os.cpu_count(), "labels": L, "runs": []}
    for n, d in ((20_000, 200), (20_000, 512), (100_000, 200), (100_000, 512)):
        x, lab = blobs(n, d, n + d)
        cm.silhouette_score(x, lab)                              # warm-up: module load, first launches
        _lib.profile_enable(True)
        _lib.profile_report()
        cm.silhouette_score(x, lab)
        prof = _lib.profile_report()
        _lib.profile_enable(False)
        t_sil, s = wall(lambda: cm.silhouette_score(x, lab))
        t_db, db = wall(lambda: cm.davies_bouldin_score(x, lab))
        t_ch, ch = wall(lambda: cm.calinski_harabasz_score(x, lab))
        dp = -(-d // 64) * 64
        k_main = prof.get("silhouette_tc_kernel<false>", {}).get("ms", float("nan"))
        k_all = sum(v["ms"] for v in prof.values())
        out["runs"].append({
            "n": n, "d": d, "silhouette": s, "silhouette_host_api_s": round(t_sil, 4),
            "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items()}, "device_total_ms": round(k_all, 3),
            "distance_kernel_ms": round(k_main, 3),
            "tflops_issued": round(8.0 * n * n * dp / (k_main * 1e-3) / 1e12, 1),
            "tflops_algorithmic": round(2.0 * n * n * d / (k_main * 1e-3) / 1e12, 1),
            "davies_bouldin": db, "davies_bouldin_host_api_s": round(t_db, 4),
            "calinski_harabasz": ch, "calinski_harabasz_host_api_s": round(t_ch, 4)})
        if n == 20_000:
            from sklearn.metrics import silhouette_score
            x64 = x.astype(np.float64)
            t0 = time.perf_counter()
            ref = silhouette_score(x64, lab)
            out["runs"][-1]["sklearn_silhouette_s"] = round(time.perf_counter() - t0, 3)
            out["runs"][-1]["abs_diff_vs_sklearn"] = abs(s - ref)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
