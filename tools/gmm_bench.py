#!/usr/bin/env python
"""Time the clustering task's GaussianMixture on the GPU (am_gmm_fit, csrc/gmm.cu).

    python tools/gmm_bench.py [--shapes 20000x60,20000x100,100000x60,100000x100] [--no-check]
                              [--covariance-type full|diag|tied|spherical]

Task-shaped fits with the reference's settings (d = 200, n_init = 10, max_iter = 100, tol = 1e-3, reg_covar = 1e-4)
on seeded standardised rows.  Per shape: per-phase device ms (CUDA events), iterations, wall time with the copies,
and the float64 tensor-core flops counted from the shapes (E-step N d^2 C with the triangle skipped, covariance N d^2 C
with the symmetric half, means 2 N d C, C = n_init K summed over the iterations each init ran, the M-step's
also over the initialisation) against the data
sheet's 67 TFLOP/s.  The output check fits n_init = 1, max_iter = 3, tol = 0 at N = 20 000, K = 60 and compares with
scikit-learn on the same rows (its time is CPU time, on this host's cores).  Prints one JSON object.  Needs a device.

--covariance-type other than 'full' (the default, whose output is unchanged) adds the type to the JSON, counts that
type's DMMA flops (diag: E-step 2 N (2 d) C, M-step means and resp^T (X o X) 2 N d C each; spherical: E-step 2 N d C,
M-step as diag; tied: E-step N d^2 n_init (the triangle skipped, X P once per init), M-step means 2 N d C, X^T X once
per fit N d^2), and with --sklearn-fit times scikit-learn's whole fit (n_init = 10, the reference's settings) at each
shape on this host's cores.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP64_TC_TFLOPS = 67.0
D = 200


def rows(N, d=D, groups=80, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((groups, d))[rng.integers(0, groups, N)] + rng.standard_normal((N, d))
    return (X - X.mean(0)) / X.std(0)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:     # the card's name is part of every number below; report that it is missing
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="20000x60,20000x100,100000x60,100000x100")
    ap.add_argument("--no-check", action="store_true")
    ap.add_argument("--covariance-type", default="full", choices=("full", "diag", "tied", "spherical"))
    ap.add_argument("--sklearn-fit", action="store_true")
    a = ap.parse_args()
    cov = a.covariance_type
    import torch
    if not torch.cuda.is_available():
        sys.exit("gmm_bench: no CUDA device; the GPU mixture has no CPU path to time")
    from audiomuse_ai_b200 import clustering_gpu as cg
    out = {"card": card(), "d": D, "n_init": 10, "fp64_tensor_core_tflops_datasheet": FP64_TC_TFLOPS, "shapes": []}
    if cov != "full":
        out["covariance_type"] = cov
    cg.gmm_fit(rows(2000), 8, n_init=2, max_iter=2, random_state=0, covariance_type=cov)   # module load, first launches
    for s in a.shapes.split(","):
        N, K = map(int, s.split("x"))
        X = rows(N)
        t0 = time.perf_counter()
        f = cg.gmm_fit(X, K, n_init=10, random_state=1, intermediates=True, covariance_type=cov)
        wall = time.perf_counter() - t0
        e_iters = int(f.init_n_iter.sum()) * K             # component E-steps in the timed loop
        m_iters = e_iters + 10 * K                          # the M-steps, with the initialisation's
        if cov == "full":
            fl = {"estep": N * D * D * e_iters, "covariance": N * D * D * m_iters, "means": 2 * N * D * m_iters}
        elif cov == "tied":
            fl = {"estep": N * D * D * e_iters // K, "covariance": N * D * D, "means": 2 * N * D * m_iters}
        else:
            fl = {"estep": 2 * N * D * (1 if cov == "spherical" else 2) * e_iters,
                  "covariance": 2 * N * D * m_iters, "means": 2 * N * D * m_iters}
        em_ms = f.phase_ms["estep"] + f.phase_ms["mstep"]
        tot = sum(fl.values())
        out["shapes"].append({
            "N": N, "K": K, "phase_ms": f.phase_ms, "wall_s": wall, "n_iter_per_init": f.init_n_iter.tolist(),
            "best_n_iter": f.n_iter, "converged": f.converged, "flops": fl,
            "estep_tflops": fl["estep"] / f.phase_ms["estep"] / 1e9,
            "mstep_tflops": (fl["covariance"] + fl["means"]) / f.phase_ms["mstep"] / 1e9,
            "dmma_share_of_datasheet": tot / em_ms / 1e9 / FP64_TC_TFLOPS})
        if a.sklearn_fit:
            from sklearn.mixture import GaussianMixture
            t0 = time.perf_counter()
            m = GaussianMixture(K, covariance_type=cov, init_params="k-means++", n_init=10, reg_covar=1e-4,
                                random_state=1).fit(X)
            out["shapes"][-1].update(sklearn_fit_s=time.perf_counter() - t0, sklearn_n_iter=int(m.n_iter_),
                                     cpu_cores=os.cpu_count())
        print(json.dumps(out["shapes"][-1]), file=sys.stderr)
    if not a.no_check:
        from sklearn.mixture import GaussianMixture
        X = rows(20000)
        f = cg.gmm_fit(X, 60, n_init=1, max_iter=3, tol=0.0, random_state=3, covariance_type=cov)
        t0 = time.perf_counter()
        m = GaussianMixture(60, covariance_type=cov, init_params="k-means++", n_init=1, max_iter=3, tol=0.0, reg_covar=1e-4,
                            random_state=3).fit(X)
        cpu = time.perf_counter() - t0
        out["check"] = {
            "N": 20000, "K": 60, "max_iter": 3,
            "lower_bounds_rel": float(np.max(np.abs(np.array(f.lower_bounds) - m.lower_bounds_) / np.abs(m.lower_bounds_))),
            "means_abs": float(np.abs(f.means - m.means_).max()),
            "covariances_abs": float(np.abs(f.covariances - m.covariances_).max()),
            "precisions_cholesky_abs": float(np.abs(f.precisions_cholesky - m.precisions_cholesky_).max()),
            "sklearn_cpu_s": cpu, "cpu_cores": os.cpu_count(), "gpu_ms": sum(f.phase_ms.values())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
