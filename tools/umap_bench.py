"""Per-stage times of the GPU UMAP (projection.umap_fit_transform) at 20 000 and 100 000 x 200 (k-NN, graph, the
initialisation split into the device eigensolver and the host's component placement, layout, host API total), the
layout kernel's summed device time against the layout's wall time (the cost of one launch per epoch), its edge
samples/s and gathered bytes over kernel time, and the CPU restatement (oracle/umap.py's numba sequential SGD,
not umap-learn) at 20 000 rows.  Prints one JSON object; needs a CUDA device.

    python tools/umap_bench.py [--sizes 20000,100000] [--cpu-rows 20000] [--repeats 3]
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


def data(n, d=200, seed=0):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((60, d)) * 0.8
    return (c[rng.integers(0, 60, n)] + rng.standard_normal((n, d))).astype(np.float32)


def layout_counts(W, eps, n_epochs, neg_rate=5.0):
    """(attractive samples, negative samples) over the whole schedule: the kernel's work, counted on the host from the
    same float64 schedule"""
    eps = np.asarray(eps, np.float64)
    epsn = eps / neg_rate
    nxt, nxn = eps.copy(), epsn.copy()
    att = neg = 0
    for n in range(n_epochs):
        e = np.flatnonzero(nxt <= n)
        att += e.size
        nxt[e] += eps[e]
        nn = ((n - nxn[e]) / epsn[e]).astype(np.int64)
        neg += int(nn.sum())
        nxn[e] += nn * epsn[e]
    return att, neg


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20000,100000")
    ap.add_argument("--cpu-rows", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from audiomuse_ai_b200 import _lib, projection
    _lib.check(_lib.load().am_init(0))
    out = {"gpu": gpu_info(), "sizes": {}}
    projection.umap_fit_transform(data(2000), n_epochs=20)          # module load, first launches
    for n in (int(s) for s in args.sizes.split(",")):
        X = data(n)
        runs = []
        for _ in range(args.repeats):
            det = {}
            projection.umap_fit_transform(X, seed=0, details=det)
            r = {k: det[k] for k in ("knn_ms", "graph_ms", "init_ms", "eigensolver_ms", "layout_ms", "total_ms")}
            r["init_host_ms"] = r["init_ms"] - r["eigensolver_ms"]      # component placement, noise, rescale
            runs.append(r)
        best = {k: min(r[k] for r in runs) for k in runs[0]}
        # launch scheme: the layout's device time summed over its per-epoch kernels (CUDA events around each launch,
        # a separate run) against the host-observed layout time; the difference is what launching costs
        _lib.profile_enable(True)
        _lib.profile_report()
        with projection.UmapGraph(X) as g:
            graph_prof = _lib.profile_report()       # the graph stage's kernels, for the per-kernel split
            G = g.graph()
            Y0 = projection.initial_layout(g.X, G["W"], seed=0)
            a, b = projection.find_ab_params()
            _lib.profile_report()
            g.layout(Y0, a, b, seed=0)
            prof = _lib.profile_report()
        _lib.profile_enable(False)
        kern = {k: v for k, v in prof.items() if "layout_epoch_kernel" in k}
        kernel_ms = sum(v["ms"] if isinstance(v, dict) else v for v in kern.values())
        att, neg = layout_counts(det["W"], det["eps"], det["n_epochs"])
        # per sample: the edge's index and schedule (4 + 8 + 8 + 8 bytes read, 16 written once sampled), the other
        # end's 8-byte row; per negative sample one 8-byte row; per vertex and epoch its row pointers and rows
        nnz = det["nnz"]
        gathered = (att * (8 + 16 + 16) + neg * 8 + det["n_epochs"] * (n * (16 + 16) + nnz * 12))
        t = kernel_ms / 1e3
        out["sizes"][n] = dict(best, runs=runs, nnz=nnz, n_epochs=det["n_epochs"], components=det.get("components"),
                               eigensolver_calls=det["eigensolver_calls"], layout_kernel_ms=kernel_ms,
                               layout_launch_gap_ms=best["layout_ms"] - kernel_ms, layout_profile=kern,
                               graph_kernels_ms={k: round(v["ms"], 3) for k, v in graph_prof.items()},
                               max_row_nnz=int(np.diff(det["W"].indptr).max()),
                               attractive_samples=att, negative_samples=neg,
                               edge_samples_per_s=(att + neg) / t, gathered_GB_per_s=gathered / t / 1e9)
        print(json.dumps({n: out["sizes"][n]}), flush=True)
    if args.cpu_rows:
        from oracle import umap as ou
        X = data(args.cpu_rows)
        g = ou.fuzzy_graph(X)
        a, b = ou.find_ab_params()
        Y0 = ou.initial_layout(X, g["W"], np.random.default_rng(0))
        ou.sgd_sequential(Y0[:10], g["W"][:10, :10], g["eps"][:0], 1, a, b, 0)   # numba compile
        t0 = time.perf_counter()
        ou.sgd_sequential(Y0, g["W"], g["eps"], g["n_epochs"], a, b, 0)
        out["cpu_restatement_sgd_s"] = {args.cpu_rows: time.perf_counter() - t0,
                                        "what": "oracle/umap.py numba sequential SGD, one thread"}
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
