"""Device time of the encoder's late phase at bench.py's shapes (256 windows of 10 s), against its floors.  Needs an H100.

Blocks 5-8 of the PhiNet trunk have more output channels than the fused block kernel takes, so each runs layer by
layer: expansion GEMM -> dw3x3 -> projection GEMM over all 256 windows.  Two views:

* per GEMM: `am_bench_gemm` (debug library) at each layer's exact (M, N, K), CUDA events around `--iters` launches after
  a warm-up, bf16 out without bias or residual; ms, achieved GB/s and TFLOP/s, and the share of the larger of the two
  floors (bf16 A + B + D bytes over 3.35 TB/s, 2 M N K flop over 989 TFLOP/s, the H100 SXM data sheet);
* per kernel: the whole bench.py step (same seeded weights and PCM) under the library's per-launch event profiler, ms
  per step of every kernel, so the dw3x3 launches, the head and the GEMMs' real epilogues (bias, ReLU6, residual)
  are there too.

--root DIR times the library built in another checkout (e.g. the parent commit's) with this script.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

HBM_TBS = 3.35
BF16_TFLOPS = 989.0

# (layer, M, N, K, residual): M = 256 windows x output pixels (126 x 16 at block 5's input, 63 x 8 after its
# stride-2 depthwise, 32 x 4 after block 7's); N, K = the padded channel counts of the 1x1 convolutions
LAYERS = [
    ("block 5 expand", 516096, 736, 144, False),
    ("block 5 project", 129024, 288, 736, False),
    ("block 6 expand", 129024, 1408, 288, False),
    ("block 6 project (+res)", 129024, 288, 1408, True),
    ("block 7 expand", 129024, 1360, 288, False),
    ("block 7 project", 32768, 576, 1360, False),
    ("block 8 expand", 32768, 2592, 576, False),
    ("block 8 project (+res)", 32768, 576, 2592, True),
]


def floors(M, N, K, residual):
    """(bytes, flop, HBM floor ms, tensor floor ms) of one launch"""
    nbytes = 2 * (M * K + N * K + M * N * (2 if residual else 1))
    flop = 2 * M * N * K
    return nbytes, flop, nbytes / (HBM_TBS * 1e12) * 1e3, flop / (BF16_TFLOPS * 1e12) * 1e3


def gpu_line():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def per_gemm(lib, _lib, iters):
    print("| layer | M x K -> N | ms | GB/s | TFLOP/s | HBM floor | tensor floor | share of the larger |")
    print("|---|---|---|---|---|---|---|---|")
    tot = tot_floor = 0.0
    for name, M, N, K, res in LAYERS:
        ms = C.c_double(0)
        _lib.check_debug(lib.am_bench_gemm(M, N, K, 3, C.byref(ms)))  # warm-up (and the first launch inside)
        _lib.check_debug(lib.am_bench_gemm(M, N, K, iters, C.byref(ms)))
        nbytes, flop, f_hbm, f_tc = floors(M, N, K, False)  # what am_bench_gemm moves: no residual
        t = ms.value
        floor = max(f_hbm, f_tc)
        tot += t
        tot_floor += floor
        print(f"| {name} | {M} x {K} -> {N} | {t:.3f} | {nbytes / t / 1e6:.0f} | {flop / t / 1e9:.0f} | {f_hbm:.3f} | "
              f"{f_tc:.3f} | {floor / t:.0%} |", flush=True)
    print(f"| sum | | {tot:.3f} | | | | | {tot_floor / tot:.0%} |")


def per_kernel(steps):
    import numpy as np  # noqa: F401
    import torch

    from audiomuse_ai_b200 import _lib, clap_analyzer as ca, corpus, weights

    n_tracks, n_samples = 256, 480000  # bench.py's step
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.check(_lib.load().am_init(0))
    sess = ca.B200Session.from_state_dict(weights.random_state_dict(0))
    plan = ca.MelPlan()
    pcm = torch.from_numpy(corpus.synth_pcm_batch(n_tracks, start=0)).to(dev)
    offs = torch.arange(n_tracks + 1, dtype=torch.int32, device=dev)
    out = torch.empty((n_tracks, sess.embedding_dim), dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev)

    def step():
        sess.embed_tracks_dev(plan, pcm.data_ptr(), n_samples, offs.data_ptr(), n_tracks, n_tracks, out.data_ptr(),
                              stream.cuda_stream)

    for _ in range(3):
        step()
    torch.cuda.synchronize(dev)
    _lib.profile_enable(True)
    _lib.profile_report()  # clear
    for _ in range(steps):
        step()
    torch.cuda.synchronize(dev)
    prof = _lib.profile_report()
    _lib.profile_enable(False)
    print(f"\nper kernel, ms per step ({steps} steps of {n_tracks} windows):")
    total = 0.0
    for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"]):
        total += v["ms"] / steps
        print(f"  {k:40s} {v['ms'] / steps:8.3f} ms  ({v['count'] // steps} launches)")
    gemm = sum(v["ms"] for k, v in prof.items() if "gemm_wgmma_kernel" in k) / steps
    print(f"  {'all gemm_wgmma_kernel':40s} {gemm:8.3f} ms\n  {'all kernels':40s} {total:8.3f} ms")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    from audiomuse_ai_b200 import _lib

    print(f"GPU: {gpu_line()}  (name, power limit, max SM clock)")
    print(f"library: {_lib.LIB_PATH}\n")
    per_gemm(_lib.load_debug(), _lib, args.iters)
    per_kernel(args.steps)


if __name__ == "__main__":
    main()
