"""Time the mel kernel (csrc/mel.cu) alone at the benchmark shape: am_mel_batch_dev over 256 seeded 10 s windows of
480 000 int16 samples, student config (n_fft 2048, hop 480, 128 mels, fmax 14 kHz), T = 1001 frames per window.

Prints ms per 256 windows (CUDA events over --iters launches after a warm-up), the algorithmic HBM rate and the FP32
rate with the byte and flop counts bench.py uses, and the card name and power limit.  With --tree DIR (repeatable) a
copy of each such tree is built in a temporary directory (tools/fused_block_phases.build_copy), and all trees are
timed in turn, round after round, in child processes; each one's log-mel output is compared bit for bit with this
tree's.  Needs an H100.

    python tools/mel_bench.py [--iters N] [--rounds R] [--tree DIR ...]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from fused_block_phases import build_copy  # noqa: E402

WINDOWS, N_SAMPLES, T, N_MELS = 256, 480000, 1001, 128
# bench.py's counts: PCM16 in + log-mel out, and 1001 frames x (real FFT + power + sparse mel + log) flops per window
BYTES = (N_SAMPLES * 2 + N_MELS * T * 4) * WINDOWS
FLOPS = T * (56320 + 3 * 1025 + 2 * 1176 + 128) * WINDOWS
HBM_GBS, FP32_TFLOPS = 3350.0, 67.0  # H100 SXM data sheet (700 W)

CHILD = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from audiomuse_ai_b200 import clap_analyzer as ca
pcm = torch.from_numpy(np.load(sys.argv[2])).cuda()
iters = int(sys.argv[4])
B, n = pcm.shape
plan = ca.MelPlan()
out = torch.empty((B, plan.cfg.n_mels, 1 + n // plan.cfg.hop), dtype=torch.float32, device="cuda")
stream = torch.cuda.current_stream()
run = lambda: plan.mel_dev(pcm.data_ptr(), True, B, n, out.data_ptr(), stream.cuda_stream)
for _ in range(3):
    run()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(stream)
for _ in range(iters):
    run()
e1.record(stream)
torch.cuda.synchronize()
np.save(sys.argv[3], out.cpu().numpy())
print(json.dumps({"ms": e0.elapsed_time(e1) / iters}))
"""


def gpu_info():
    if not shutil.which("nvidia-smi"):
        return "nvidia-smi not found"
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True).stdout.strip()


def run_child(tree, pcm_path, out_path, iters):
    r = subprocess.run([sys.executable, "-c", CHILD, tree, pcm_path, out_path, str(iters)], capture_output=True,
                       text=True)
    if r.returncode != 0:
        sys.exit(f"mel child for {tree} failed:\n{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])["ms"]


def report(label, ms):
    gbs = BYTES / (ms * 1e-3) / 1e9
    tfs = FLOPS / (ms * 1e-3) / 1e12
    print(f"  {label:8s} {ms:8.3f} ms / {WINDOWS} windows   {gbs:7.1f} GB/s ({gbs / HBM_GBS:.3f} of HBM)   "
          f"{tfs:6.2f} TFLOP/s fp32 ({tfs / FP32_TFLOPS:.3f} of peak)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50, help="timed launches per measurement (at least 20)")
    ap.add_argument("--rounds", type=int, default=3, help="measurements per tree, alternating with --tree")
    ap.add_argument("--tree", action="append", default=[], help="another repository tree to build and compare "
                                                                 "against (repeatable)")
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")
    print("gpu: " + gpu_info())
    sys.path.insert(0, ROOT)
    from audiomuse_ai_b200 import corpus
    tmp = tempfile.mkdtemp(prefix="mel_bench_")
    try:
        pcm_path = os.path.join(tmp, "pcm.npy")
        np.save(pcm_path, corpus.synth_pcm_batch(WINDOWS))
        trees = {"this": ROOT}  # label -> built tree
        names = {"this": ROOT}  # label -> tree as given
        for i, src in enumerate(args.tree):
            label = f"tree{i + 1}"
            trees[label] = os.path.join(tmp, label)
            names[label] = src
            os.makedirs(trees[label])
            build_copy(os.path.abspath(src), trees[label], nvcc_flags="")
        times = {k: [] for k in trees}
        for _ in range(args.rounds):
            for k, tree in trees.items():
                times[k].append(run_child(tree, pcm_path, os.path.join(tmp, k + ".npy"), args.iters))
        for k, ts in times.items():
            print(f"{k} ({names[k]}), {args.iters} launches per measurement:")
            for ms in ts:
                report("", ms)
        a = np.load(os.path.join(tmp, "this.npy"))
        for k in list(trees)[1:]:
            b = np.load(os.path.join(tmp, k + ".npy"))
            if np.array_equal(a.view(np.uint32), b.view(np.uint32)):
                print(f"{k}: log-mel bit-identical to this tree's ({a.size} values)")
            else:
                d = np.abs(a.astype(np.float64) - b)
                print(f"{k}: log-mel differs from this tree's in {int(np.count_nonzero(a != b))} of {a.size} values, "
                      f"max |dB| = {d.max():.3e}")
            print(f"{k}: this tree is {np.median(times[k]) / np.median(times['this']):.2f}x as fast (median over rounds)")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
