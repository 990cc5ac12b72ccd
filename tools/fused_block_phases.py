"""Where the cycles of each fused inverted-residual block (csrc/fused_block.cu) go, at the benchmark shape: the shipped
student (alpha 3), 256 windows of T = 1001 frames.

Builds a copy of the package with -DAM_FUSED_PHASES in a directory of its own (the tree's library is not touched), so
that the kernel's producer and each consumer warpgroup sum clock64 deltas per phase and the launcher prints the sums of
every launch.  One warm-up step, then one measured step in a child process; prints per block the cycles per 64-channel
chunk of each phase (per CTA, averaged over CTAs and early-phase passes) for the producer and both consumers.  The
counters add a few instructions per phase, so the totals run slightly above an uninstrumented build.  Needs an H100.

    python tools/fused_block_phases.py [--tree DIR] [--build-dir DIR]
"""
import argparse
import math
import os
import re
import shutil
import subprocess
import sys
import tempfile

WINDOWS, T = 256, 1001
# (H, W, cin_p, cmid_p or None without expansion, cout_p, stride) of the blocks that fuse, alpha 3, T = 1001
BLOCKS = [(501, 64, 144, None, 80, 1), (501, 64, 80, 432, 80, 2), (251, 32, 80, 416, 80, 1),
          (251, 32, 80, 400, 144, 2), (126, 16, 144, 768, 144, 1)]
CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from audiomuse_ai_b200 import clap_analyzer as ca, weights
cfg = weights.StudentConfig()
sess = ca.B200Session.from_state_dict(weights.random_state_dict(0, cfg), cfg)
mel = (np.random.default_rng(0).standard_normal((%d, 1, 128, %d)) * 12 - 30).astype(np.float32)
sess.run(None, {"mel_spectrogram": mel})
print("measured step", file=sys.stderr, flush=True)
sess.run(None, {"mel_spectrogram": mel})
""" % (WINDOWS, T)
LINE = re.compile(r"fused_phases H=(\d+) W=(\d+) cin=(\d+) cmid=(\d+) cout=(\d+) S=(\d+) stages=(\d+) grid=(\d+) "
                  r"tiles=(\d+)(.*)")


def build_copy(tree, dst, nvcc_flags="-DAM_FUSED_PHASES"):
    """The package and its import stub from `tree`, built into `dst` with `nvcc_flags` (by default the phase
    counters compiled in)."""
    for name in ("audiomuse-ai_b200", "include"):
        shutil.copytree(os.path.join(tree, name), os.path.join(dst, name), dirs_exist_ok=True,
                        ignore=shutil.ignore_patterns("*.so", "build", "__pycache__"))
    shutil.copy(os.path.join(tree, "audiomuse_ai_b200.py"), dst)
    env = dict(os.environ, AM_EXTRA_NVCC_FLAGS=nvcc_flags)
    subprocess.run([sys.executable, os.path.join(dst, "audiomuse-ai_b200", "build_native.py")], env=env, check=True,
                   stdout=subprocess.DEVNULL)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="repository tree whose kernel is measured (default: this one)")
    ap.add_argument("--build-dir", default=None, help="where to build the instrumented copy (default: a temporary "
                                                      "directory, removed afterwards)")
    args = ap.parse_args()
    if shutil.which("nvidia-smi"):
        print("gpu: " + subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    tmp = None if args.build_dir else tempfile.mkdtemp(prefix="fused_phases_")
    dst = args.build_dir or tmp
    try:
        os.makedirs(dst, exist_ok=True)
        build_copy(os.path.abspath(args.tree), dst)
        r = subprocess.run([sys.executable, "-c", CHILD, dst], capture_output=True, text=True)
        if r.returncode != 0:
            sys.exit(r.stderr[-3000:])
    finally:
        if tmp:
            shutil.rmtree(tmp, ignore_errors=True)
    lines = r.stderr.split("measured step", 1)[1].splitlines()
    sums = {}  # block -> [launches, CTAs, tiles, stages, {(wg, phase): cycles}]
    for ln in lines:
        m = LINE.search(ln)
        if not m:
            continue
        H, W, cin, cmid, cout, S, stages, grid, tiles = (int(v) for v in m.groups()[:9])
        blk = next(i for i, (h, w, ci, _, co, s) in enumerate(BLOCKS) if (h, w, ci, co, s) == (H, W, cin, cout, S))
        e = sums.setdefault(blk, [0, 0, 0, stages, {}])
        e[0] += 1
        e[1] += grid
        e[2] += tiles
        for kv in m.group(10).split():
            k, v = kv.split("=")
            e[4][k] = e[4].get(k, 0) + int(v)
    assert sorted(sums) == list(range(len(BLOCKS))), f"blocks seen: {sorted(sums)}"
    for blk, (launches, ctas, tiles, stages, cyc) in sorted(sums.items()):
        H, W, cin, cmid, cout, S = BLOCKS[blk]
        chunks = math.ceil((cmid or cin) / 64)
        per_cta_chunks = tiles / ctas * chunks  # chunks each CTA runs, on average
        print(f"\nblock {blk}: {H}x{W}x{cin} -> {cmid or '-'} -> {cout}, stride {S}; {launches} launches, "
              f"{stages}-stage ring, {tiles / ctas:.0f} tiles x {chunks} chunks per CTA")
        phases = [k.split(".", 1)[1] for k in cyc if k.startswith("wg1.")]
        print(f"  {'cycles per chunk':16s} {'producer':>9s} {'consumer 1':>11s} {'consumer 2':>11s}")
        for p in phases:
            row = [cyc.get(f"wg{w}.{p}", 0) / ctas / per_cta_chunks for w in range(3)]
            if any(row):
                print(f"  {p:16s} {row[0]:9.0f} {row[1]:11.0f} {row[2]:11.0f}")
        tot = [sum(v for k, v in cyc.items() if k.startswith(f"wg{w}.")) / ctas / per_cta_chunks for w in range(3)]
        print(f"  {'total':16s} {tot[0]:9.0f} {tot[1]:11.0f} {tot[2]:11.0f}")


if __name__ == "__main__":
    main()
