"""Device time of each fused inverted-residual block (csrc/fused_block.cu) at the benchmark shape: the shipped student
(alpha 3), 256 windows of T = 1001 frames.  torch.profiler (CUDA activities, a run of its own) records every kernel of
a few steps; the fused launches of one step come in a fixed order (blocks 0-3 per early-phase pass, then block 4 over
all windows), which attributes them to blocks.  Prints ms, issued MMA TFLOP/s and compulsory HBM GB/s per block
against the H100 SXM data-sheet floors (989 TFLOP/s dense bf16, 3.35 TB/s), with the card's name and power limit.
Needs an H100."""
import math
import subprocess
import sys

import numpy as np

sys.path.insert(0, ".")
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from audiomuse_ai_b200 import clap_analyzer as ca, weights  # noqa: E402

WINDOWS, T, STEPS = 256, 1001, 3
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
# (H, W, cin_p, cmid_p or None without expansion, cout_p, stride, tile height) of the blocks that fuse, alpha 3,
# T = 1001; the plan gives blocks 0 and 2 tall (16 x 8) tiles
BLOCKS = [(501, 64, 144, None, 80, 1, 16), (501, 64, 80, 432, 80, 2, 8), (251, 32, 80, 416, 80, 1, 16),
          (251, 32, 80, 400, 144, 2, 8), (126, 16, 144, 768, 144, 1, 8)]


def per_window(H, W, cin_p, cmid_p, cout_p, S, th):
    """(issued MMA FLOP, compulsory HBM bytes) of one window: th x 8 output tiles, the expansion over the halo pixels
    ((th - 1) S + 3 rows of 7 S + 3, 184 per 128 outputs for the tall tile) rounded up to 8-pixel atoms (its N) with
    the K steps of 16 past cin_p skipped, the projection over the tile's pixels and cout_p columns."""
    Ho, Wo = (H - 1) // S + 1, (W - 1) // S + 1
    tiles = math.ceil(Ho / th) * math.ceil(Wo / 8)
    hp = math.ceil((((th - 1) * S + 3) * (7 * S + 3)) / 8) * 8
    cm = cmid_p or cin_p
    chunks = math.ceil(cm / 64)
    expand = 0 if cmid_p is None else 2 * hp * 64 * chunks * cin_p
    project = 2 * th * 8 * cout_p * cm
    return tiles * (expand + project), 2 * (H * W * cin_p + Ho * Wo * cout_p)


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"gpu: {gpu}")
    cfg = weights.StudentConfig()
    sess = ca.B200Session.from_state_dict(weights.random_state_dict(0, cfg), cfg)
    mel = (np.random.default_rng(0).standard_normal((WINDOWS, 1, 128, T)) * 12 - 30).astype(np.float32)
    for _ in range(2):
        sess.run(None, {"mel_spectrogram": mel})
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(STEPS):
            sess.run(None, {"mel_spectrogram": mel})
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                  and "fused_block_kernel" in e.name), key=lambda e: e.time_range.start)
    per_step = len(evs) // STEPS
    assert per_step * STEPS == len(evs) and (per_step - 1) % 4 == 0, f"{len(evs)} fused launches in {STEPS} steps"
    passes = (per_step - 1) // 4
    us = [0.0] * len(BLOCKS)
    for s in range(STEPS):
        step = evs[s * per_step:(s + 1) * per_step]
        for i, e in enumerate(step):
            us[4 if i == per_step - 1 else i % 4] += e.time_range.end - e.time_range.start
    total = 0.0
    print(f"{passes} early-phase passes per step; per 256-window step:")
    print("block   ms     TFLOP/s  GB/s   share of the larger floor")
    for b, shape in enumerate(BLOCKS):
        ms = us[b] / STEPS / 1e3
        flop, byt = (v * WINDOWS for v in per_window(*shape))
        floor_ms = max(flop / PEAK_TFLOPS / 1e9, byt / PEAK_TBS / 1e9)
        total += ms
        print(f"{b:5d} {ms:7.3f} {flop / ms / 1e9:8.1f} {byt / ms / 1e6:7.1f}  {floor_ms / ms:6.1%}")
    print(f"total {total:7.3f} ms")


if __name__ == "__main__":
    main()
