"""Tracks per second of analyze_track's tempo / energy / chroma (am_track_features: tempo, per-frame RMS and the tuned
chromagram in one device call per batch) on batches of seeded 16 kHz tracks of 30 s, 3 min and 10 min
(oracle/track_features.synth_track 'drums'), against oracle/track_features.py's numpy restatement of the same three
librosa 0.11.0 calls on the CPU (one track at a time, as analyze_track runs them).  The CPU side is the float64
restatement, not librosa, which this project does not depend on.  A host clock around each device call (it returns after its
results are copied back), after a warm-up call of the same batch; median of --reps calls.  Prints the card and its
power limit, then one JSON line per track length.

    python tools/track_features_bench.py [--batch 16] [--reps 5] [--cpu-tracks 1]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiomuse_ai_b200 import track_features as tf  # noqa: E402
from oracle import track_features as otf  # noqa: E402
from tools.radius_walk_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-tracks", type=int, default=1)
    args = ap.parse_args()
    print(card())
    for seconds in (30.0, 180.0, 600.0):
        ys = [otf.synth_track("drums", seconds, 16000, 100 + i) for i in range(args.batch)]
        tf.compute(ys, 16000)                       # warm-up: plan, module load, allocation sizes
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r = tf.compute(ys, 16000)
            times.append(time.perf_counter() - t0)
        dev = float(np.median(times))
        t0 = time.perf_counter()
        for y in ys[:args.cpu_tracks]:
            o = otf.track_features(y, 16000)
        cpu = (time.perf_counter() - t0) / args.cpu_tracks
        same = r["tempo"][0] == o["tempo"] if args.cpu_tracks == 1 else None
        print(json.dumps({"seconds": seconds, "batch": args.batch, "device_s": round(dev, 5),
                          "device_tracks_per_s": round(args.batch / dev, 2),
                          "cpu_restatement_s_per_track": round(cpu, 3),
                          "cpu_restatement_tracks_per_s": round(1.0 / cpu, 3),
                          "speedup": round(cpu * args.batch / dev, 1), "first_track_tempo_equal": same}))


if __name__ == "__main__":
    main()
