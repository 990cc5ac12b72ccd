#!/usr/bin/env python
"""CLAP text tower: per-query latency (B = 1, T = 77, the reference's single text-search query) and batch throughput
(B = 64, T = 77) of B200TextSession on roberta-base-sized random weights, each beside

* the weight-streaming floor: every split-bf16 weight byte (hi + lo = 4 bytes per non-embedding parameter) read once
  at the data sheet's 3.35 TB/s -- derived, not measured;
* the float32 oracle on the CPU (oracle/clap_text.py through PyTorch), the stand-in for the reference's CPU
  onnxruntime session.

Prints the card's name and power limit from the same run.  One JSON line per figure.

    python tools/text_bench.py [--iters 50] [--cpu-iters 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiomuse_ai_b200.clap_analyzer import B200TextSession  # noqa: E402
from oracle import clap_text as ct  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the figure is still printed, without its card
        return f"unknown ({e})"


def weight_bytes(cfg):
    H, F, P = cfg.hidden, cfg.ffn, cfg.proj
    per_layer = 4 * H * H + 2 * H * F  # Q, K, V, out; FFN up and down
    params = cfg.layers * per_layer + H * H + H * P + P * P
    return params, 4 * params


def feeds(cfg, B, T, seed=0):
    g = np.random.default_rng(seed)
    ids = g.integers(3, cfg.vocab, size=(B, T)).astype(np.int64)
    ids[:, 0] = 0
    mask = np.ones((B, T), np.int64)
    for b in range(B):  # queries of different lengths, padded to 77 as the reference's tokenizer does
        n = 4 + (b * 5) % (T - 4)
        ids[b, n:] = cfg.pad_id
        mask[b, n:] = 0
    return {"input_ids": ids, "attention_mask": mask}


def time_gpu(sess, feed, iters, warmup=5):
    for _ in range(warmup):
        sess.run(None, feed)
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        sess.run(None, feed)  # ends in a stream synchronise (the D2H copy of the embeddings)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def time_cpu(model, feed, iters):
    ids, mask = torch.from_numpy(feed["input_ids"]), torch.from_numpy(feed["attention_mask"])
    with torch.no_grad():
        model(ids, mask)
        ts = []
        for _ in range(iters):
            t0 = time.perf_counter()
            model(ids, mask)
            ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-iters", type=int, default=5)
    a = ap.parse_args()
    cfg = ct.ROBERTA_BASE
    model = ct.TextCLAP(cfg, "sdpa", "where").init_random(0).float().eval()
    sess = B200TextSession(blob=ct.export_onnx_bytes(model))
    params, wbytes = weight_bytes(cfg)
    floor = wbytes / HBM_BYTES_PER_S
    dev = card()
    print(json.dumps({"card": dev, "torch_cpu_threads": torch.get_num_threads(), "non_embedding_params": params,
                      "split_weight_bytes": wbytes, "weight_streaming_floor_ms": floor * 1e3}))
    for B, T, iters in ((1, 77, a.iters), (64, 77, max(5, a.iters // 5))):
        feed = feeds(cfg, B, T)
        g = time_gpu(sess, feed, iters)
        c = time_cpu(model, feed, a.cpu_iters)
        print(json.dumps({"B": B, "T": T, "gpu_ms": g * 1e3, "gpu_queries_per_s": B / g,
                          "floor_ms": floor * 1e3, "gpu_over_floor": g / floor, "cpu_fp32_ms": c * 1e3,
                          "cpu_queries_per_s": B / c, "speedup_vs_cpu": c / g, "card": dev}))
    sess.close()


if __name__ == "__main__":
    main()
