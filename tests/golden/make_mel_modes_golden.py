#!/usr/bin/env python
"""Bits of the existing log-mel modes, so that a change to the mel kernel can be checked to leave them alone.

    python tests/golden/make_mel_modes_golden.py [--out PATH]     # needs a GPU; default tests/golden/mel_modes_golden.json

Runs the library of the tree this file sits in over seeded 1 s inputs: the CLAP student configuration (48 kHz, n_fft
2048, hop 480, 128 mels to 14 kHz) on float32 and int16 input with reflect padding (am_mel_cfg.framing 0), the
teacher's transposed n_fft 1024 layout, and the MusiCNN front end (16 kHz, n_fft 512, hop 256, 96 mels) with frames
starting at t * hop (framing 1), in both compressions, and records each output's shape and the SHA-256 of its bytes.
mel_modes_golden.json was written by the library as it was before the zero-pad mode (framing 2) was added to the
kernel."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CLAP = (48000, 2048, 480, 128, 0.0, 14000.0, 0)
TEACHER = (48000, 1024, 480, 64, 50.0, 14000.0, 1)
MUSICNN = (16000, 512, 256, 96, 0.0, 8000.0, 0)
# name -> (cfg, int16 input, framing, log_mode, seed)
CASES = {
    "clap_f32": (CLAP, False, 0, 0, 1),
    "clap_i16": (CLAP, True, 0, 0, 2),
    "teacher_f32": (TEACHER, False, 0, 0, 3),
    "musicnn_log1p": (MUSICNN, False, 1, 1, 4),
    "musicnn_db": (MUSICNN, False, 1, 0, 5),
    "clap_center0": (CLAP, False, 1, 0, 6),
}


def mel_case(name):
    from audiomuse_ai_b200 import _lib
    cfg_t, i16, framing, log_mode, seed = CASES[name]
    cfg = _lib.MelCfg(*cfg_t, framing, log_mode)
    lib = _lib.load()
    rng = np.random.default_rng(seed)
    n = cfg_t[0]
    x = (0.3 * rng.standard_normal((2, n))).clip(-1, 1).astype(np.float32)
    T = lib.am_mel_num_frames(C.byref(cfg), n)
    out = np.zeros((2, T, cfg_t[3]) if cfg_t[6] else (2, cfg_t[3], T), np.float32)
    pcm = (x * 32767.0).astype(np.int16) if i16 else x
    _lib.check(lib.am_mel_batch(_lib.ptr(pcm), int(i16), 2, n, C.byref(cfg), _lib.ptr(out)))
    return out


def digest(a):
    return {"shape": list(a.shape), "sha256": hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "mel_modes_golden.json"))
    args = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    with open(args.out, "w") as f:
        json.dump({name: digest(mel_case(name)) for name in CASES}, f, indent=1, sort_keys=True)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
