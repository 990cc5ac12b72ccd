"""Mirror of the MusiCNN spectrogram front end of ``tasks/analysis.py:368-391`` on the GPU mel kernel (SURVEY 8(f)
row 4: a sibling tower sharing K1's machinery).

    musicnn_patches(audio, sr=16000) -> float32 (n_patches, 187, 96) | None

The reference computes ``librosa.feature.melspectrogram(y, sr=16000, n_fft=512, hop_length=256, n_mels=96,
window='hann', center=False, power=2.0, norm='slaney', htk=False)``, compresses with ``log10(1 + 10000 x)`` and cuts
non-overlapping patches of 187 frames, transposed to (frames, mels).  Here the mel + compression is one launch of
``mel_kernel`` in its center=False / log1p-style mode (``am_mel_batch`` with framing 1, log_mode 1); the patch cut is
a reshape.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib

N_MELS, HOP, N_FFT, FRAME_SIZE = 96, 256, 512, 187


def musicnn_log_mel(audio: np.ndarray, sr: int = 16000) -> np.ndarray:
    """float32 (96, T): log10(1 + 10000 * mel_power), T = 1 + (len - 512) // 256."""
    lib = _lib.load()
    x = np.ascontiguousarray(audio, dtype=np.float32).reshape(1, -1)
    cfg = _lib.MelCfg(int(sr), N_FFT, HOP, N_MELS, 0.0, float(sr) / 2.0, 0, framing=1, log_mode=1)
    T = int(lib.am_mel_num_frames(C.byref(cfg), x.shape[1]))
    if T <= 0:  # shorter than one frame
        return np.zeros((N_MELS, 0), dtype=np.float32)
    out = np.empty((1, N_MELS, T), dtype=np.float32)
    _lib.check(lib.am_mel_batch(_lib.ptr(x), 0, 1, x.shape[1], C.byref(cfg), _lib.ptr(out)))
    return out[0]


def musicnn_patches(audio: np.ndarray, sr: int = 16000) -> Optional[np.ndarray]:
    """(n_patches, 187, 96) float32, or None when the track is too short for one patch (analysis.py:378-381)."""
    log_mel = musicnn_log_mel(audio, sr)
    n = log_mel.shape[1] // FRAME_SIZE
    if n == 0:
        return None
    return np.ascontiguousarray(log_mel[:, : n * FRAME_SIZE].reshape(N_MELS, n, FRAME_SIZE).transpose(1, 2, 0), dtype=np.float32)
