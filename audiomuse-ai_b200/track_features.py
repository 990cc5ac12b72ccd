"""analyze_track's tempo, energy and key on the GPU (tasks/analysis.py:344-365).

The per-track analysis job calls three librosa 0.11.0 functions on the 16 kHz waveform before the MusiCNN models:

    tempo, _ = librosa.beat.beat_track(y=audio, sr=sr)
    average_energy = np.mean(librosa.feature.rms(y=audio))
    chroma = librosa.feature.chroma_stft(y=audio, sr=sr)         # key and scale from its mean

All three run in one device call, am_track_features (csrc/track_features.cu), for a batch of tracks of any lengths:

    track_features(audios, sr=16000)  -> one dict per track: tempo, energy, key, scale, tuning, chroma_mean
    LibrosaFacade(original)           -> what tasks.analysis sees as `librosa` (integration.apply(analysis=...)):
                                         beat.beat_track(y=, sr=), feature.rms(y=) and feature.chroma_stft(y=, sr=) on
                                         the device, everything else from the original librosa module

beat_track's beat positions are not computed: the facade returns an empty int array for them, and analyze_track, the
only caller, discards them.  Input is validated on the host before the library is loaded: an empty track, a non-finite
sample or a sample rate outside [8000, 48000] raises ValueError.  There is no CPU fallback.

Parity is pinned against oracle/track_features.py, a float64 restatement of librosa 0.11.0's source, and its known
answers, not against librosa itself, which this project does not depend on.
"""
from __future__ import annotations

import ctypes as C
import threading

import numpy as np

from . import _lib

TEMPO, RMS, CHROMA = 1, 2, 4
HOP = 512
N_HIST = 100
MIN_SR, MAX_SR = 8000, 48000
KEYS = ['C', 'C#', 'D', 'D#', 'E', 'F', 'F#', 'G', 'G#', 'A', 'A#', 'B']
MAJOR_PROFILE = np.array([1, 0, 1, 0, 1, 1, 0, 1, 0, 1, 0, 1])
MINOR_PROFILE = np.array([1, 0, 1, 1, 0, 1, 0, 1, 1, 0, 1, 0])

_plans = {}
_plans_lock = threading.Lock()


def validate(audios, sr):
    """-> (samples f32, offsets i64[n + 1]); raises ValueError before any library load"""
    if not isinstance(sr, (int, np.integer)) or not MIN_SR <= int(sr) <= MAX_SR:
        raise ValueError(f"track features: sample rate {sr!r} is not an integer in [{MIN_SR}, {MAX_SR}]")
    if len(audios) == 0:
        raise ValueError("track features: no tracks")
    arrs = []
    for i, a in enumerate(audios):
        a = np.ascontiguousarray(a, dtype=np.float32)
        if a.ndim != 1 or a.size == 0:
            raise ValueError(f"track features: track {i} must be a non-empty 1-D waveform, got shape {a.shape}")
        if not np.isfinite(a).all():
            raise ValueError(f"track features: track {i} has non-finite samples")
        arrs.append(a)
    offsets = np.zeros(len(arrs) + 1, np.int64)
    offsets[1:] = np.cumsum([a.size for a in arrs])
    return np.concatenate(arrs), offsets


def _plan(sr: int):
    with _plans_lock:
        p = _plans.get(sr)
        if p is None:
            lib = _lib.load()
            h = C.c_void_p()
            _lib.check(lib.am_track_features_plan_create(int(sr), C.byref(h)))
            p = _plans[sr] = h
        return p


def plan_info(sr: int):
    """(tempogram lags, piptrack's first bin, one past its last bin) of the plan for sr"""
    win, kmin, kmax = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.load().am_track_features_plan_info(_plan(sr), C.byref(win), C.byref(kmin), C.byref(kmax)))
    return win.value, kmin.value, kmax.value


def compute(audios, sr=16000, what=TEMPO | RMS | CHROMA, intermediates=False):
    """One device call for a batch of tracks.  -> dict of per-track lists: 'tempo' float, 'rms' f32[1, T],
    'chroma' f32[12, T], 'tuning' float (for the flags asked), and with intermediates also 'onset_env' f32[T],
    'tempogram' f64[win], 'histogram' i32[100] and 'threshold' f32."""
    samples, offsets = validate(audios, sr)
    sr = int(sr)
    n = len(offsets) - 1
    T = 1 + np.diff(offsets) // HOP
    foff = np.zeros(n + 1, np.int64)
    foff[1:] = np.cumsum(T)
    lib = _lib.load()
    plan = _plan(sr)
    win = plan_info(sr)[0]
    tempo = np.zeros(n, np.float64) if what & TEMPO else None
    rms = np.zeros(int(foff[-1]), np.float32) if what & RMS else None
    chroma = np.zeros(12 * int(foff[-1]), np.float32) if what & CHROMA else None
    tuning = np.zeros(n, np.float64) if what & CHROMA else None
    env = np.zeros(int(foff[-1]), np.float32) if intermediates and what & TEMPO else None
    tg = np.zeros((n, win), np.float64) if intermediates and what & TEMPO else None
    hist = np.zeros((n, N_HIST), np.int32) if intermediates and what & CHROMA else None
    thr = np.zeros(n, np.float32) if intermediates and what & CHROMA else None

    def p(a):
        return None if a is None else _lib.ptr(a)

    _lib.check(lib.am_track_features(plan, _lib.ptr(samples), _lib.ptr(offsets), n, int(what), p(tempo), p(rms),
                                     p(chroma), p(tuning), p(env), p(tg), p(hist), p(thr)))
    out = {}
    if tempo is not None:
        out["tempo"] = [float(v) for v in tempo]
    if rms is not None:
        out["rms"] = [rms[foff[i]:foff[i + 1]][None, :] for i in range(n)]
    if chroma is not None:
        out["chroma"] = [chroma[12 * foff[i]:12 * foff[i + 1]].reshape(12, T[i]) for i in range(n)]
        out["tuning"] = [float(v) for v in tuning]
    if env is not None:
        out["onset_env"] = [env[foff[i]:foff[i + 1]] for i in range(n)]
        out["tempogram"] = list(tg)
    if hist is not None:
        out["histogram"] = list(hist)
        out["threshold"] = [np.float32(v) for v in thr]
    return out


def key_scale(chroma_mean):
    """tasks/analysis.py:349-365 as written: (key, scale).  Each major profile is its relative minor's profile rolled,
    so the best major and best minor correlations are equal and the strict `>` answers the relative minor."""
    major_correlations = np.array([np.corrcoef(chroma_mean, np.roll(MAJOR_PROFILE, i))[0, 1] for i in range(12)])
    minor_correlations = np.array([np.corrcoef(chroma_mean, np.roll(MINOR_PROFILE, i))[0, 1] for i in range(12)])
    major_key_idx = np.argmax(major_correlations)
    minor_key_idx = np.argmax(minor_correlations)
    if major_correlations[major_key_idx] > minor_correlations[minor_key_idx]:
        return KEYS[major_key_idx], 'major'
    return KEYS[minor_key_idx], 'minor'


def track_features(audios, sr=16000):
    """analyze_track's features for a batch of waveforms: one dict per track with tempo (float, bpm), energy
    (np.mean of the per-frame RMS, float32), key, scale, tuning and chroma_mean (f32[12])."""
    r = compute(audios, sr)
    out = []
    for i in range(len(r["tempo"])):
        cm = np.mean(r["chroma"][i], axis=1)
        key, scale = key_scale(cm)
        out.append({"tempo": r["tempo"][i], "energy": np.mean(r["rms"][i]), "key": key, "scale": scale,
                    "tuning": r["tuning"][i], "chroma_mean": cm})
    return out


# ------------------------------------------------------------------------------------------------ librosa facade
class _Forwarding:
    """Attribute access falls through to the same-named submodule of the original librosa."""

    def __init__(self, facade, name):
        self._facade, self._name = facade, name

    def __getattr__(self, attr):
        return getattr(getattr(self._facade._original(), self._name), attr)


class _Beat(_Forwarding):
    def beat_track(self, *args, **kwargs):
        """beat_track(y=, sr=) -> (np.array([tempo]), empty int array): beat positions are not computed"""
        if args or not set(kwargs) <= {"y", "sr"} or not self._facade._serves(kwargs.get("y")):
            return self._facade._original().beat.beat_track(*args, **kwargs)
        r = compute([kwargs["y"]], kwargs.get("sr", 22050), TEMPO)
        return np.array([r["tempo"][0]]), np.array([], dtype=int)


class _Feature(_Forwarding):
    def rms(self, *args, **kwargs):
        """rms(y=) -> f32[1, T]"""
        if args or set(kwargs) != {"y"} or not self._facade._serves(kwargs["y"]):
            return self._facade._original().feature.rms(*args, **kwargs)
        # rms never reads the sample rate; any supported rate gives the same frames
        return compute([kwargs["y"]], 16000, RMS)["rms"][0]

    def chroma_stft(self, *args, **kwargs):
        """chroma_stft(y=, sr=) -> f32[12, T]"""
        if args or not set(kwargs) <= {"y", "sr"} or "y" not in kwargs or not self._facade._serves(kwargs["y"]):
            return self._facade._original().feature.chroma_stft(*args, **kwargs)
        return compute([kwargs["y"]], kwargs.get("sr", 22050), CHROMA)["chroma"][0]


class LibrosaFacade:
    """Stands in for the `librosa` module inside tasks.analysis.  The three calls analyze_track makes, with exactly the
    keyword arguments it passes and a 1-D float32 waveform, run on the device, one track per call; any other argument,
    input or attribute (librosa.load, feature.melspectrogram, ...) goes to `original`, the module tasks.analysis
    imported (imported on first use when None)."""

    def __init__(self, original=None):
        self.__dict__["_orig"] = original
        self.__dict__["beat"] = _Beat(self, "beat")
        self.__dict__["feature"] = _Feature(self, "feature")

    def _original(self):
        if self._orig is None:
            import importlib

            self.__dict__["_orig"] = importlib.import_module("librosa")
        return self._orig

    @staticmethod
    def _serves(y):
        return isinstance(y, np.ndarray) and y.ndim == 1 and y.dtype == np.float32

    def __getattr__(self, name):
        return getattr(self._original(), name)
