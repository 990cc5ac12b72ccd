"""Host-side mirror of the reference's ``tasks/clap_analyzer.py`` audio path on the GPU library.

Same names, argument meaning and error behaviour as the reference functions they replace:

    compute_mel_spectrogram(audio_data, sr=48000)     tasks/clap_analyzer.py:417-464
    analyze_audio_file(audio_path)                    tasks/clap_analyzer.py:467-574
    initialize_clap_audio_model / get_clap_audio_model / unload_clap_audio_only /
    unload_clap_model / is_clap_model_loaded / is_clap_audio_loaded / is_clap_available
                                                      tasks/clap_analyzer.py:47-165,387-393,690-699
    B200Session.run(None, {'mel_spectrogram': mel})   the ORT-session duck type used at :534

plus the batched entry points the reference lacks (it feeds one 10 s window per call):

    analyze_audio_batch(waveforms)    many tracks -> one fused PCM -> mel -> encoder -> pool pass
    embed_pcm16_windows(...)          lowest-level: int16 windows + offsets -> track embeddings

There is no CPU fallback here: if libaudiomuse_b200.so or the GPU is missing the lifecycle
functions return False / raise like the reference does when onnxruntime cannot load the model,
and ``analyze_audio_file`` returns ``(None, 0, 0)`` after logging, exactly the reference contract.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
import threading
from types import SimpleNamespace
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .weights import StudentConfig, export_blob

logger = logging.getLogger("tasks.clap_analyzer")

SAMPLE_RATE = 48000
SEGMENT_LENGTH = 480000   # 10 s at 48 kHz
HOP_LENGTH = 240000       # 5 s (50 % overlap)

try:  # inside the AudioMuse-AI tree the real config module wins (config.py:374-408)
    import config as config  # type: ignore
    if not hasattr(config, "CLAP_ENABLED"):
        raise ImportError
except Exception:  # standalone: same names, same defaults
    config = SimpleNamespace(
        CLAP_ENABLED=True,
        CLAP_EMBEDDING_DIMENSION=512,
        CLAP_AUDIO_N_MELS=128, CLAP_AUDIO_N_FFT=2048, CLAP_AUDIO_HOP_LENGTH=480,
        CLAP_AUDIO_FMIN=0, CLAP_AUDIO_FMAX=14000, CLAP_AUDIO_MEL_TRANSPOSE=False,
        CLAP_AUDIO_MODEL_PATH=os.environ.get("CLAP_AUDIO_MODEL_PATH", "/app/model/model_epoch_36.onnx"),
        AUDIO_LOAD_TIMEOUT=int(os.environ.get("AUDIO_LOAD_TIMEOUT", "600")),
        CLAP_B200_WEIGHTS_PATH=os.environ.get("CLAP_B200_WEIGHTS_PATH", ""),
    )

_audio_session = None          # module-global singleton, like the reference's _audio_session
_session_lock = threading.Lock()


def _mel_cfg(transpose=None) -> _lib.MelCfg:
    tr = getattr(config, "CLAP_AUDIO_MEL_TRANSPOSE", False) if transpose is None else transpose
    return _lib.MelCfg(SAMPLE_RATE,
                       int(getattr(config, "CLAP_AUDIO_N_FFT", 2048)),
                       int(getattr(config, "CLAP_AUDIO_HOP_LENGTH", 480)),
                       int(getattr(config, "CLAP_AUDIO_N_MELS", 128)),
                       float(getattr(config, "CLAP_AUDIO_FMIN", 0)),
                       float(getattr(config, "CLAP_AUDIO_FMAX", 14000)),
                       1 if tr else 0)


# --------------------------------------------------------------------------- K1
def compute_mel_spectrogram(audio_data: np.ndarray, sr: int = 48000) -> np.ndarray:
    """Log-mel of one waveform on the GPU; parameters are read from ``config`` at call time.
    Returns float32 (1, 1, n_mels, T), or (1, 1, T, n_mels) when CLAP_AUDIO_MEL_TRANSPOSE."""
    return compute_mel_spectrogram_batch(np.asarray(audio_data, dtype=np.float32)[np.newaxis, :], sr)[0:1]


def compute_mel_spectrogram_batch(audio: np.ndarray, sr: int = 48000) -> np.ndarray:
    """audio f32[B, n] (or int16[B, n] PCM windows) -> f32 (B, 1, n_mels, T)."""
    lib = _lib.load()
    cfg = _mel_cfg()
    cfg.sr = int(sr)
    audio = np.ascontiguousarray(audio)
    if audio.ndim != 2:
        raise ValueError("audio must be [B, n_samples]")
    B, n = audio.shape
    T = 1 + n // cfg.hop
    shape = (B, 1, T, cfg.n_mels) if cfg.transpose else (B, 1, cfg.n_mels, T)
    out = np.empty(shape, dtype=np.float32)
    is_i16 = audio.dtype == np.int16
    if not is_i16:
        audio = np.ascontiguousarray(audio, dtype=np.float32)
    _lib.check(lib.am_mel_batch(_lib.ptr(audio), int(is_i16), B, n, C.byref(cfg), _lib.ptr(out)))
    return out


class MelPlan:
    """Device-resident tables (window, twiddles, mel CSR) for am_mel_batch_dev / embed_tracks_dev."""

    def __init__(self, cfg: Optional[_lib.MelCfg] = None):
        self._lib = _lib.load()
        self.cfg = cfg if cfg is not None else _mel_cfg(transpose=False)
        h = C.c_void_p()
        _lib.check(self._lib.am_mel_plan_create(C.byref(self.cfg), C.byref(h)))
        self.handle = h

    def mel_dev(self, pcm_ptr: int, is_i16: bool, B: int, n_samples: int, out_ptr: int, stream: int = 0) -> None:
        _lib.check(self._lib.am_mel_batch_dev(self.handle, C.c_void_p(pcm_ptr), 1 if is_i16 else 0, int(B),
                                              int(n_samples), C.c_void_p(out_ptr), C.c_void_p(stream)))

    def close(self):
        if getattr(self, "handle", None):
            self._lib.am_mel_plan_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------------- session
class B200Session:
    """Duck type of the onnxruntime.InferenceSession the reference keeps in ``_audio_session``
    (tasks/clap_analyzer.py:111-116): ``run(None, {'mel_spectrogram': mel}) -> [emb]``.
    Unlike the exported student graph (fixed batch 1, student_onnx_model.py:611-626) it
    accepts any leading batch dimension."""

    def __init__(self, blob: Optional[bytes] = None, path: Optional[str] = None):
        """`path`: the model file the reference deploys (ONNX, tensor data inline or in `<name>.onnx.data`
        next to it) or an AMW1 blob; `blob`: the same as bytes (ONNX without external data, or AMW1)."""
        lib = _lib.load()
        self._lib = lib
        self._h = None
        h = C.c_void_p()
        if path is not None:
            _lib.check(lib.am_clap_load(os.fsencode(path), C.byref(h)))
        elif blob is not None:
            buf = (C.c_char * len(blob)).from_buffer_copy(blob)
            _lib.check(lib.am_clap_load_mem(C.cast(buf, C.c_void_p), len(blob), C.byref(h)))
        else:
            raise ValueError("B200Session needs a model path or a model blob")
        self._h = h
        self.embedding_dim = int(lib.am_clap_embedding_dim(h))
        self.n_mels = int(lib.am_clap_n_mels(h))
        self._mu = threading.RLock()
        self._streaming = False

    @classmethod
    def from_file(cls, path: str) -> "B200Session":
        return cls(path=path)

    @classmethod
    def from_state_dict(cls, state_dict, cfg: StudentConfig = StudentConfig()) -> "B200Session":
        return cls(export_blob(state_dict, cfg))

    def get_providers(self):
        return ["B200ExecutionProvider"]

    def get_inputs(self):
        return [SimpleNamespace(name="mel_spectrogram", shape=[None, 1, self.n_mels, None])]

    def flops_per_segment(self, T: int = 1001) -> float:
        return float(self._lib.am_clap_flops_per_segment(self._h, int(T)))

    def flops_split(self, T: int = 1001):
        """(flops per window in the standalone GEMM kernel, flops per window in the fused block kernel,
        algorithmic HBM bytes per window of the fused blocks)."""
        g, f, fb = C.c_double(0), C.c_double(0), C.c_double(0)
        _lib.check(self._lib.am_clap_flops_split(self._h, int(T), C.byref(g), C.byref(f), C.byref(fb)))
        return float(g.value), float(f.value), float(fb.value)

    def run(self, output_names, input_feed):
        mel = input_feed["mel_spectrogram"]
        mel = np.ascontiguousarray(mel, dtype=np.float32)
        if mel.ndim != 4 or mel.shape[1] != 1 or mel.shape[2] != self.n_mels:
            raise ValueError(f"mel_spectrogram must be (B,1,{self.n_mels},T), got {mel.shape}")
        B, _, _, T = mel.shape
        out = np.empty((B, self.embedding_dim), dtype=np.float32)
        with self._mu:
            if self._streaming:
                raise RuntimeError("B200Session.run: the session is owned by an embed_tracks_stream in progress")
            _lib.check(self._lib.am_clap_embed(self._h, _lib.ptr(mel), B, T, _lib.ptr(out)))
        return [out]

    def embed_tracks(self, pcm16: np.ndarray, seg_offsets: np.ndarray) -> np.ndarray:
        """Fused path: int16[S, n] windows + int32[n_tracks+1] offsets -> f32[n_tracks, dim]."""
        pcm16 = np.ascontiguousarray(pcm16, dtype=np.int16)
        seg_offsets = np.ascontiguousarray(seg_offsets, dtype=np.int32)
        n_tracks = len(seg_offsets) - 1
        if pcm16.ndim != 2 or n_tracks < 0 or (n_tracks and int(seg_offsets[-1]) != pcm16.shape[0]):
            raise ValueError("pcm16 must be [S, n_samples] and seg_offsets[-1] == S")
        out = np.empty((max(n_tracks, 0), self.embedding_dim), dtype=np.float32)
        if n_tracks <= 0:
            return out
        cfg = _mel_cfg(transpose=False)
        with self._mu:
            if self._streaming:
                raise RuntimeError("B200Session.embed_tracks: the session is owned by an embed_tracks_stream in progress")
            _lib.check(self._lib.am_clap_embed_tracks(self._h, C.byref(cfg), _lib.ptr(pcm16), pcm16.shape[1],
                                                      _lib.ptr(seg_offsets), n_tracks, _lib.ptr(out)))
        return out

    def embed_tracks_stream(self, batches):
        """Pipelined bulk analysis: `batches` yields (pcm16 int16[S, n], seg_offsets int32[n_tracks+1]); yields
        f32[n_tracks, dim] per batch, in order.  Batch i+1 is submitted before batch i is collected, so its H2D
        copies and early blocks run under batch i's late blocks / head / D2H (am_clap_embed_tracks_submit).
        The stream OWNS the session until it is exhausted or closed: other threads block on the session lock;
        a blocking call (run / embed_tracks) from the consuming thread inside the loop raises instead of deadlocking.
        Closing (or dropping) the generator drains what is still in flight."""
        cfg = _mel_cfg(transpose=False)
        pending = []  # (pcm16, seg_offsets, out): the inputs stay referenced until collected
        with self._mu:
            if self._streaming:
                raise RuntimeError("embed_tracks_stream: this session is already streaming")
            self._streaming = True
            try:
                for pcm16, seg_offsets in batches:
                    pcm16 = np.ascontiguousarray(pcm16, dtype=np.int16)
                    seg_offsets = np.ascontiguousarray(seg_offsets, dtype=np.int32)
                    n_tracks = len(seg_offsets) - 1
                    if pcm16.ndim != 2 or n_tracks < 0 or (n_tracks and int(seg_offsets[-1]) != pcm16.shape[0]):
                        raise ValueError("pcm16 must be [S, n_samples] and seg_offsets[-1] == S")
                    out = np.empty((max(n_tracks, 0), self.embedding_dim), dtype=np.float32)
                    if len(pending) == 2:
                        _lib.check(self._lib.am_clap_embed_tracks_collect(self._h))
                        yield pending.pop(0)[2]
                    _lib.check(self._lib.am_clap_embed_tracks_submit(self._h, C.byref(cfg), _lib.ptr(pcm16), pcm16.shape[1],
                                                                     _lib.ptr(seg_offsets), n_tracks, _lib.ptr(out)))
                    pending.append((pcm16, seg_offsets, out))
                while pending:
                    _lib.check(self._lib.am_clap_embed_tracks_collect(self._h))
                    yield pending.pop(0)[2]
            finally:
                while pending:  # an exception (or an abandoned generator): drain what is still in flight
                    try:
                        self._lib.am_clap_embed_tracks_collect(self._h)
                    except Exception:
                        pass
                    pending.pop(0)
                self._streaming = False

    def embed_tracks_dev(self, plan: "MelPlan", pcm_ptr: int, n_samples: int, offsets_ptr: int, n_tracks: int,
                         n_segments: int, out_ptr: int, stream: int = 0) -> None:
        """Device-pointer variant (no copies, no synchronisation): int16[S, n] windows and int32 offsets
        already in HBM -> f32[n_tracks, dim] in HBM, enqueued on ``stream`` (a cudaStream_t)."""
        _lib.check(self._lib.am_clap_embed_tracks_dev(self._h, plan.handle, C.c_void_p(pcm_ptr), int(n_samples),
                                                      C.c_void_p(offsets_ptr), int(n_tracks), int(n_segments),
                                                      C.c_void_p(out_ptr), C.c_void_p(stream)))

    def release_workspace(self) -> None:
        """Frees activation / staging buffers (weights stay): the cleanup of the reference's OOM retry."""
        with self._mu:
            _lib.check(self._lib.am_clap_release_workspace(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.am_clap_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200TextSession:
    """Duck type of the onnxruntime.InferenceSession the reference keeps in ``_text_session``
    (tasks/clap_analyzer.py:168-240): ``run(None, {'input_ids': i64[B, T], 'attention_mask': i64[B, T]}) ->
    [f32[B, dim]]``, plus ``get_inputs`` and ``get_providers``.  `path` is the deployed clap_text_model.onnx (tensor
    data inline or in `<name>.onnx.data`), `blob` the same bytes with inline data; both are lowered by am_text_load.
    Calls from several threads are serialised on the session's lock."""

    def __init__(self, blob: Optional[bytes] = None, path: Optional[str] = None):
        lib = _lib.load()
        self._lib = lib
        self._h = None
        h = C.c_void_p()
        if path is not None:
            _lib.check(lib.am_text_load(os.fsencode(path), C.byref(h)))
        elif blob is not None:
            buf = (C.c_char * len(blob)).from_buffer_copy(blob)
            _lib.check(lib.am_text_load_mem(C.cast(buf, C.c_void_p), len(blob), C.byref(h)))
        else:
            raise ValueError("B200TextSession needs a model path or a model blob")
        self._h = h
        self.embedding_dim = int(lib.am_text_embedding_dim(h))
        self._mu = threading.Lock()

    @staticmethod
    def describe(path: str) -> str:
        """The program am_text_load would run for `path` (needs no GPU)."""
        lib = _lib.load()
        buf = C.create_string_buffer(1 << 16)
        _lib.check(min(0, lib.am_text_describe_file(os.fsencode(path), buf, len(buf))))
        return buf.value.decode()

    def get_providers(self):
        return ["B200ExecutionProvider"]

    def get_inputs(self):
        return [SimpleNamespace(name="input_ids", shape=["batch_size", "sequence_length"], type="tensor(int64)"),
                SimpleNamespace(name="attention_mask", shape=["batch_size", "sequence_length"], type="tensor(int64)")]

    def run(self, output_names, input_feed):
        ids = np.ascontiguousarray(input_feed["input_ids"], dtype=np.int64)
        mask = np.ascontiguousarray(input_feed["attention_mask"], dtype=np.int64)
        if ids.ndim != 2 or mask.shape != ids.shape:
            raise ValueError(f"input_ids and attention_mask must both be [B, T], got {ids.shape} and {mask.shape}")
        B, T = ids.shape
        out = np.empty((B, self.embedding_dim), dtype=np.float32)
        if B == 0:
            return [out]
        with self._mu:
            if self._h is None:
                raise RuntimeError("B200TextSession.run: the session is closed")
            _lib.check(self._lib.am_text_embed(self._h, _lib.ptr(ids), _lib.ptr(mask), B, T, _lib.ptr(out)))
        return [out]

    def release_workspace(self) -> None:
        with self._mu:
            _lib.check(self._lib.am_text_release_workspace(self._h))

    def close(self):
        with self._mu:
            if getattr(self, "_h", None):
                self._lib.am_text_free(self._h)
                self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _weights_path() -> str:
    """The reference's own model file, config.CLAP_AUDIO_MODEL_PATH (config.py:375; an ONNX ModelProto, read and
    lowered by am_clap_load); CLAP_B200_WEIGHTS_PATH, when set, overrides it (an AMW1 blob or another ONNX file)."""
    p = getattr(config, "CLAP_B200_WEIGHTS_PATH", "") or os.environ.get("CLAP_B200_WEIGHTS_PATH", "")
    if p:
        return p
    return getattr(config, "CLAP_AUDIO_MODEL_PATH", "") or ""


def _load_audio_model() -> bool:
    """Lazy singleton load (reference: _load_audio_model, :47-165)."""
    global _audio_session
    with _session_lock:
        if _audio_session is not None:
            return True
        if not getattr(config, "CLAP_ENABLED", True):
            logger.info("CLAP is disabled in config. Skipping audio model load.")
            return False
        path = _weights_path()
        if not path or not os.path.exists(path):
            logger.error(f"CLAP audio model not found at {path!r}")
            return False
        try:
            _audio_session = B200Session.from_file(path)
            logger.info(f"CLAP audio model loaded on the GPU from {path}")
            return True
        except Exception as e:
            logger.error(f"Failed to load CLAP audio model on the GPU: {e}")
            _audio_session = None
            return False


def set_clap_audio_session(session: Optional[B200Session]) -> None:
    """Install an already-built session as the module singleton (tests, bench, distributed workers)."""
    global _audio_session
    with _session_lock:
        _audio_session = session


def initialize_clap_audio_model() -> bool:
    return _load_audio_model()


def get_clap_audio_model():
    if _audio_session is None and not _load_audio_model():
        raise RuntimeError("Failed to initialize CLAP audio model")
    return _audio_session


def unload_clap_audio_only() -> bool:
    global _audio_session
    with _session_lock:
        if _audio_session is None:
            return False
        try:
            _audio_session.close()
        finally:
            _audio_session = None
        return True


def unload_clap_model() -> bool:
    return unload_clap_audio_only()


def is_clap_audio_loaded() -> bool:
    return _audio_session is not None


def is_clap_model_loaded() -> bool:
    return _audio_session is not None


def is_clap_available() -> bool:
    p = _weights_path()
    return bool(getattr(config, "CLAP_ENABLED", True) and p and os.path.exists(p) and os.path.exists(_lib.LIB_PATH))


# --------------------------------------------------------------------------- pre-processing
def pcm_to_segments(audio: np.ndarray) -> np.ndarray:
    """clip -> *32767 -> int16 (truncation) -> 10 s / 5 s-hop windows incl. the tail window
    (tasks/clap_analyzer.py:502-523).  f32[L] -> int16[S, 480000] (value q stands for q/32767)."""
    lib = _lib.load()
    audio = np.ascontiguousarray(audio, dtype=np.float32).reshape(-1)
    n = C.c_int(0)
    _lib.check(lib.am_pcm_to_segments(_lib.ptr(audio), audio.size, None, 0, C.byref(n)))
    seg = np.empty((n.value, SEGMENT_LENGTH), dtype=np.int16)
    _lib.check(lib.am_pcm_to_segments(_lib.ptr(audio), audio.size, _lib.ptr(seg), n.value, C.byref(n)))
    return seg


def decode_wav(audio_path: str, max_seconds: Optional[float] = None) -> Tuple[np.ndarray, int]:
    """RIFF/WAVE -> (mono float32 at the file's own rate, sample rate) through the library's host decoder
    (am_wav_decode_mono: PCM 8/16/24/32, float 32/64, any channels; channel mean like librosa.to_mono).
    ctypes releases the GIL during the call, so a thread pool decodes files in parallel."""
    lib = _lib.load()
    sr, ch, frames, bits = C.c_int(0), C.c_int(0), C.c_int64(0), C.c_int(0)
    p = os.fsencode(audio_path)
    _lib.check(lib.am_wav_info(p, C.byref(sr), C.byref(ch), C.byref(frames), C.byref(bits)))
    limit = -1 if max_seconds is None else int(float(max_seconds) * sr.value)
    n = int(frames.value) if limit < 0 else min(int(frames.value), limit)
    out = np.empty((n,), dtype=np.float32)
    got = C.c_int64(0)
    _lib.check(lib.am_wav_decode_mono(p, limit, _lib.ptr(out), n, C.byref(got), C.byref(sr)))
    return out[: int(got.value)], int(sr.value)


def resample(x: np.ndarray, sr_in: int, sr_out: int = SAMPLE_RATE) -> np.ndarray:
    """Rational polyphase resampling on the GPU (am_resample: scipy.signal.resample_poly's algorithm).  The reference
    goes through librosa's soxr_hq here (analysis.py:181), which is not installable: parity pinned against scipy only."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if sr_in == sr_out or x.size == 0:
        return x
    lib = _lib.load()
    g = int(np.gcd(int(sr_in), int(sr_out)))
    cap = (x.size * (sr_out // g) + (sr_in // g) - 1) // (sr_in // g)
    y = np.empty((cap,), dtype=np.float32)
    n = C.c_int64(0)
    _lib.check(lib.am_resample(_lib.ptr(x), x.size, int(sr_in), int(sr_out), _lib.ptr(y), cap, C.byref(n)))
    return y[: int(n.value)]


def load_audio(audio_path: str, target_sr: int = SAMPLE_RATE) -> Tuple[Optional[np.ndarray], int]:
    """What robust_load_audio_with_fallback(path, target_sr) returns (tasks/analysis.py:170-250), for WAV files:
    mono float32 at target_sr, at most AUDIO_LOAD_TIMEOUT seconds of the file (librosa's `duration`).  WAV of any
    PCM / float encoding and rate is decoded by the library (host) and resampled on the GPU; any other container is
    delegated to the reference's own loader when it is importable (pydub / ffmpeg: decode stays on the host)."""
    try:
        x, sr = decode_wav(audio_path, float(getattr(config, "AUDIO_LOAD_TIMEOUT", 600)))
        if x.size:  # an empty signal is a failure of the direct load: fall through (analysis.py:184-185)
            return (x if sr == target_sr else resample(x, sr, target_sr)), target_sr
    except _lib.B200Error as e:
        if e.code not in (_lib.AM_ERR_IO, _lib.AM_ERR_INVALID):
            raise
    try:
        from tasks.analysis import robust_load_audio_with_fallback  # type: ignore
    except Exception as e:
        raise RuntimeError(f"cannot decode {audio_path!r}: not a readable WAV file and the reference loader is "
                           f"unavailable ({e})")
    return robust_load_audio_with_fallback(audio_path, target_sr=target_sr)


# --------------------------------------------------------------------------- analysis
def embed_pcm16_windows(pcm16: np.ndarray, seg_offsets: Sequence[int]) -> np.ndarray:
    return get_clap_audio_model().embed_tracks(pcm16, np.asarray(seg_offsets, dtype=np.int32))


def analyze_audio_batch(waveforms: Sequence[np.ndarray]) -> List[Tuple[Optional[np.ndarray], float, int]]:
    """Many decoded tracks (float32, 48 kHz mono) in ONE fused device pass.  Each result is the
    (embedding, duration_sec, num_segments) triple analyze_audio_file returns."""
    segs, offs, durs = [], [0], []
    for w in waveforms:
        w = np.asarray(w, dtype=np.float32).reshape(-1)
        s = pcm_to_segments(w)
        segs.append(s)
        offs.append(offs[-1] + len(s))
        durs.append(len(w) / SAMPLE_RATE)
    pcm = np.concatenate(segs, axis=0) if segs else np.zeros((0, SEGMENT_LENGTH), np.int16)
    embs = embed_pcm16_windows(pcm, offs)
    return [(embs[i], durs[i], offs[i + 1] - offs[i]) for i in range(len(durs))]


def is_memory_error(error: Exception) -> bool:
    """tasks/memory_utils.py:375-382: the strings the reference's OOM detection looks for."""
    s = str(error)
    return "Failed to allocate memory" in s or "BFCArena" in s or "OOM" in s or "out of memory" in s.lower()


def handle_memory_error(error: Exception, context: str, cleanup_func=None, retry_func=None):
    """Same policy as tasks/memory_utils.py:327-426 (handle_onnx_memory_error) without the CPU fallback this
    library does not have: not a memory error -> re-raise; else clean up, retry ONCE, re-raise a failing retry."""
    if not is_memory_error(error):
        raise error
    logger.warning(f"GPU memory allocation error detected in {context}: {error}")
    if cleanup_func:
        try:
            cleanup_func()
        except Exception as cleanup_error:
            logger.error(f"Cleanup failed for {context}: {cleanup_error}")
    if retry_func is None:
        raise error
    logger.info(f"Retrying {context} after cleanup...")
    return retry_func()


def analyze_audio_files(paths: Sequence[str], batch_tracks: int = 256, workers: Optional[int] = None, stats: Optional[dict] = None):
    """Bulk analysis FROM FILES: a thread pool decodes (and, off 48 kHz, resamples) the files of the next batch straight
    into a reusable (pinned, when torch is importable) batch buffer while the GPU embeds the previous batches
    (B200Session.embed_tracks_stream, two batches in flight).  Yields one (embedding | None, duration_sec, num_segments)
    per path, in order -- analyze_audio_file's triple; a file that cannot be decoded yields (None, 0, 0) like the
    reference.  `stats`, when a dict, receives the seconds spent in decode (summed over the pool's threads) and in
    the whole call."""
    import time
    from concurrent.futures import ThreadPoolExecutor

    session = get_clap_audio_model()
    workers = workers or min(32, (os.cpu_count() or 4))
    t_all = time.perf_counter()
    decode_s = [0.0]
    lock = threading.Lock()
    lib = _lib.load()
    max_s = float(getattr(config, "AUDIO_LOAD_TIMEOUT", 600))

    def probe(path):
        """(n_windows, duration) of a 48 kHz WAV from its header alone, or (-1, 0) when the file needs the slow path"""
        n, dur = C.c_int(0), C.c_double(0.0)
        st = lib.am_wav_to_segments(os.fsencode(path), max_s, None, 0, C.byref(n), C.byref(dur))
        return (n.value, float(dur.value)) if st == _lib.AM_OK else (-1, 0.0)

    def slow_decode(path):
        try:  # another rate (GPU resample) or another container (the reference's loader)
            x, _sr = load_audio(path, SAMPLE_RATE)
            return (pcm_to_segments(x), len(x) / SAMPLE_RATE) if x is not None and x.size else (None, 0.0)
        except Exception as e:
            logger.error(f"CLAP analysis failed for {path}: {e}")
            return None, 0.0

    def timed(fn, *a):
        t0 = time.perf_counter()
        try:
            return fn(*a)
        finally:
            with lock:
                decode_s[0] += time.perf_counter() - t0

    def fill(path, dst):
        n = C.c_int(0)
        st = lib.am_wav_to_segments(os.fsencode(path), max_s, _lib.ptr(dst), dst.shape[0], C.byref(n), None)
        return st == _lib.AM_OK

    ring: list = []   # batch buffers, reused round robin: at most two batches are in flight + one being filled

    def buffer_for(n_seg, slot):
        while len(ring) <= slot:
            ring.append(None)
        if ring[slot] is None or ring[slot].shape[0] < n_seg:
            try:
                import torch
                ring[slot] = torch.empty((max(n_seg, batch_tracks), SEGMENT_LENGTH), dtype=torch.int16,
                                         pin_memory=torch.cuda.is_available()).numpy()
            except Exception:
                ring[slot] = np.empty((max(n_seg, batch_tracks), SEGMENT_LENGTH), dtype=np.int16)
        return ring[slot][:n_seg]

    meta: list = []

    def batches(pool):
        for bi, b0 in enumerate(range(0, len(paths), batch_tracks)):
            group = list(paths[b0:b0 + batch_tracks])
            info = list(pool.map(lambda p: timed(probe, p), group))
            slow = {i: f for i, f in ((i, pool.submit(timed, slow_decode, group[i])) for i, (n, _) in enumerate(info) if n < 0)}
            slow_res = {i: f.result() for i, f in slow.items()}
            counts = [n if n >= 0 else (0 if slow_res[i][0] is None else len(slow_res[i][0])) for i, (n, _) in enumerate(info)]
            offs = np.zeros(len(group) + 1, dtype=np.int32)
            offs[1:] = np.cumsum(counts)
            pcm = buffer_for(int(offs[-1]), bi % 3)
            jobs = []
            for i, (n, _) in enumerate(info):
                dst = pcm[offs[i]:offs[i + 1]]
                if n >= 0:
                    jobs.append((i, pool.submit(timed, fill, group[i], dst)))
                elif counts[i]:
                    dst[...] = slow_res[i][0]
            ok = {i: f.result() for i, f in jobs}
            decoded = []
            for i, (n, dur) in enumerate(info):
                if n >= 0:
                    decoded.append((counts[i], dur) if ok[i] else (None, 0.0))
                else:
                    decoded.append((counts[i], slow_res[i][1]) if slow_res[i][0] is not None else (None, 0.0))
            meta.append(decoded)
            yield pcm, offs

    with ThreadPoolExecutor(max_workers=workers) as pool:
        for bi, embs in enumerate(session.embed_tracks_stream(batches(pool))):
            for ti, (nseg, dur) in enumerate(meta[bi]):
                yield (None, 0, 0) if nseg is None else (embs[ti], dur, nseg)
    if stats is not None:
        stats["decode_thread_seconds"] = decode_s[0]
        stats["wall_seconds"] = time.perf_counter() - t_all
        stats["workers"] = workers


def analyze_audio_file(audio_path: str) -> Tuple[Optional[np.ndarray], float, int]:
    """Same contract as the reference: (512-d float32 unit vector, duration_sec, num_segments),
    or (None, 0, 0) when CLAP is disabled or anything fails.  Never raises."""
    if not getattr(config, "CLAP_ENABLED", True):
        return None, 0, 0
    try:
        session = get_clap_audio_model()
        audio_data, _sr = load_audio(audio_path, SAMPLE_RATE)
        if audio_data is None or audio_data.size == 0:
            logger.warning(f"Could not load audio for CLAP analysis: {audio_path}")
            return None, 0, 0
        try:
            (emb, dur, nseg), = analyze_audio_batch([audio_data])
        except Exception as e:  # reference :536-549: memory errors get one cleanup + retry
            (emb, dur, nseg), = handle_memory_error(
                e, f"CLAP analysis of {os.path.basename(audio_path)}",
                cleanup_func=session.release_workspace, retry_func=lambda: analyze_audio_batch([audio_data]))
        logger.info(f"CLAP: Processing {nseg} segments ({dur:.1f}s audio)")
        return emb, dur, nseg
    except Exception as e:  # reference: log, clean up, (None, 0, 0)
        logger.error(f"CLAP analysis failed for {audio_path}: {e}")
        return None, 0, 0
