#!/usr/bin/env python
"""Goldens of the reference's analyze_track features, so that the tests need no reference checkout.

    AUDIOMUSE_REFERENCE=<checkout of AudioMuse-AI> python tests/golden/make_track_features_golden.py
    # writes tests/golden/track_features_golden.npz

Runs the reference's analyze_track (tasks/analysis.py:324-573), UNMODIFIED, on seeded 16 kHz signals
(oracle/track_features.synth_track) with these stand-ins: robust_load_audio_with_fallback returns the seeded audio,
stub ONNX sessions are passed through onnx_sessions=, and a recording fake librosa answers beat.beat_track, feature.rms
and feature.chroma_stft from the float64 restatement (oracle/track_features.py) and feature.melspectrogram from numpy.
Records per case the calls analyze_track made (name, keyword names, returned shapes and dtypes), the tempo / key /
scale / energy it returned, and the restatement's margins for the three decisions."""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import mel as omel  # noqa: E402
from oracle import track_features as otf  # noqa: E402
from tests import ref_harness as rh  # noqa: E402

GOLDEN = os.path.join(HERE, "track_features_golden.npz")
SR = 16000
# (kind, seconds, seed)
CASES = [("drums", 20.0, 21), ("chord", 9.5, 22), ("detuned", 6.0, 23), ("clicks", 15.0, 24), ("drums", 45.3, 25)]


class RecordingLibrosa(types.ModuleType):
    """The three feature calls from the restatement, melspectrogram from numpy; every call is recorded."""

    def __init__(self):
        super().__init__("librosa")
        self.calls = []
        self.beat = types.SimpleNamespace(beat_track=self._beat_track)
        self.feature = types.SimpleNamespace(rms=self._rms, chroma_stft=self._chroma_stft,
                                             melspectrogram=self._melspectrogram)

    def _record(self, name, kwargs, out):
        outs = out if isinstance(out, tuple) else (out,)
        self.calls.append({"name": name, "kwargs": sorted(kwargs),
                           "shapes": [list(np.shape(o)) for o in outs],
                           "dtypes": [np.asarray(o).dtype.str for o in outs]})
        return out

    def _beat_track(self, **kw):
        o = otf.track_features(kw["y"], kw["sr"])
        return self._record("beat_track", kw, (np.array([o["tempo"]]), np.array([], dtype=int)))

    def _rms(self, **kw):
        return self._record("rms", kw, otf.rms(kw["y"]))

    def _chroma_stft(self, **kw):
        return self._record("chroma_stft", kw, otf.track_features(kw["y"], kw["sr"])["chroma"].astype(np.float32))

    def _melspectrogram(self, **kw):
        y, n_fft, hop = kw["y"], kw["n_fft"], kw["hop_length"]
        T = 1 + (len(y) - n_fft) // hop
        idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
        spec = np.fft.rfft(omel.hann_periodic(n_fft)[None, :] * y[idx], axis=1).astype(np.complex64)
        power = (np.abs(spec) ** 2).T.astype(np.float32)
        fb = omel.mel_filterbank(kw["sr"], n_fft, kw["n_mels"], 0.0, kw["sr"] / 2.0)
        return self._record("melspectrogram", {}, fb @ power)


class StubSession:
    def __init__(self, inp, out, dim):
        self._in, self._out, self._dim = inp, out, dim

    def get_inputs(self):
        return [types.SimpleNamespace(name=self._in)]

    def get_outputs(self):
        return [types.SimpleNamespace(name=self._out)]

    def run(self, outs, feeds):
        x = next(iter(feeds.values()))
        return [np.zeros((x.shape[0], self._dim), np.float32)]


def load_analysis(fake_librosa):
    """tasks.analysis with `librosa` = fake_librosa and inert stand-ins for the modules it imports"""
    if rh.REF not in sys.path:
        sys.path.insert(0, rh.REF)
    for k in [k for k in sys.modules if k == "tasks" or k.startswith("tasks.") or k == "config"]:
        del sys.modules[k]
    import config  # noqa: F401  the reference's config.py (pure env-var defaults)

    noop = lambda *a, **k: None  # noqa: E731
    sys.modules["librosa"] = fake_librosa
    rh._stub("pydub", AudioSegment=object)
    rh._stub("onnx")
    state = types.SimpleNamespace(RuntimeException=type("RuntimeException", (Exception,), {}))
    rh._stub("onnxruntime", get_available_providers=lambda: ["CPUExecutionProvider"], InferenceSession=None,
             capi=types.SimpleNamespace(onnxruntime_pybind11_state=state))
    rh._stub("rq", get_current_job=noop, Retry=object)
    rh._stub("rq.job", Job=object)
    rh._stub("rq.exceptions", NoSuchJobError=Exception)
    rh._stub("ai", get_ai_playlist_name=noop, creative_prompt_template="")
    rh._stub("psycopg2", OperationalError=Exception)
    rh._stub("redis")
    rh._stub("redis.exceptions", TimeoutError=Exception)
    tasks_pkg = rh._stub("tasks")
    tasks_pkg.__path__ = [os.path.join(rh.REF, "tasks")]
    rh._stub("tasks.commons", score_vector=noop)
    rh._stub("tasks.voyager_manager", build_and_store_voyager_index=noop)
    rh._stub("tasks.clap_text_search", build_and_store_clap_index=noop)
    rh._stub("tasks.lyrics_manager", build_and_store_lyrics_index=noop, build_and_store_lyrics_axes_index=noop)
    rh._stub("tasks.artist_gmm_manager", build_and_store_artist_index=noop)
    rh._stub("tasks.mediaserver", get_recent_albums=noop, get_tracks_from_album=noop, download_track=noop)
    rh._stub("tasks.memory_utils", cleanup_cuda_memory=noop, cleanup_onnx_session=noop, handle_onnx_memory_error=noop,
             SessionRecycler=object, comprehensive_memory_cleanup=noop)
    return rh._load("tasks.analysis", "tasks/analysis.py")


def main():
    if not rh.available():
        sys.exit("set AUDIOMUSE_REFERENCE to a checkout of AudioMuse-AI")
    fake = RecordingLibrosa()
    analysis = load_analysis(fake)
    waveforms = {}
    analysis.robust_load_audio_with_fallback = lambda path, target_sr=16000: (waveforms[path], target_sr)
    sessions = {"embedding": StubSession("model/Placeholder", "model/dense/BiasAdd", 200),
                "prediction": StubSession("serving_default_model_Placeholder", "PartitionedCall", 50)}
    out, meta = {}, []
    for i, (kind, seconds, seed) in enumerate(CASES):
        path = f"case{i}.wav"
        waveforms[path] = otf.synth_track(kind, seconds, SR, seed)
        fake.calls.clear()
        result, _ = analysis.analyze_track(path, [f"mood{j}" for j in range(50)], {}, onnx_sessions=sessions)
        o = otf.track_features(waveforms[path], SR)
        out[f"energy_{i}"] = np.float64(result["energy"])
        out[f"tempo_{i}"] = np.float64(result["tempo"])
        out[f"tuning_{i}"] = np.float64(o["tuning"])
        meta.append({"kind": kind, "seconds": seconds, "seed": seed, "key": result["key"], "scale": result["scale"],
                     "calls": [c for c in fake.calls if c["name"] != "melspectrogram"],
                     "tempo_margin": o["tempo_margin"], "tuning_gap": o["tuning_gap"],
                     "tuning_fragile": o["tuning_fragile"], "key_margin": o["key_margin"]})
        print(kind, seconds, seed, result["tempo"], result["key"], result["scale"], result["energy"])
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
