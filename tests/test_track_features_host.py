"""Host checks of the track-feature path: the float64 restatement's known answers (oracle/track_features.py), its STFT
against torchaudio, the expressions the device copies from numpy, the librosa facade's plumbing with the device call
replaced, validation before any library load, and integration.apply(analysis=...)."""
import sys
import types

import numpy as np
import pytest

from oracle import track_features as otf

SR = 16000


def _clicks(k, seconds=20):
    y = np.zeros(seconds * SR, np.float32)
    y[::k * 512] = 1.0
    return y


@pytest.mark.parametrize("k", [15, 16, 20])
def test_click_trains_give_exact_tempo(k):
    o = otf.track_features(_clicks(k))
    assert o["tempo"] == 1875.0 / k
    assert o["tempo"] == 60.0 * SR / (512 * k)
    assert o["tempo_margin"] > 1e-3


def test_single_impulse_pins_onset_alignment():
    s0 = 32000
    y = np.zeros(4 * SR, np.float32)
    y[s0] = 1.0
    env = otf.onset_envelope(otf.stft_power(y), SR)
    # first frame whose window (samples 512 t - 1024 .. + 2048, Hann zero at its first sample) holds the impulse
    t1 = min(t for t in range(len(env)) if 0 < s0 - (512 * t - 1024) < 2048)
    assert t1 == 61
    # env[t] is the rise from frame t - 3 to t - 2 (lag 1 plus n_fft // (2 hop) = 2 frames of centring)
    assert int(np.argmax(env)) == t1 + 2
    assert not env[:t1 + 2].any()
    assert np.all(env[:3] == 0)


@pytest.mark.parametrize("cents", [-20.5, -0.5, 0.5, 10.5, 33.5, 49.5])
def test_tone_at_bin_centre_gives_its_tuning(cents):
    t = np.arange(5 * SR) / SR
    y = (0.5 * np.sin(2 * np.pi * 3520.0 * 2 ** (cents / 1200) * t)).astype(np.float32)
    o = otf.track_features(y)
    assert o["tuning"] == otf.hist_edges()[int(np.floor(cents)) + 50]
    assert abs(o["tuning"] - np.floor(cents) / 100) < 1e-12
    assert o["tuning_gap"] > o["tuning_fragile"]


def _triad(notes_hz, seconds=10):
    t = np.arange(seconds * SR) / SR
    return sum(0.3 * np.sin(2 * np.pi * f * t) for f in notes_hz).astype(np.float32)


def test_major_profiles_are_relative_minor_profiles():
    for i in range(12):
        assert np.array_equal(np.roll(otf.MAJOR, i), np.roll(otf.MINOR, i + 9))
    maj, mnr = otf.key_correlations(np.random.default_rng(0).random(12).astype(np.float32))
    assert np.array_equal(maj, np.roll(mnr, -9))


def test_triads_give_key_and_scale():
    """analysis.py:360 compares the best major and best minor correlation with a strict `>`; they are always equal
    (above), so the reference answers the relative minor of the best major key: a C-major triad gives A minor."""
    o = otf.track_features(_triad([261.63, 329.63, 392.0]))
    assert (o["key"], o["scale"]) == ("A", "minor")
    assert otf.KEYS[int(np.argmax(o["major_corr"]))] == "C" and o["key_margin"] > 1e-3
    o = otf.track_features(_triad([220.0, 261.63, 329.63]))
    assert o["scale"] == "minor"
    assert o["key"] == otf.KEYS[(int(np.argmax(o["major_corr"])) + 9) % 12]
    from audiomuse_ai_b200 import track_features as tf
    assert tf.key_scale(o["chroma_mean"]) == (o["key"], o["scale"])


def test_rms_closed_forms_with_zero_padded_edges():
    n, c = 5000, 0.25
    r = otf.rms(np.full(n, c, np.float32))[0]
    assert r.shape == (1 + n // 512,)
    for t in range(len(r)):
        count = min(n, 512 * t + 1024) - max(0, 512 * t - 1024)
        assert abs(r[t] - c * np.sqrt(count / 2048)) <= 1e-7
    f = SR * 64 / 2048                      # 64 whole cycles per frame
    y = (0.5 * np.sin(2 * np.pi * f * np.arange(3 * SR) / SR)).astype(np.float32)
    r = otf.rms(y)[0]
    np.testing.assert_allclose(r[2:-3], 0.5 / np.sqrt(2), rtol=1e-6)
    assert r[0] < r[1] < r[2]


def test_silence_gives_zero_tempo_energy_tuning():
    o = otf.track_features(np.zeros(3 * SR, np.float32))
    assert o["tempo"] == 0.0 and o["energy"] == 0.0 and o["tuning"] == 0.0
    assert len(o["peaks"]["mag"]) == 0 and not o["chroma"].any()


def test_stft_matches_torchaudio_zero_padding():
    import torch
    import torchaudio
    y = otf.synth_track("chord", 2.0, SR, 1)
    S = otf.stft_power(y)
    spec = torchaudio.transforms.Spectrogram(n_fft=2048, hop_length=512, center=True, pad_mode="constant", power=2.0,
                                             window_fn=torch.hann_window)(torch.from_numpy(y).double()).numpy()
    assert spec.shape == S.shape
    assert np.max(np.abs(spec - S)) <= 1e-5 * np.max(S)


def test_device_expressions_match_numpy():
    """What csrc/track_features.cu computes in closed form instead of calling numpy."""
    edges = otf.hist_edges()
    assert all(edges[i] == i * 0.01 + -0.5 for i in range(100))
    for sr in (16000, 22050):
        kmin, kmax = otf.pip_bins(sr)
        val = 1.0 / (2048 * (1.0 / sr))
        assert [k for k in range(1025) if 150.0 <= k * val < min(4000.0, sr / 2)] == list(range(kmin, kmax))
        assert otf.tempogram_win(sr) == int(8.0 * sr) // 512
    # linear_ramp padding of the envelope: left ramp from env[0], right ramp down from env[-1]
    env = np.array([0.0, 0.0, 0.0, 1.5, 0.25, 3.0, 0.7], np.float32)
    h = 5
    pad = np.pad(env, h, mode="linear_ramp", end_values=0)
    T = len(env)
    for p in range(-h, T + h):
        if p < 0:
            want = np.float32((p + h) * (float(env[0]) / h))
        elif p >= T:
            want = np.float32((h - 1 - (p - T)) * (float(env[-1]) / h))
        else:
            want = env[p]
        assert pad[p + h] == want, p


def test_numpy_median_of_float32_is_the_float32_mean_of_the_middle_pair():
    rng = np.random.default_rng(3)
    for n in (1, 2, 7, 100, 101):
        v = rng.random(n).astype(np.float32) * 1e3
        assert otf.median_f32(v) == np.median(v) and np.median(v).dtype == np.float32


# ------------------------------------------------------------------------------------------------ facade plumbing
@pytest.fixture
def fake_compute(monkeypatch):
    from audiomuse_ai_b200 import track_features as tf
    calls = []

    def compute(audios, sr=16000, what=7, intermediates=False):
        calls.append((len(audios), len(audios[0]), sr, what))
        T = 1 + len(audios[0]) // 512
        out = {}
        if what & tf.TEMPO:
            out["tempo"] = [123.0]
        if what & tf.RMS:
            out["rms"] = [np.full((1, T), 0.5, np.float32)]
        if what & tf.CHROMA:
            out["chroma"] = [np.ones((12, T), np.float32)]
            out["tuning"] = [0.0]
        return out

    monkeypatch.setattr(tf, "compute", compute)
    return calls


class _FakeLibrosa(types.ModuleType):
    def __init__(self):
        super().__init__("librosa")
        self.calls = []
        self.beat = types.SimpleNamespace(beat_track=lambda *a, **k: self.calls.append(("beat_track", a, k)) or "orig")
        self.feature = types.SimpleNamespace(
            rms=lambda *a, **k: self.calls.append(("rms", a, k)) or "orig",
            chroma_stft=lambda *a, **k: self.calls.append(("chroma_stft", a, k)) or "orig",
            melspectrogram=lambda *a, **k: self.calls.append(("melspectrogram", a, k)) or "orig")
        self.load = lambda *a, **k: "loaded"


def test_facade_serves_the_three_calls(fake_compute):
    from audiomuse_ai_b200 import track_features as tf
    orig = _FakeLibrosa()
    lb = tf.LibrosaFacade(orig)
    y = np.zeros(16000, np.float32)
    tempo, beats = lb.beat.beat_track(y=y, sr=16000)
    assert tempo.shape == (1,) and tempo[0] == 123.0 and beats.size == 0 and beats.dtype.kind == "i"
    r = lb.feature.rms(y=y)
    assert r.shape == (1, 32) and r.dtype == np.float32
    c = lb.feature.chroma_stft(y=y, sr=16000)
    assert c.shape == (12, 32) and c.dtype == np.float32
    assert [w for *_, w in fake_compute] == [tf.TEMPO, tf.RMS, tf.CHROMA]
    assert all(n == 1 for n, *_ in fake_compute)
    assert orig.calls == []


def test_facade_forwards_everything_else(fake_compute):
    from audiomuse_ai_b200 import track_features as tf
    orig = _FakeLibrosa()
    lb = tf.LibrosaFacade(orig)
    y = np.zeros(16000, np.float32)
    assert lb.beat.beat_track(y=y, sr=16000, hop_length=256) == "orig"
    assert lb.feature.rms(y=y, frame_length=1024) == "orig"
    assert lb.feature.chroma_stft(y=y, sr=16000, n_chroma=24) == "orig"
    assert lb.feature.chroma_stft(y=y.astype(np.float64), sr=16000) == "orig"
    assert lb.feature.rms(S=np.ones((3, 3))) == "orig"
    assert lb.feature.melspectrogram(y=y, sr=16000) == "orig"
    assert lb.load("x.wav") == "loaded"
    assert [c[0] for c in orig.calls] == ["beat_track", "rms", "chroma_stft", "chroma_stft", "rms", "melspectrogram"]
    assert fake_compute == []


def test_facade_imports_librosa_lazily(fake_compute, monkeypatch):
    from audiomuse_ai_b200 import track_features as tf
    lb = tf.LibrosaFacade(None)
    fake = _FakeLibrosa()
    monkeypatch.setitem(sys.modules, "librosa", fake)
    assert lb.load("a") == "loaded"
    assert lb._orig is fake


def test_validation_happens_before_any_library_load(monkeypatch):
    from audiomuse_ai_b200 import _lib, track_features as tf

    def no_load():
        raise AssertionError("library loaded")

    monkeypatch.setattr(_lib, "load", no_load)
    good = np.zeros(1000, np.float32)
    for audios, sr in (([np.zeros(0, np.float32)], 16000), ([np.array([0, np.inf], np.float32)], 16000),
                       ([good], 96000), ([good], 4000), ([good], 16000.5), ([], 16000), ([np.zeros((2, 5))], 16000)):
        with pytest.raises(ValueError):
            tf.compute(audios, sr)
    with pytest.raises(ValueError):
        tf.track_features([good, np.array([np.nan], np.float32)])


def test_integration_apply_sets_the_facade_only_on_the_module():
    from audiomuse_ai_b200 import integration, track_features as tf
    before = sys.modules.get("librosa")
    orig = _FakeLibrosa()
    analysis = types.ModuleType("tasks.analysis")
    analysis.librosa = orig
    integration.apply(analysis=analysis)
    assert isinstance(analysis.librosa, tf.LibrosaFacade) and analysis.librosa._orig is orig
    integration.apply(analysis=analysis)   # applying twice keeps the original as the fallback
    assert analysis.librosa._orig is orig
    assert sys.modules.get("librosa") is before
