"""am_track_features on the GPU against the float64 restatement of librosa 0.11.0 (oracle/track_features.py): seeded
music-like sets (drum and click loops with noise, chords, detuned tones; 1 s to 600 s; ragged batches; 16 and 22.05
kHz), stage by stage, with every discrete decision checked only where its margin clears a floor measured in the same
run -- a set whose margin does not clear it fails."""
import types

import numpy as np
import pytest

from oracle import track_features as otf

pytestmark = pytest.mark.gpu

ONSET_ATOL = 2e-3        # dB
TEMPOGRAM_ATOL = 1e-6
RMS_RTOL = 1e-5
CHROMA_ATOL = 1e-4
THRESHOLD_RTOL = 1e-4

# (kind, seconds, seed) per batch; every batch is ragged
SETS = {
    16000: [("drums", 30.0, 0), ("chord", 7.3, 1), ("detuned", 4.0, 2), ("clicks", 12.0, 3), ("drums", 1.0, 4),
            ("chord", 61.7, 5)],
    22050: [("drums", 20.0, 6), ("chord", 3.1, 7), ("detuned", 9.0, 8), ("clicks", 15.5, 9)],
}
LONG = ("drums", 600.0, 10)


def _tf():
    from audiomuse_ai_b200 import track_features as tf
    return tf


def _check_set(ys, sr, tag):
    tf = _tf()
    got = tf.compute(ys, sr, intermediates=True)
    for i, y in enumerate(ys):
        o = otf.track_features(y, sr)
        name = f"{tag}[{i}] ({len(y) / sr:.1f} s, sr {sr})"
        T = o["T"]
        # onset envelope
        env = got["onset_env"][i]
        assert env.shape == (T,)
        d_env = float(np.max(np.abs(env.astype(np.float64) - o["onset_env"])))
        # tempogram: the device's envelope through the restatement's tempogram
        tg_ref = otf.tempogram_mean(env, sr) if env.any() else np.zeros(len(got["tempogram"][i]))
        d_tg = float(np.max(np.abs(got["tempogram"][i] - tg_ref)))
        # tempo: the decision on the oracle's scores, floor from the observed score difference
        if o["onset_env"].any():
            s_gpu, s_ref = otf.tempo_scores(got["tempogram"][i], sr), o["tempo_score"]
            fin = np.isfinite(s_ref)
            best = float(np.max(s_ref[fin]))
            t_floor = max(1e-12, 10 * float(np.max(np.abs(s_gpu[fin] - s_ref[fin]))) / abs(best))
        else:
            t_floor = 0.0
        # rms / energy
        rms = got["rms"][i]
        d_rms = float(np.max(np.abs(rms.astype(np.float64) - o["rms"]) / np.maximum(np.abs(o["rms"]), 1e-30)))
        # chroma: against the oracle's chroma under the oracle's tuning
        ch = got["chroma"][i]
        d_ch = float(np.max(np.abs(ch.astype(np.float64) - o["chroma"])))
        maj_g, mnr_g = otf.key_correlations(np.mean(ch, axis=1))
        k_floor = 10 * float(max(np.max(np.abs(maj_g - o["major_corr"])), np.max(np.abs(mnr_g - o["minor_corr"]))))
        d_thr = abs(float(got["threshold"][i]) - float(o["threshold"])) / max(float(o["threshold"]), 1e-30)
        print(f"{name}: onset {d_env:.2e} dB, tempogram {d_tg:.2e}, tempo {got['tempo'][i]} vs {o['tempo']} "
              f"margin {o['tempo_margin']:.3e} floor {t_floor:.3e}, rms rel {d_rms:.2e}, tuning {got['tuning'][i]} vs "
              f"{o['tuning']} gap {o['tuning_gap']} fragile {o['tuning_fragile']}, threshold rel {d_thr:.2e}, "
              f"chroma {d_ch:.2e}, key {o['key']} {o['scale']} margin {o['key_margin']:.3e} floor {k_floor:.3e}")
        assert d_env <= ONSET_ATOL, name
        assert d_tg <= TEMPOGRAM_ATOL, name
        assert o["tempo_margin"] > t_floor, f"{name}: tempo margin below its floor"
        assert got["tempo"][i] == o["tempo"], name
        assert d_rms <= RMS_RTOL, name
        np.testing.assert_allclose(np.mean(rms), o["energy"], rtol=RMS_RTOL, err_msg=name)
        assert o["tuning_gap"] > o["tuning_fragile"], f"{name}: tuning gap does not clear the fragile peaks"
        assert got["tuning"][i] == o["tuning"], name
        assert d_thr <= THRESHOLD_RTOL, name
        assert ch.shape == (12, T) and ch.dtype == np.float32
        assert d_ch <= CHROMA_ATOL, name
        assert o["key_margin"] > k_floor, f"{name}: key margin below its floor"
        key, scale = tf.key_scale(np.mean(ch, axis=1))
        assert (key, scale) == (o["key"], o["scale"]), name
    return got


@pytest.mark.parametrize("sr", sorted(SETS))
def test_ragged_batch_against_oracle(sr):
    ys = [otf.synth_track(k, s, sr, seed) for k, s, seed in SETS[sr]]
    _check_set(ys, sr, f"set{sr}")


def test_ten_minute_track_against_oracle():
    ys = [otf.synth_track(*LONG[:2], 16000, LONG[2]), otf.synth_track("chord", 2.0, 16000, 11)]
    _check_set(ys, 16000, "long")


def test_silence_and_tiny_tracks():
    tf = _tf()
    r = tf.compute([np.zeros(16000, np.float32), np.zeros(1, np.float32), np.full(700, 0.25, np.float32)],
                   16000, intermediates=True)
    for i in range(2):
        assert r["tempo"][i] == 0.0 and float(np.mean(r["rms"][i])) == 0.0 and r["tuning"][i] == 0.0
        assert not r["chroma"][i].any() and not r["onset_env"][i].any()
    assert r["rms"][1].shape == (1, 1) and r["chroma"][1].shape == (12, 1)
    o = otf.track_features(np.full(700, 0.25, np.float32))
    np.testing.assert_allclose(r["rms"][2][0], o["rms"][0], rtol=RMS_RTOL)
    f = tf.track_features([np.zeros(16000, np.float32)])[0]
    assert f["tempo"] == 0.0 and f["energy"] == 0.0 and f["tuning"] == 0.0


def test_two_calls_bit_identical_and_batch_independent():
    tf = _tf()
    ys = [otf.synth_track(k, s, 16000, seed) for k, s, seed in SETS[16000]]
    a = tf.compute(ys, 16000, intermediates=True)
    b = tf.compute(ys, 16000, intermediates=True)
    for key in a:
        for x, y in zip(a[key], b[key]):
            assert np.array_equal(np.asarray(x), np.asarray(y)), key
    for i in (0, 2, 5):
        alone = tf.compute([ys[i]], 16000, intermediates=True)
        for key in a:
            assert np.array_equal(np.asarray(alone[key][0]), np.asarray(a[key][i])), (key, i)
    rev = tf.compute(ys[::-1], 16000, intermediates=True)
    for key in a:
        for x, y in zip(a[key], rev[key][::-1]):
            assert np.array_equal(np.asarray(x), np.asarray(y)), key


def test_single_flags_match_the_full_call():
    tf = _tf()
    ys = [otf.synth_track("drums", 5.0, 16000, 3), otf.synth_track("chord", 2.5, 16000, 4)]
    full = tf.compute(ys, 16000)
    for flag, keys in ((tf.TEMPO, ("tempo",)), (tf.RMS, ("rms",)), (tf.CHROMA, ("chroma", "tuning"))):
        r = tf.compute(ys, 16000, flag)
        assert set(r) == set(keys)
        for k in keys:
            for x, y in zip(r[k], full[k]):
                assert np.array_equal(np.asarray(x), np.asarray(y)), k


def test_known_answers_on_the_device():
    tf = _tf()
    clicks = []
    for k in (15, 16, 20):
        y = np.zeros(20 * 16000, np.float32)
        y[::k * 512] = 1.0
        clicks.append(y)
    assert tf.compute(clicks, 16000, tf.TEMPO)["tempo"] == [1875.0 / 15, 1875.0 / 16, 1875.0 / 20]
    t = np.arange(5 * 16000) / 16000
    for c in (-20.5, 10.5, 33.5):
        y = (0.5 * np.sin(2 * np.pi * 3520.0 * 2 ** (c / 1200) * t)).astype(np.float32)
        assert tf.compute([y], 16000, tf.CHROMA)["tuning"][0] == otf.hist_edges()[int(np.floor(c)) + 50]


def test_invalid_input_is_rejected_before_device_work():
    import ctypes as C
    from audiomuse_ai_b200 import _lib
    tf = _tf()
    lib = _lib.load()
    plan = tf._plan(16000)
    x = np.ones(1000, np.float32)
    tempo = np.zeros(2)
    for offs, xs in ((np.array([0, 0, 1000], np.int64), x), (np.array([0, 500, 1000], np.int64),
                                                             np.where(np.arange(1000) == 7, np.nan, x).astype(np.float32))):
        assert lib.am_track_features(plan, _lib.ptr(xs), _lib.ptr(offs), 2, 1, _lib.ptr(tempo), None, None, None,
                                     None, None, None, None) == _lib.AM_ERR_INVALID
    h = C.c_void_p()
    assert lib.am_track_features_plan_create(96000, C.byref(h)) == _lib.AM_ERR_INVALID


def test_existing_mel_modes_replay_their_golden():
    """The reflect (framing 0) and frame-start (framing 1) modes of the mel kernel, in both compressions and both input
    types, give the bits they gave before the zero-pad mode was added (tests/golden/mel_modes_golden.json, written by
    the library before that change)."""
    import json
    import os
    from tests.golden.make_mel_modes_golden import CASES, digest, mel_case
    with open(os.path.join(os.path.dirname(__file__), "golden", "mel_modes_golden.json")) as f:
        g = json.load(f)
    assert sorted(g) == sorted(CASES)
    for name in CASES:
        assert digest(mel_case(name)) == g[name], name


def test_zero_pad_framing_against_oracle():
    from audiomuse_ai_b200 import _lib
    import ctypes as C
    y = otf.synth_track("chord", 3.0, 16000, 12)
    cfg = _lib.MelCfg(16000, 2048, 512, 128, 0.0, 8000.0, 0, framing=2)
    T = 1 + len(y) // 512
    out = np.zeros((1, 128, T), np.float32)
    _lib.check(_lib.load().am_mel_batch(_lib.ptr(y), 0, 1, len(y), C.byref(cfg), _lib.ptr(out)))
    ref = otf.mel_db(otf.stft_power(y), 16000)
    assert np.max(np.abs(out[0] - np.maximum(ref, -100.0))) <= 2e-3


def test_reference_golden_calls_and_results():
    """tests/golden/track_features_golden.npz: what the reference's analyze_track asked of librosa and returned, with
    the restatement answering (make_track_features_golden.py).  The facade answers the same calls with the same shapes
    and dtypes, and track_features reproduces tempo / key / scale / energy where the margins clear their floors."""
    import json
    import os
    tf = _tf()
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "track_features_golden.npz"))
    meta = json.loads(str(g["meta"]))
    fake = types.ModuleType("librosa")
    lb = tf.LibrosaFacade(fake)
    for i, m in enumerate(meta):
        y = otf.synth_track(m["kind"], m["seconds"], 16000, m["seed"])
        assert [c["name"] for c in m["calls"]] == ["beat_track", "rms", "chroma_stft"]
        for c in m["calls"]:
            kw = {k: (y if k == "y" else 16000) for k in c["kwargs"]}
            fn = lb.beat.beat_track if c["name"] == "beat_track" else getattr(lb.feature, c["name"])
            out = fn(**kw)
            outs = out if isinstance(out, tuple) else (out,)
            assert [list(np.shape(o)) for o in outs] == c["shapes"], c
            assert [np.asarray(o).dtype.str for o in outs] == c["dtypes"], c
        f = tf.track_features([y])[0]
        print(f"golden {i} {m['kind']}: tempo {f['tempo']} vs {float(g[f'tempo_{i}'])} margin {m['tempo_margin']:.3e}, "
              f"tuning gap {m['tuning_gap']} fragile {m['tuning_fragile']}, key {f['key']} {f['scale']} vs "
              f"{m['key']} {m['scale']} margin {m['key_margin']:.3e}, energy {f['energy']} vs {float(g[f'energy_{i}'])}")
        assert m["tempo_margin"] > 1e-6 and m["key_margin"] > 1e-3 and m["tuning_gap"] > m["tuning_fragile"]
        assert f["tempo"] == float(g[f"tempo_{i}"])
        assert f["tuning"] == float(g[f"tuning_{i}"])
        assert (f["key"], f["scale"]) == (m["key"], m["scale"])
        np.testing.assert_allclose(float(f["energy"]), float(g[f"energy_{i}"]), rtol=RMS_RTOL)


def test_batch_larger_than_one_workspace_group():
    """20 ten-minute tracks need more than the 2 GB workspace of one group, so the call runs them in two groups; the
    first and last tracks give the same bits as alone."""
    tf = _tf()
    base = otf.synth_track("drums", 10.0, 16000, 13)
    ys = [np.tile(base, 60)[:600 * 16000 - 777 * i].copy() for i in range(20)]
    r = tf.compute(ys, 16000)
    for i in (0, 19):
        alone = tf.compute([ys[i]], 16000)
        for key in r:
            assert np.array_equal(np.asarray(alone[key][0]), np.asarray(r[key][i])), (key, i)
