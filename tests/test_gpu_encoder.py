"""K2/K3 parity: batched CUDA encoder vs the PyTorch-CPU fp32 oracle (cosine >= 1 - 1e-3, the
tolerance BASELINE.json's north_star states), and the whole analysis path vs the oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import mel as omel
from oracle import phinet, segments as oseg

COS_TOL = 1e-3


def _cos(a, b):
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-30))


@pytest.fixture(scope="module")
def small():
    from audiomuse_ai_b200 import clap_analyzer as ca, weights
    cfg_o = phinet.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256)
    cfg_w = weights.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256)
    model = phinet.make_random_student(3, cfg_o)
    return model, ca.B200Session.from_state_dict(model.state_dict(), cfg_w)


@pytest.fixture(scope="module")
def full():
    from audiomuse_ai_b200 import clap_analyzer as ca
    model = phinet.make_random_student(0)
    return model, ca.B200Session.from_state_dict(model.state_dict())


@pytest.mark.parametrize("T", [101, 201, 333])
def test_small_config_matches_oracle(small, T):
    model, sess = small
    mel = phinet.synthetic_mel(3, 128, T, 11).numpy()
    want = phinet.embed_segments(model, mel)
    got = sess.run(None, {"mel_spectrogram": mel})[0]
    assert got.shape == want.shape == (3, 512)
    np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-5)
    for g, w in zip(got, want):
        assert 1.0 - _cos(g, w) <= COS_TOL


def test_full_student_matches_oracle_on_10s_windows(full):
    model, sess = full
    mel = phinet.synthetic_mel(2, 128, 1001, 5).numpy()
    want = phinet.embed_segments(model, mel)
    got = sess.run(None, {"mel_spectrogram": mel})[0]
    for g, w in zip(got, want):
        assert 1.0 - _cos(g, w) <= COS_TOL
    assert sess.get_providers() == ["B200ExecutionProvider"]


def test_batch_is_independent_of_batch_size(full):
    _, sess = full
    mel = phinet.synthetic_mel(5, 128, 301, 9).numpy()
    a = sess.run(None, {"mel_spectrogram": mel})[0]
    b = np.vstack([sess.run(None, {"mel_spectrogram": mel[i:i + 1]})[0] for i in range(5)])
    np.testing.assert_allclose(a, b, atol=1e-6)


def test_analysis_path_matches_oracle_end_to_end(full):
    """PCM -> round trip -> windows -> mel -> encoder -> mean + L2, incl. a multi-window track with
    the duplicated tail window (L = 720000) and a short zero-padded track."""
    from audiomuse_ai_b200 import clap_analyzer as ca, corpus
    model, sess = full
    ca.set_clap_audio_session(sess)
    try:
        tracks = [corpus.pcm16_to_float(corpus.synth_track(6)),
                  corpus.pcm16_to_float(corpus.synth_track(7, length=720000)),
                  corpus.pcm16_to_float(corpus.synth_track(8, length=300000))]
        res = ca.analyze_audio_batch(tracks)
        for wav, (emb, dur, nseg) in zip(tracks, res):
            x, _ = oseg.int16_round_trip(wav)
            segs = oseg.segment_audio(x)
            mels = np.concatenate([omel.compute_mel_spectrogram(s) for s in segs])
            want = oseg.pool_segments(phinet.embed_segments(model, mels))
            assert nseg == len(segs) and abs(dur - len(wav) / 48000) < 1e-9
            assert emb.shape == (512,) and emb.dtype == np.float32
            assert 1.0 - _cos(emb, want) <= COS_TOL
    finally:
        ca.set_clap_audio_session(None)


def test_analyze_audio_file_contract(tmp_path, full):
    import wave
    from audiomuse_ai_b200 import clap_analyzer as ca, corpus
    _, sess = full
    pcm = corpus.synth_track(9)
    p = tmp_path / "t.wav"
    with wave.open(str(p), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(48000); w.writeframes(pcm.tobytes())
    ca.set_clap_audio_session(sess)
    try:
        emb, dur, nseg = ca.analyze_audio_file(str(p))
        assert emb is not None and emb.shape == (512,) and nseg == 1 and abs(dur - 10.0) < 1e-9
        assert abs(np.linalg.norm(emb) - 1.0) < 1e-5
        assert ca.analyze_audio_file(str(tmp_path / "missing.wav")) == (None, 0, 0)   # never raises
        ca.config.CLAP_ENABLED = False
        assert ca.analyze_audio_file(str(p)) == (None, 0, 0)
    finally:
        ca.config.CLAP_ENABLED = True
        ca.set_clap_audio_session(None)


def test_config2_full_batch_properties(full):
    """BASELINE.json configs[1] at full size (256 x 10 s): size-independent properties -- unit norms,
    batch invariance (a track embeds the same alone and inside the batch), permutation equivariance --
    plus an oracle check on sampled tracks."""
    from audiomuse_ai_b200 import corpus
    model, sess = full
    pcm = corpus.synth_pcm_batch(256, start=0)
    offs = np.arange(257, dtype=np.int32)
    emb = sess.embed_tracks(pcm, offs)
    assert emb.shape == (256, 512) and np.isfinite(emb).all()
    np.testing.assert_allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-5)
    for i in (0, 77, 255):
        alone = sess.embed_tracks(pcm[i:i + 1], np.array([0, 1], np.int32))[0]
        np.testing.assert_allclose(alone, emb[i], atol=2e-6)
    perm = np.random.default_rng(0).permutation(256)
    emb_p = sess.embed_tracks(np.ascontiguousarray(pcm[perm]), offs)
    np.testing.assert_allclose(emb_p, emb[perm], atol=2e-6)
    for i in (3, 200):
        x = (pcm[i] / 32767.0).astype(np.float32)
        want = phinet.embed_segments(model, omel.compute_mel_spectrogram(x))[0]
        assert 1.0 - _cos(emb[i], want) <= COS_TOL
    # two windows of one track pool to the normalised mean of the single-window embeddings
    pooled = sess.embed_tracks(pcm[:2], np.array([0, 2], np.int32))[0]
    m = emb[:2].mean(0)
    np.testing.assert_allclose(pooled, m / (np.linalg.norm(m) + 1e-9), atol=2e-6)


def test_config2_edge_and_sampled_tracks_vs_oracle(full):
    """SURVEY 8(d) config 2: the six edge tracks (#0 silence -> every bin -100 dB, #1 full-scale sine, #2 white
    noise, #3 clipping, #4 one sample short (zero-padded window), #5 25 s = 5 windows incl. the tail window) plus
    ten tracks sampled from the 256-track bench batch, every one through PCM -> mel -> encoder -> pooling and
    against the CPU oracle (numpy mel + PyTorch fp32 encoder, one window per call).  Prints the margin."""
    from audiomuse_ai_b200 import clap_analyzer as ca, corpus
    model, sess = full
    ca.set_clap_audio_session(sess)
    try:
        waves = [corpus.pcm16_to_float(corpus.synth_track(i)) for i in range(6)]
        batch = corpus.synth_pcm_batch(256, start=0)
        picks = [0, 17, 33, 64, 99, 128, 150, 201, 230, 255]
        waves += [corpus.pcm16_to_float(batch[i]) for i in picks]
        res = ca.analyze_audio_batch(waves)
        worst = 0.0
        for ti, (wav, (emb, dur, nseg)) in enumerate(zip(waves, res)):
            x, _ = oseg.int16_round_trip(wav)
            segs = oseg.segment_audio(x)
            mels = np.concatenate([omel.compute_mel_spectrogram(s) for s in segs])
            if ti == 0:
                assert np.abs(mels + 100.0).max() < 1e-4      # silence: -100 dB everywhere
            want = oseg.pool_segments(phinet.embed_segments(model, mels))
            assert nseg == len(segs) and emb.shape == (512,)
            margin = 1.0 - _cos(emb, want)
            worst = max(worst, margin)
            print(f"[config-2 parity] track {ti}: windows {nseg}, 1 - cos = {margin:.2e}")
            assert margin <= COS_TOL
        assert res[5][2] == 5 and res[4][2] == 1
        print(f"[config-2 parity] 16 tracks, max(1 - cos) = {worst:.2e} (bar {COS_TOL:g})")
    finally:
        ca.set_clap_audio_session(None)


def test_embed_tracks_stream_matches_blocking_calls():
    """The pipelined bulk path (am_clap_embed_tracks_submit / _collect, two batches in flight) returns, batch by
    batch and in order, exactly what one blocking am_clap_embed_tracks call per batch returns -- also when batch
    sizes differ and when the generator is abandoned half way."""
    from audiomuse_ai_b200 import clap_analyzer as ca, corpus, weights
    sess = ca.B200Session.from_state_dict(weights.random_state_dict(0))
    batches = []
    for bi, n in enumerate([5, 2, 9, 1]):
        pcm = corpus.synth_pcm_batch(n, start=20 + 10 * bi)
        batches.append((pcm, np.arange(n + 1, dtype=np.int32)))
    want = [sess.embed_tracks(p, o) for p, o in batches]
    got = list(sess.embed_tracks_stream(iter(batches)))
    assert len(got) == len(want)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
    it = sess.embed_tracks_stream(iter(batches))
    first = next(it)
    np.testing.assert_array_equal(first, want[0])
    it.close()                                  # in-flight batches are drained
    np.testing.assert_array_equal(sess.embed_tracks(*batches[1]), want[1])
    assert list(sess.embed_tracks_stream(iter([]))) == []


def test_embed_tracks_refuses_mel_modes_other_than_clap():
    """The encoder is defined on CLAP's mel only: am_clap_embed_tracks_submit refuses another framing or compression
    before it opens a ticket, and the session keeps working."""
    import ctypes as C
    from audiomuse_ai_b200 import _lib, clap_analyzer as ca, corpus, weights
    sess = ca.B200Session.from_state_dict(weights.random_state_dict(0))
    pcm = corpus.synth_pcm_batch(2, start=30)
    offs = np.arange(3, dtype=np.int32)
    want = sess.embed_tracks(pcm, offs)
    out = np.empty_like(want)
    for framing, log_mode in ((1, 0), (2, 0), (0, 1)):
        cfg = ca._mel_cfg(transpose=False)
        cfg.framing, cfg.log_mode = framing, log_mode
        st = sess._lib.am_clap_embed_tracks_submit(sess._h, C.byref(cfg), _lib.ptr(pcm), pcm.shape[1],
                                                   _lib.ptr(offs), 2, _lib.ptr(out))
        assert st == _lib.AM_ERR_INVALID and "does not match the model" in _lib.last_error()
    np.testing.assert_array_equal(sess.embed_tracks(pcm, offs), want)
    np.testing.assert_array_equal(next(sess.embed_tracks_stream(iter([(pcm, offs)]))), want)
