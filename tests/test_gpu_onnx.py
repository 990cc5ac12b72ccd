"""The engine on the model file the reference deploys: an ONNX ModelProto read and lowered by am_clap_load
(tasks/clap_analyzer.py:109-116,132-147,534).  Files are exported from the oracle modules with the reference's
exporter arguments (tests/onnx_export.py); parity bar: cosine >= 1 - 1e-3 against the PyTorch module AND against
the independent ONNX interpreter (oracle/onnx_ref.py), for the PhiNet student and for a structurally different
MobileNetV3 / EfficientAT-style graph (squeeze-excite, hardswish, 5x5 depthwise, Gemm head) -- the loader is
graph driven, not a PhiNet reader.  Also: the lifecycle functions and the out-of-memory convention."""
import os
import wave

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mel as omel
from oracle import mobilenet, onnx_ref, phinet, segments as oseg
from tests import onnx_export, onnx_rewrite

COS_TOL = 1e-3


def _cos(a, b):
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-30))


def _check(sess, model, path, T, n=3, seed=11):
    mel = phinet.synthetic_mel(n, 128, T, seed).numpy()
    with torch.no_grad():
        want = torch.cat([model(torch.from_numpy(mel[i:i + 1])) for i in range(n)]).numpy()
    g = onnx_ref.load(path)
    want2 = np.concatenate([onnx_ref.run(g, {"mel_spectrogram": mel[i:i + 1]})[0] for i in range(n)])
    assert np.abs(want - want2).max() < 1e-5          # the two oracles agree (reference's own export check)
    got = sess.run(None, {"mel_spectrogram": mel})[0]
    assert got.shape == want.shape
    np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-5)
    worst = max(1.0 - _cos(a, b) for a, b in zip(got, want))
    print(f"[onnx parity] {os.path.basename(path)} T={T}: max(1-cos) = {worst:.2e}")
    assert worst <= COS_TOL
    return got


def test_student_onnx_small_and_equals_blob_session(tmp_path):
    from audiomuse_ai_b200 import clap_analyzer as ca, weights
    cfg = phinet.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256)
    model = phinet.make_random_student(3, cfg)
    path = onnx_export.export_onnx(model, str(tmp_path / "student_small.onnx"))
    sess = ca.B200Session.from_file(path)
    assert sess.embedding_dim == 512 and sess.n_mels == 128
    for T in (101, 333):
        got = _check(sess, model, path, T)
    blob = ca.B200Session.from_state_dict(model.state_dict(), weights.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256))
    mel = phinet.synthetic_mel(3, 128, 333, 11).numpy()
    ref = blob.run(None, {"mel_spectrogram": mel})[0]
    # same layer program, weights folded by two different routes (exporter's constant folding vs weights.py)
    assert max(1.0 - _cos(a, b) for a, b in zip(got, ref)) < 2e-5


def test_student_onnx_full_size_10s_windows_external_data(tmp_path):
    """The shipped configuration (alpha 3.0, 8 blocks, 2048-d trunk) at the reference's 10 s window, with the tensor
    data in `model.onnx.data` next to the file (the layout of model_epoch_36.onnx, clap_analyzer.py:132-147)."""
    from audiomuse_ai_b200 import clap_analyzer as ca
    model = phinet.make_random_student(0)
    path = onnx_export.export_onnx(model, str(tmp_path / "model_epoch_36.onnx"), external_data=True)
    assert os.path.getsize(path) < 200_000 and os.path.getsize(path + ".data") > 10_000_000
    sess = ca.B200Session.from_file(path)
    _check(sess, model, path, 1001, n=2, seed=5)


@pytest.mark.parametrize("encoding", ["attrs", "inputs"])
def test_mobilenet_onnx_small(tmp_path, encoding):
    from audiomuse_ai_b200 import clap_analyzer as ca
    cfg = mobilenet.MNConfig(rows=mobilenet.SMALL_ROWS, head_dim=256)
    model = mobilenet.make_random_mobilenet(5, cfg)
    raw = onnx_export.export_onnx_bytes(model)
    if encoding == "inputs":
        raw = onnx_rewrite.attrs_to_inputs(raw)
    path = str(tmp_path / "mn_small.onnx")
    with open(path, "wb") as f:
        f.write(raw)
    sess = ca.B200Session.from_file(path)
    for T in (129, 400):
        _check(sess, model, path, T)
    # bytes route (am_clap_load_mem) gives the same embeddings
    mel = phinet.synthetic_mel(2, 128, 129, 3).numpy()
    a = sess.run(None, {"mel_spectrogram": mel})[0]
    b = ca.B200Session(blob=raw).run(None, {"mel_spectrogram": mel})[0]
    np.testing.assert_array_equal(a, b)


def test_mobilenet_onnx_large_10s_window(tmp_path):
    """MobileNetV3-large rows at width 1.0 (the EfficientAT mn10 shape) on a 10 s window, through the fused PCM path."""
    from audiomuse_ai_b200 import clap_analyzer as ca, corpus
    model = mobilenet.make_random_mobilenet(1)
    path = onnx_export.export_onnx(model, str(tmp_path / "mn10.onnx"))
    sess = ca.B200Session.from_file(path)
    _check(sess, model, path, 1001, n=2, seed=2)
    ca.set_clap_audio_session(sess)
    try:
        wav = corpus.pcm16_to_float(corpus.synth_track(7, length=720000))
        (emb, dur, nseg), = ca.analyze_audio_batch([wav])
        x, _ = oseg.int16_round_trip(wav)
        segs = oseg.segment_audio(x)
        mels = np.concatenate([omel.compute_mel_spectrogram(s) for s in segs])
        want = oseg.pool_segments(mobilenet.embed_segments(model, mels))
        assert nseg == len(segs) == 3
        assert 1.0 - _cos(emb, want) <= COS_TOL
    finally:
        ca.set_clap_audio_session(None)


def test_unsupported_graph_fails_the_load_loudly(tmp_path):
    from audiomuse_ai_b200 import _lib, clap_analyzer as ca
    cfg = mobilenet.MNConfig(rows=mobilenet.SMALL_ROWS, head_dim=256)
    raw = onnx_export.export_onnx_bytes(mobilenet.make_random_mobilenet(5, cfg))
    bad = str(tmp_path / "bad.onnx")
    with open(bad, "wb") as f:
        f.write(raw.replace(b"\x22\x04Relu", b"\x22\x04Selu", 1))
    with pytest.raises(_lib.B200Error) as e:
        ca.B200Session.from_file(bad)
    assert "Selu" in str(e.value)


def test_lifecycle_over_clap_audio_model_path(tmp_path):
    """tasks/clap_analyzer.py:47-165,387-393,690-699: lazy singleton load from config.CLAP_AUDIO_MODEL_PATH (the ONNX
    file itself, no private blob), idempotent unload, is_* predicates, analyze_audio_file on top."""
    from audiomuse_ai_b200 import clap_analyzer as ca, corpus
    cfg = phinet.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=256)
    model = phinet.make_random_student(3, cfg)
    path = onnx_export.export_onnx(model, str(tmp_path / "model_epoch_36.onnx"))
    old = (ca.config.CLAP_AUDIO_MODEL_PATH, getattr(ca.config, "CLAP_B200_WEIGHTS_PATH", ""))
    ca.unload_clap_model()
    try:
        ca.config.CLAP_B200_WEIGHTS_PATH = ""
        ca.config.CLAP_AUDIO_MODEL_PATH = str(tmp_path / "missing.onnx")
        assert not ca.is_clap_available() and not ca.is_clap_audio_loaded() and not ca.is_clap_model_loaded()
        assert ca.initialize_clap_audio_model() is False
        with pytest.raises(RuntimeError):
            ca.get_clap_audio_model()
        assert ca.unload_clap_audio_only() is False               # nothing loaded: reference returns False
        ca.config.CLAP_AUDIO_MODEL_PATH = path
        assert ca.is_clap_available()
        assert ca.initialize_clap_audio_model() is True
        assert ca.is_clap_audio_loaded() and ca.is_clap_model_loaded()
        s1 = ca.get_clap_audio_model()
        assert ca.initialize_clap_audio_model() is True and ca.get_clap_audio_model() is s1   # singleton
        assert s1.get_providers() == ["B200ExecutionProvider"] and s1.get_inputs()[0].name == "mel_spectrogram"
        wav_path = tmp_path / "t.wav"
        pcm = corpus.synth_track(9)
        with wave.open(str(wav_path), "wb") as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(48000); w.writeframes(pcm.tobytes())
        emb, dur, nseg = ca.analyze_audio_file(str(wav_path))
        x, _ = oseg.int16_round_trip(corpus.pcm16_to_float(pcm))
        want = oseg.pool_segments(phinet.embed_segments(model, omel.compute_mel_spectrogram(x)))
        assert nseg == 1 and abs(dur - 10.0) < 1e-9 and 1.0 - _cos(emb, want) <= COS_TOL
        assert ca.unload_clap_model() is True
        assert not ca.is_clap_audio_loaded()
        assert ca.unload_clap_model() is False                     # idempotent
        emb2, _, _ = ca.analyze_audio_file(str(wav_path))           # lazy reload inside analyze_audio_file
        np.testing.assert_array_equal(emb, emb2)
        ca.config.CLAP_ENABLED = False
        ca.unload_clap_model()
        assert ca.initialize_clap_audio_model() is False            # disabled: no load (reference :53-55)
    finally:
        ca.config.CLAP_ENABLED = True
        ca.config.CLAP_AUDIO_MODEL_PATH, ca.config.CLAP_B200_WEIGHTS_PATH = old
        ca.unload_clap_model()


def test_out_of_memory_convention_and_retry(tmp_path, monkeypatch, caplog):
    """include/audiomuse_b200.h: allocation failures return AM_ERR_OOM with 'out of memory' in the message, so the
    reference's string match (tasks/memory_utils.py:375-382) detects them; analyze_audio_file then cleans up and
    retries once (tasks/clap_analyzer.py:536-549).  A failed submit leaves the session usable (ADVICE r1)."""
    import ctypes as C
    from audiomuse_ai_b200 import _lib, clap_analyzer as ca, corpus, weights
    lib = _lib.load()
    # 1. a REAL allocation failure: an index of 2^31 - 2 x 512 floats (4 TiB; the most rows an index takes) cannot be
    # allocated
    x = torch.zeros(512, device="cuda")
    h = C.c_void_p()
    st = lib.am_knn_build_dev(C.c_void_p(x.data_ptr()), (1 << 31) - 2, 512, 0, None, C.byref(h))
    assert st == _lib.AM_ERR_OOM and "out of memory" in _lib.last_error()
    with pytest.raises(_lib.B200OutOfMemory) as e:
        _lib.check(st)
    assert isinstance(e.value, MemoryError) and ca.is_memory_error(e.value)
    assert not ca.is_memory_error(ValueError("bad shape"))
    # 2. the library keeps working after it
    sess = ca.B200Session.from_state_dict(weights.random_state_dict(0))
    pcm = corpus.synth_pcm_batch(3, start=40)
    offs = np.arange(4, dtype=np.int32)
    want = sess.embed_tracks(pcm, offs)
    # 3. a submit that fails mid-stream (injected after its allocations) must not strand a ticket
    batches = [(pcm, offs), (pcm[:2], offs[:3]), (pcm, offs)]
    it = sess.embed_tracks_stream(iter(batches))
    first_error = None
    monkeypatch.setenv("AM_TEST_FAIL_SUBMIT", "1")
    try:
        next(it)
    except _lib.B200OutOfMemory as err:
        first_error = err
    monkeypatch.delenv("AM_TEST_FAIL_SUBMIT")
    assert first_error is not None and "out of memory" in str(first_error)
    np.testing.assert_array_equal(sess.embed_tracks(pcm, offs), want)           # blocking call still works
    got = list(sess.embed_tracks_stream(iter(batches)))                         # and so does a new stream
    np.testing.assert_array_equal(got[0], want)
    np.testing.assert_array_equal(got[2], want)
    # 4. analyze_audio_file: first attempt fails with OOM, cleanup + one retry succeeds (reference :536-549)
    wav_path = tmp_path / "t.wav"
    with wave.open(str(wav_path), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(48000); w.writeframes(corpus.synth_track(9).tobytes())
    ca.set_clap_audio_session(sess)
    calls = {"n": 0}
    real = ca.embed_pcm16_windows

    def flaky(pcm16, seg_offsets):
        calls["n"] += 1
        if calls["n"] == 1:
            raise _lib.B200OutOfMemory(_lib.AM_ERR_OOM, "out of memory: cudaMalloc failed (injected)")
        return real(pcm16, seg_offsets)

    monkeypatch.setattr(ca, "embed_pcm16_windows", flaky)
    try:
        emb, dur, nseg = ca.analyze_audio_file(str(wav_path))
        assert calls["n"] == 2 and emb is not None and nseg == 1
        # a non-memory error is NOT retried: (None, 0, 0) after one call
        calls["n"] = 0
        monkeypatch.setattr(ca, "embed_pcm16_windows", lambda *a: (_ for _ in ()).throw(ValueError("boom")))
        assert ca.analyze_audio_file(str(wav_path)) == (None, 0, 0)
    finally:
        ca.set_clap_audio_session(None)
