"""CPU-side checks of the C-ABI boundary: the library loads, exports exactly what
include/audiomuse_b200.h declares, and its host-only entry points agree with the oracle / goldens.
No GPU compute is issued here."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from audiomuse_ai_b200 import _lib
    return _lib.load()


def _header_symbols():
    txt = open(os.path.join(ROOT, "include", "audiomuse_b200.h")).read()
    return sorted(set(re.findall(r"AM_API\s+[\w\s\*]+?\b(am_\w+)\s*\(", txt)))


def test_library_exports_every_declared_symbol(lib):
    from audiomuse_ai_b200 import _lib
    names = _header_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    assert set(_lib.SIGNATURES) == set(names), set(_lib.SIGNATURES) ^ set(names)


def test_debug_and_trace_entry_points_live_in_the_debug_library_only(lib):
    """The probes, self tests, debug entry points and the encoder trace (include/audiomuse_b200_debug.h,
    am_debug_kmeans_step and am_debug_encoder_trace among them) live in libaudiomuse_b200_debug.so only."""
    from audiomuse_ai_b200 import _lib
    txt = open(os.path.join(ROOT, "include", "audiomuse_b200_debug.h")).read()
    dbg_names = sorted(set(re.findall(r"AM_API\s+[\w\s\*]+?\b(am_\w+)\s*\(", txt)))
    assert set(dbg_names) == set(_lib.DEBUG_SIGNATURES) == {"am_selftest_gemm", "am_bench_gemm", "am_probe_pipe",
                                                            "am_debug_block", "am_debug_kmeans_step",
                                                            "am_debug_encoder_plan", "am_debug_encoder_trace"}
    dbg = _lib.load_debug()
    for n in dbg_names:
        assert hasattr(dbg, n)
        assert not hasattr(lib, n), f"{n} is exported by the product library"


def test_no_cuda_at_import_and_loud_failure_without_gpu(lib):
    import torch
    from audiomuse_ai_b200 import _lib, clap_analyzer as ca
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.am_init(-1) == _lib.AM_ERR_NO_DEVICE
    assert "no CPU fallback" in _lib.last_error()
    with pytest.raises(_lib.B200Error):
        ca.compute_mel_spectrogram(np.zeros(48000, np.float32))


def test_filterbank_bit_identical_to_oracle(lib):
    from audiomuse_ai_b200 import _lib
    from oracle import mel as omel
    for n_mels, fmin, fmax in ((128, 0.0, 14000.0), (64, 50.0, 14000.0), (96, 0.0, 24000.0)):
        cfg = _lib.MelCfg(48000, 2048, 480, n_mels, fmin, fmax, 0)
        out = np.zeros((n_mels, 1025), np.float32)
        assert lib.am_mel_filterbank(C.byref(cfg), _lib.ptr(out)) == 0
        ref = omel.mel_filterbank(48000, 2048, n_mels, fmin, fmax)
        assert np.abs(out - ref).max() <= 1e-9
    assert lib.am_mel_num_frames(C.byref(cfg), 480000) == 1001


def test_mel_framings_and_out_of_range_modes(lib):
    """am_mel_num_frames counts frames under each framing and refuses a window shorter than the framing accepts; a
    framing, log_mode or covariance type outside its values is AM_ERR_INVALID before any device work."""
    from audiomuse_ai_b200 import _lib

    def cfg(framing=0, log_mode=0):
        return _lib.MelCfg(16000, 512, 256, 96, 0.0, 8000.0, 0, framing, log_mode)
    for framing, n, T in ((0, 48000, 188), (0, 257, 2), (1, 48000, 186), (1, 512, 1), (2, 48000, 188), (2, 1, 1)):
        assert lib.am_mel_num_frames(C.byref(cfg(framing)), n) == T, (framing, n)
    for framing, n in ((0, 256), (1, 511), (2, 0)):
        assert lib.am_mel_num_frames(C.byref(cfg(framing)), n) == _lib.AM_ERR_INVALID, (framing, n)
    plan = C.c_void_p()
    for framing, log_mode, word in ((3, 0, "framing"), (-1, 0, "framing"), (0, 2, "log_mode")):
        assert lib.am_mel_plan_create(C.byref(cfg(framing, log_mode)), C.byref(plan)) == _lib.AM_ERR_INVALID
        assert word in _lib.last_error() and not plan.value
        assert lib.am_mel_num_frames(C.byref(cfg(framing, log_mode)), 48000) == _lib.AM_ERR_INVALID
    assert lib.am_gmm_fit(None, 100, 2, 2, 4, 1, 10, 1e-3, 1e-6, None, 0, *[None] * 15) == _lib.AM_ERR_INVALID
    assert "am_gmm_fit: covariance_type 4" in _lib.last_error()


def test_pcm_to_segments_matches_reference_goldens(lib, golden_dir):
    """C-ABI windowing + int16 truncation == the reference's analyze_audio_file (golden)."""
    from make_golden import SEGMENT_CASE_LENGTHS, golden_waveform
    from audiomuse_ai_b200 import clap_analyzer as ca
    g = np.load(os.path.join(golden_dir, "segments_golden.npz"))
    for ci, L in enumerate(SEGMENT_CASE_LENGTHS):
        seg = ca.pcm_to_segments(golden_waveform(100 + ci, L))
        assert seg.dtype == np.int16 and seg.shape == (int(g[f"nseg_{ci}"]), 480000)
        f = (seg / 32767.0).astype(np.float32)
        np.testing.assert_array_equal(f[:, :8], g[f"seg_head_{ci}"])
        np.testing.assert_array_equal(f[:, -8:], g[f"seg_tail_{ci}"])
        np.testing.assert_array_equal(f.astype(np.float64).sum(axis=1), g[f"seg_sum_{ci}"])


def test_weights_blob_roundtrip_structure():
    from audiomuse_ai_b200 import weights
    cfg = weights.StudentConfig(alpha=0.5, num_layers=5, trunk_dim=64)
    sd = weights.random_state_dict(1, cfg)
    blob = weights.export_blob(sd, cfg)
    assert blob[:4] == b"AMW1"
    c0, blocks = weights.block_plan(cfg)
    n_rec = int.from_bytes(blob[16:20], "little")
    assert n_rec == 1 + sum(3 if b.block_id else 2 for b in blocks) + 1
    # the production config: 8.3 M parameters, ~4.3 GMAC per 10 s window
    macs = weights.count_macs()
    assert 4.0e9 < sum(macs.values()) < 4.6e9
    c0, blocks = weights.block_plan(weights.StudentConfig())
    assert c0 == 144 and [b.cout for b in blocks] == [72, 72, 72, 144, 144, 288, 288, 576, 576]
    assert [b.stride for b in blocks] == [1, 2, 1, 2, 1, 2, 1, 2, 1]


def test_product_weights_load_into_oracle_model():
    """state_dict naming of the product generator == StudentCLAPAudio's (oracle restatement)."""
    import torch
    from audiomuse_ai_b200 import weights
    from oracle import phinet
    cfg_w = weights.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=128)
    cfg_o = phinet.StudentConfig(alpha=0.5, num_layers=6, trunk_dim=128)
    m = phinet.StudentCLAPAudio(cfg_o)
    res = m.load_state_dict({k: torch.from_numpy(v) for k, v in weights.random_state_dict(2, cfg_w).items()},
                            strict=False)
    assert not res.unexpected_keys
    assert all(k.endswith("num_batches_tracked") for k in res.missing_keys)
    out = m.eval()(phinet.synthetic_mel(1, 128, 101, 0))
    assert out.shape == (1, 512) and torch.isfinite(out).all()


def test_voyager_compat_host_logic():
    from audiomuse_ai_b200 import voyager_compat as vc
    idx = vc.Index(vc.Space.Cosine, num_dimensions=8, M=64, ef_construction=1024)
    x = np.random.default_rng(0).standard_normal((10, 8)).astype(np.float32)
    assert idx.add_items(x, ids=np.arange(10)) == list(range(10))
    assert len(idx) == 10 and idx.num_elements == 10 and 3 in idx and 11 not in idx
    with pytest.raises(vc.RecallError):
        idx.query(x[0], 11)                      # voyager_manager.py:1448 catches this
    with pytest.raises(ValueError):
        idx.add_items(np.zeros((2, 7), np.float32))
    import io
    buf = io.BytesIO()
    idx.save(buf)
    buf.seek(0)
    idx2 = vc.Index.load(buf)
    assert len(idx2) == 10 and idx2.space == vc.Space.Cosine and idx2.num_dimensions == 8
    np.testing.assert_array_equal(idx2._rows, x)
    ids, d = idx.query(x[:0].reshape(0, 8), 3)
    assert ids.shape == (0, 3)
