"""Bit-identity of the encoder across two builds of the library.

    python tools/encoder_equiv.py dump FILE.npz       # on the build to compare against
    python tools/encoder_equiv.py compare FILE.npz    # on the build under test: every array np.array_equal

Seeded inputs only.  Models: the default student, alpha 6 (every block in one stage of the fused kernel), 64 mel bins,
and the MobileNetV3-style ONNX graph of the tests (squeeze-excite, hardswish, 5x5 depthwise); each with the fused
block kernel and with AM_FUSED_BLOCKS=0 (read when the model is loaded).  Per model: embeddings from a mel batch
(am_clap_embed -> am_clap_embed_dev) at T = 1001 and T = 333, from PCM windows (am_clap_embed_tracks), from two
overlapping submits (am_clap_embed_tracks_submit / _collect), a second mel batch at the first T after the other T
(the plan follows T), and am_clap_flops_per_segment / am_clap_flops_split at both T.  Needs an H100."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiomuse_ai_b200 import clap_analyzer as ca, weights  # noqa: E402

LENGTHS = (1001, 333)
HOP = 480


def _student(**kw):
    cfg = weights.StudentConfig(**kw)
    return lambda: ca.B200Session.from_state_dict(weights.random_state_dict(0, cfg), cfg)


def _mobilenet():
    from oracle import mobilenet
    from tests import onnx_export
    raw = onnx_export.export_onnx_bytes(mobilenet.make_random_mobilenet(5, mobilenet.MNConfig(rows=mobilenet.SMALL_ROWS,
                                                                                               head_dim=256)))
    return lambda: ca.B200Session(blob=raw)


# name -> (session factory, windows of the mel batch at T = 1001 and at T = 333)
MODELS = {
    "student": (_student(), (256, 7)),
    "alpha6": (_student(alpha=6.0), (5, 7)),
    "mels64": (_student(n_mels=64), (5, 7)),
    "mobilenet": (_mobilenet(), (5, 7)),
}


def _collect():
    out = {}
    for name, (make, windows) in MODELS.items():
        for fused in ("1", "0"):
            os.environ["AM_FUSED_BLOCKS"] = fused
            sess = make()
            ca.config.CLAP_AUDIO_N_MELS = sess.n_mels
            key = f"{name}/fused{fused}"
            for T, n in zip(LENGTHS, windows):
                rng = np.random.default_rng(1000 * n + T)
                mel = (rng.standard_normal((n, 1, sess.n_mels, T)) * 12 - 30).astype(np.float32)
                out[f"{key}/embed/T{T}"] = sess.run(None, {"mel_spectrogram": mel})[0]
                out[f"{key}/flops/T{T}"] = np.array([sess.flops_per_segment(T), *sess.flops_split(T)])
                batches = []
                for bi, tracks in enumerate(((2, 1, 3), (1, 2))):   # windows per track
                    offs = np.concatenate([[0], np.cumsum(tracks)]).astype(np.int32)
                    pcm = np.random.default_rng(T + bi).integers(-8000, 8000, (int(offs[-1]), (T - 1) * HOP)).astype(np.int16)
                    batches.append((pcm, offs))
                out[f"{key}/tracks/T{T}"] = sess.embed_tracks(*batches[0])
                for bi, emb in enumerate(sess.embed_tracks_stream(iter(batches + batches[:1]))):
                    out[f"{key}/stream{bi}/T{T}"] = emb
            mel = (np.random.default_rng(5).standard_normal((3, 1, sess.n_mels, LENGTHS[0])) * 12 - 30).astype(np.float32)
            out[f"{key}/embed_again/T{LENGTHS[0]}"] = sess.run(None, {"mel_spectrogram": mel})[0]
            sess.close()
    return out


def main():
    mode, path = sys.argv[1], sys.argv[2]
    got = _collect()
    if mode == "dump":
        np.savez(path, **got)
        print(f"wrote {len(got)} arrays to {path}")
        return 0
    want = np.load(path)
    bad = [k for k in sorted(set(want.files) | set(got)) if k not in got or k not in want.files or
           not np.array_equal(want[k], got[k])]
    for k in bad:
        print(f"DIFFERENT: {k}")
    print(f"{len(got) - len(bad)} of {len(got)} arrays equal")
    return 1 if bad or len(got) != len(want.files) else 0


if __name__ == "__main__":
    sys.exit(main())
