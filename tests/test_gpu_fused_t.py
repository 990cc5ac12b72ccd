"""The fused inverted-residual block kernel (csrc/fused_block.cu) against the layer-by-layer path (AM_FUSED_BLOCKS=0:
expansion GEMM, depthwise kernel, projection GEMM).  The choice is read from the environment when the model is
loaded, so every variant runs in its own process."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r"""
import sys, numpy as np
sys.path.insert(0, %r)
from audiomuse_ai_b200 import clap_analyzer as ca, weights
sess = ca.B200Session.from_state_dict(weights.random_state_dict(0))
rng = np.random.default_rng(0)
mel = (rng.standard_normal((3, 1, 128, %d)) * 12 - 30).astype(np.float32)
mel[1, :, :, :] = -100.0                      # digital silence: every bin on the floor
from audiomuse_ai_b200 import _lib
_lib.profile_enable(True)
np.save(sys.argv[1], sess.run(None, {"mel_spectrogram": mel})[0])
open(sys.argv[1] + ".kernels", "w").write("\n".join(_lib.profile_report()))
"""


def _embed(tmp_path, name, env, T=1001):
    out = str(tmp_path / f"{name}.npy")
    r = subprocess.run([sys.executable, "-c", CHILD % (ROOT, T), out], env=dict(os.environ, **env), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    fused_ran = any("fused_block_kernel" in k for k in open(out + ".kernels").read().splitlines())
    assert fused_ran == (env.get("AM_FUSED_BLOCKS") != "0"), f"{name}: fused kernel ran = {fused_ran}"
    return np.load(out)


def _cos(a, b):
    return np.array([float(np.dot(x, y) / (np.linalg.norm(x) * np.linalg.norm(y))) for x, y in zip(a, b)])


def test_fused_block_kernel_matches_the_layer_by_layer_path(tmp_path):
    ref = _embed(tmp_path, "layer_by_layer", {"AM_FUSED_BLOCKS": "0"})
    got = _embed(tmp_path, "fused", {})
    c = _cos(got, ref)
    print(f"fused: min cosine vs layer by layer {c.min():.7f}, max |diff| {np.abs(got - ref).max():.2e}")
    # both round the expanded tensor and the depthwise output to bf16; the depthwise sums in fp32 here, in fp16 pairs
    # on the layer path
    assert c.min() > 1 - 1e-4, c
    assert np.abs(got - ref).max() < 2e-3


def test_one_model_follows_a_changing_window_length():
    """The execution plan is kept per window length: 1001, 333 and again 1001 frames on one model give what a fresh
    model gives for each length, also after the workspace was released."""
    from audiomuse_ai_b200 import clap_analyzer as ca, weights

    def embed(sess, T):
        mel = (np.random.default_rng(T).standard_normal((3, 1, 128, T)) * 12 - 30).astype(np.float32)
        return sess.run(None, {"mel_spectrogram": mel})[0]

    blob = weights.export_blob(weights.random_state_dict(0))
    fresh = {T: embed(ca.B200Session(blob), T) for T in (1001, 333)}
    sess = ca.B200Session(blob)
    for T in (1001, 333, 1001):
        np.testing.assert_array_equal(embed(sess, T), fresh[T])
    sess.release_workspace()
    for T in (333, 1001):
        np.testing.assert_array_equal(embed(sess, T), fresh[T])


def test_short_window_runs_through_the_partial_tiles(tmp_path):
    """T = 333 frames: spatial sizes that are no multiple of the 8 x 8 tile (the last tiles of every block are partial)."""
    ref = _embed(tmp_path, "layer_by_layer_s", {"AM_FUSED_BLOCKS": "0"}, T=333)
    new = _embed(tmp_path, "fused_s", {}, T=333)
    assert _cos(new, ref).min() > 1 - 1e-4
    assert np.abs(new - ref).max() < 2e-3
