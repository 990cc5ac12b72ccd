"""The fused inverted-residual block kernel (csrc/fused_block.cu) against the layer-by-layer path (AM_FUSED_BLOCKS=0)
for a student with 80 mel bins.  Its block widths along the mel axis are 40, 20 and 10: block 0's output (40 wide)
fills whole 8-pixel tiles, the outputs of blocks 1-4 (20 and 10 wide) leave partial tiles along the mel axis as well
as along time.  The fused/layer choice is read from the environment when a model
is loaded, so each variant runs in a process of its own; the fused run also checks that the fused kernel ran."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_MELS, LENGTHS = 80, (333, 1001)
CHILD = r"""
import sys, json, numpy as np
sys.path.insert(0, %r)
from audiomuse_ai_b200 import _lib, clap_analyzer as ca, weights
_lib.profile_enable(True)
cfg = weights.StudentConfig(n_mels=%d)
sess = ca.B200Session.from_state_dict(weights.random_state_dict(0, cfg), cfg)
_lib.profile_report()
for T in %r:
    mel = (np.random.default_rng(T).standard_normal((3, 1, cfg.n_mels, T)) * 12 - 30).astype(np.float32)
    np.save(f"{sys.argv[1]}/t{T}.npy", sess.run(None, {"mel_spectrogram": mel})[0])
json.dump(any("fused_block_kernel" in k for k in _lib.profile_report()), open(sys.argv[1] + "/fused_ran.json", "w"))
"""


def _run_variant(out_dir, env):
    os.makedirs(out_dir, exist_ok=True)
    r = subprocess.run([sys.executable, "-c", CHILD % (ROOT, N_MELS, LENGTHS), out_dir],
                       env=dict(os.environ, **env), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.load(open(os.path.join(out_dir, "fused_ran.json")))


@pytest.fixture(scope="module")
def variants(tmp_path_factory):
    root = tmp_path_factory.mktemp("fused_mels")
    ref, fused = str(root / "layer_by_layer"), str(root / "fused")
    return ref, _run_variant(ref, {"AM_FUSED_BLOCKS": "0"}), fused, _run_variant(fused, {})


@pytest.mark.parametrize("T", LENGTHS)
def test_fused_block_matches_layer_by_layer_at_80_mels(variants, T):
    ref_dir, ref_ran, fused_dir, fused_ran = variants
    assert not ref_ran, "the layer-by-layer run launched the fused kernel"
    assert fused_ran, "the fused kernel did not run"
    ref = np.load(f"{ref_dir}/t{T}.npy")
    got = np.load(f"{fused_dir}/t{T}.npy")
    cos = np.array([float(np.dot(x, y) / (np.linalg.norm(x) * np.linalg.norm(y))) for x, y in zip(got, ref)])
    print(f"n_mels {N_MELS} T {T}: min cosine {cos.min():.7f}, max |diff| {np.abs(got - ref).max():.2e}")
    assert cos.min() > 1 - 1e-4, cos
    assert np.abs(got - ref).max() < 2e-3
