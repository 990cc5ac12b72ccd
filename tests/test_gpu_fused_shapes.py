"""The fused inverted-residual block kernel (csrc/fused_block.cu) against the layer-by-layer path (AM_FUSED_BLOCKS=0)
across student widths and window lengths.  alpha 0.5 .. 3 gives block inputs of 16 to 144 padded channels (K tails of
the 64-channel halo loads), stride-2, residual and no-expansion blocks; alpha 6 makes block 1 (144 -> 144 channels at
stride 2) too large for a two-stage weight ring, so it runs the kernel's one-stage ring.  T = 333 and 517 leave
partial output tiles along time; T = 1001 is the shipped window.  With 128 mel bins the block widths are 64, 32 and 16,
so tiles are never partial along the mel axis.  The fused/layer choice is read from the environment when a model is
loaded, so each variant runs every case in one process of its own."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {0.5: (333, 517, 1001), 1.0: (333, 517, 1001), 2.0: (333, 517, 1001), 3.0: (333, 517, 1001), 6.0: (333,)}
CHILD = r"""
import sys, json, numpy as np
sys.path.insert(0, %r)
from audiomuse_ai_b200 import _lib, clap_analyzer as ca, weights
_lib.profile_enable(True)
ran = {}
for alpha, lengths in %r.items():
    cfg = weights.StudentConfig(alpha=alpha)
    sess = ca.B200Session.from_state_dict(weights.random_state_dict(0, cfg), cfg)
    _lib.profile_report()
    for T in lengths:
        rng = np.random.default_rng(T)
        mel = (rng.standard_normal((3, 1, 128, T)) * 12 - 30).astype(np.float32)
        np.save(f"{sys.argv[1]}/a{alpha}_t{T}.npy", sess.run(None, {"mel_spectrogram": mel})[0])
    ran[str(alpha)] = any("fused_block_kernel" in k for k in _lib.profile_report())
json.dump(ran, open(sys.argv[1] + "/fused_ran.json", "w"))
"""
CASE_IDS = [(a, t) for a, ts in CASES.items() for t in ts]


def _run_variant(out_dir, env):
    os.makedirs(out_dir, exist_ok=True)
    r = subprocess.run([sys.executable, "-c", CHILD % (ROOT, CASES), out_dir],
                       env=dict(os.environ, **env), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.load(open(os.path.join(out_dir, "fused_ran.json")))


@pytest.fixture(scope="module")
def variants(tmp_path_factory):
    root = tmp_path_factory.mktemp("fused_shapes")
    ref, fused = str(root / "layer_by_layer"), str(root / "fused")
    return ref, _run_variant(ref, {"AM_FUSED_BLOCKS": "0"}), fused, _run_variant(fused, {})


@pytest.mark.parametrize("alpha,T", CASE_IDS)
def test_fused_block_matches_layer_by_layer(variants, alpha, T):
    ref_dir, ref_ran, fused_dir, fused_ran = variants
    assert not ref_ran[str(alpha)], f"alpha {alpha}: the layer-by-layer run launched the fused kernel"
    assert fused_ran[str(alpha)], f"alpha {alpha}: the fused kernel did not run"
    ref = np.load(f"{ref_dir}/a{alpha}_t{T}.npy")
    got = np.load(f"{fused_dir}/a{alpha}_t{T}.npy")
    cos = np.array([float(np.dot(x, y) / (np.linalg.norm(x) * np.linalg.norm(y))) for x, y in zip(got, ref)])
    print(f"alpha {alpha} T {T}: min cosine {cos.min():.7f}, max |diff| {np.abs(got - ref).max():.2e}")
    assert cos.min() > 1 - 1e-4, cos
    assert np.abs(got - ref).max() < 2e-3
