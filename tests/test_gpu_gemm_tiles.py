"""wgmma/TMA GEMM vs the SIMT reference kernel (am_selftest_gemm) on the shapes the bf16 TMA-store epilogue has to get
right: every kind of staging box (64-column SWIZZLE_128B boxes and a last box of 16 / 32 / 48 columns with
SWIZZLE_32B / _64B / none), N tails inside a tile (odd N included), M tails that leave a warpgroup's rows partly or
wholly below the matrix, and bias + ReLU6 + residual epilogues; plus the late encoder blocks' widths (288 and 2592 as
144-column tiles, 1360 / 1408 as 128-column tiles).  Each case runs in a subprocess under a timeout."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

CASES = [
    # M, N, K, flags (1 bias, 2 relu6, 4 residual, 8 f32 out, 16 m_fastest)
    # the late encoder blocks: 144 = 2 x 64 + a 16-column box, 128 = 2 x 64
    (300, 288, 736, 3), (333, 288, 1408, 7), (1000, 2592, 576, 3), (260, 576, 2592, 7), (200, 1408, 288, 7),
    (130, 1360, 288, 7), (129, 736, 144, 3),
    # last boxes: 16 (BN 80), 32 (BN 32, 96, 160, 224), 48 (BN 48, 112), 64-column boxes only (BN 64, 128, 192, 256)
    (256, 72, 64, 7), (256, 24, 64, 7), (192, 150, 96, 7), (128, 200, 64, 7), (256, 40, 80, 7), (300, 100, 64, 7),
    (256, 64, 64, 7), (256, 184, 128, 7), (256, 250, 64, 7),
    # odd N (the last column pair is half outside), M tails: 1 row, 65 rows (warpgroup 1 wholly outside), 191
    (200, 17, 64, 7), (64, 33, 48, 5), (1, 288, 64, 7), (65, 144, 64, 7), (191, 2592, 64, 3), (65, 1360, 128, 7 | 16),
]

SCRIPT = r"""
import ctypes as C, sys
sys.path.insert(0, %r)
from audiomuse_ai_b200 import _lib
lib = _lib.load_debug()
d = C.c_double(-1)
st = lib.am_selftest_gemm(%d, %d, %d, %d, C.byref(d))
print("RESULT", st, d.value, lib.am_last_error().decode() if st else "")
"""


@pytest.mark.parametrize("M,N,K,flags", CASES)
def test_wgmma_gemm_tile_shapes_match_simt(M, N, K, flags):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", SCRIPT % (root, M, N, K, flags)], capture_output=True, text=True,
                       timeout=120)
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT")]
    assert line, f"no result: rc={r.returncode}\n{r.stdout}\n{r.stderr[-2000:]}"
    _, st, diff, *msg = line[0].split(" ", 3)
    assert int(st) == 0, msg
    # both sides accumulate bf16 products in fp32; only summation order and one bf16 rounding differ
    assert float(diff) <= 0.08, f"max |wgmma - simt| = {diff}"
