"""wgmma/TMA GEMM vs the SIMT reference kernel, on device (am_selftest_gemm).  Each case runs in
a subprocess under a timeout so a pipeline hang cannot wedge the test session."""
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

CASES = [
    # M, N, K, flags (1 bias, 2 relu6, 4 residual, 8 f32 out, 16 m_fastest, 32 col_sub/alpha)
    (128, 64, 64, 0), (128, 256, 64, 0), (256, 80, 144, 3), (1000, 432, 80, 3), (4096, 80, 432, 5),
    (333, 2592, 576, 3), (512, 576, 2592, 5), (130, 1360, 288, 3), (128, 5000, 512, 8 | 16),
    (256, 4100, 256, 8 | 16 | 32), (64, 48, 16, 1),
    # the remaining tile widths: 16, 32, 96, 112 (+ N % 8 != 0 with a residual: the unstaged bf16 epilogue), 128, 160
    (256, 16, 64, 1), (300, 24, 48, 3), (512, 96, 96, 5), (200, 100, 64, 4 | 1), (333, 128, 144, 3), (257, 136, 80, 5),
]

SCRIPT = r"""
import ctypes as C, sys
sys.path.insert(0, %r)
from audiomuse_ai_b200 import _lib
lib = _lib.load_debug()   # the self test lives in libaudiomuse_b200_debug.so (include/audiomuse_b200_debug.h)
d = C.c_double(-1)
st = lib.am_selftest_gemm(%d, %d, %d, %d, C.byref(d))
print("RESULT", st, d.value, lib.am_last_error().decode() if st else "")
"""


@pytest.mark.parametrize("M,N,K,flags", CASES)
def test_wgmma_gemm_matches_simt(M, N, K, flags):
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", SCRIPT % (root, M, N, K, flags)], capture_output=True, text=True,
                       timeout=120)
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT")]
    assert line, f"no result: rc={r.returncode}\n{r.stdout}\n{r.stderr[-2000:]}"
    _, st, diff, *msg = line[0].split(" ", 3)
    assert int(st) == 0, msg
    # both sides accumulate bf16 products in fp32; only summation order and one bf16 rounding differ
    tol = 0.08 if not (flags & 8) else 2e-3
    assert float(diff) <= tol, f"max |wgmma - simt| = {diff}"
