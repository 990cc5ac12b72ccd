"""Device-time sweep of the wgmma GEMM (am_bench_gemm): TFLOP/s by shape.  Needs an H100."""
import ctypes as C
import sys

sys.path.insert(0, ".")
import audiomuse_ai_b200 as am  # noqa: E402
from audiomuse_ai_b200 import _lib  # noqa: E402

lib = _lib.load_debug()
for (M, N, K) in [(8192, 8192, 4096), (8192, 8192, 512), (16384, 1408, 288), (131072, 1408, 288),
                  (131072, 288, 1408), (8192, 64, 4096), (8192, 128, 4096), (8192, 256, 4096)]:
    ms = C.c_double(0)
    _lib.check_debug(lib.am_bench_gemm(M, N, K, 10, C.byref(ms)))
    print(f"M={M} N={N} K={K}: {ms.value:.4f} ms  {2.0 * M * N * K / ms.value / 1e9:.1f} TFLOP/s", flush=True)
