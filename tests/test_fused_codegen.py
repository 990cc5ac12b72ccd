"""The fused inverted-residual block kernel stays within its register budget: every fused_block_kernel instantiation
(stride 1 / 2, with and without an expansion) in the built library has a zero-byte stack frame and no local-memory
loads or stores in its SASS.  The consumer warpgroups run at 232 registers (setmaxnreg) and hold up to 96 fp32
accumulators of the expansion and projection MMAs while the depthwise keeps its taps and output rows in registers;
a spill there would put local-memory traffic into the per-chunk loop.

Reads the library build() makes (AM_FUSED_CODEGEN_LIB names another one).  Needs cuobjdump, not a GPU."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.environ.get("AM_FUSED_CODEGEN_LIB") or os.path.join(ROOT, "audiomuse-ai_b200", "libaudiomuse_b200.so")
# the launcher instantiates stride 1 / 2 x with / without an expansion conv
N_INSTANTIATIONS = 4


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip("cuobjdump not found")


def _dump(*flags):
    assert os.path.exists(LIB), f"{LIB} is not built"
    r = subprocess.run([_cuobjdump(), *flags, LIB], capture_output=True, text=True, check=True)
    return r.stdout


def _resource_usage():
    """[(mangled name, resource line)] of every fused_block_kernel instantiation"""
    usage = re.findall(r"Function (\S*fused_block_kernel\S*):\s*\n\s*(REG:.*)", _dump("-res-usage"))
    assert len(usage) == N_INSTANTIATIONS, usage
    return usage


def test_fused_block_kernel_has_no_stack_frame():
    for name, res in _resource_usage():
        assert re.search(r"\bSTACK:0\b", res), f"{name}: {res}"


def test_fused_block_kernel_sass_has_no_local_memory_access():
    sass = _dump("-sass", "-fun", ",".join(name for name, _ in _resource_usage()))
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    fused = [f for f in funcs if "fused_block_kernel" in f.split("\n", 1)[0]]
    assert len(fused) == N_INSTANTIATIONS
    for f in fused:
        name, body = f.split("\n", 1)
        local = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not local, f"{name.strip()}: {len(local)} local-memory instructions"
