"""The mel kernel keeps its FFT in registers: every mel_kernel instantiation in the built library has a zero-byte stack
frame and no local-memory loads or stores in its SASS.  A rolled FFT stage loop once put the 32-point FFT's re/im
arrays in local memory (a 256-byte frame) and made the kernel several times slower; this catches that at build time.

Reads the library build() makes (AM_MEL_CODEGEN_LIB names another one).  Needs cuobjdump, not a GPU."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.environ.get("AM_MEL_CODEGEN_LIB") or os.path.join(ROOT, "audiomuse-ai_b200", "libaudiomuse_b200.so")
# the launcher instantiates int16 / f32 input x 19 / 32 weighted 32-bin groups
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
    """[(mangled name, resource line)] of every mel_kernel instantiation"""
    usage = re.findall(r"Function (\S*mel_kernel\S*):\s*\n\s*(REG:.*)", _dump("-res-usage"))
    assert len(usage) == N_INSTANTIATIONS, usage
    return usage


def test_mel_kernel_has_no_stack_frame():
    for name, res in _resource_usage():
        assert re.search(r"\bSTACK:0\b", res), f"{name}: {res}"


def test_mel_kernel_sass_has_no_local_memory_access():
    sass = _dump("-sass", "-fun", ",".join(name for name, _ in _resource_usage()))
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    mel = [f for f in funcs if "mel_kernel" in f.split("\n", 1)[0]]
    assert len(mel) == N_INSTANTIATIONS
    for f in mel:
        name, body = f.split("\n", 1)
        local = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not local, f"{name.strip()}: {len(local)} local-memory instructions"
