"""The wgmma GEMM kernel keeps its MMAs asynchronous and within its register budget: every gemm_wgmma_kernel<BN>
instantiation in the built library has a zero-byte stack frame, no local-memory loads or stores, and keeps one wgmma
group in flight across K blocks (wgmma.wait_group 1 -> WARPGROUP.DEPBAR.LE gsb0, 0x1); and ptxas, compiling gemm.cu
with the build's flags, reports no serialised wgmma (C7514 / C7515 / C7520).  A non-wgmma instruction that defines an
accumulator register (an epilogue that works in place in them) makes ptxas serialise every wgmma of the kernel; a
spill puts local-memory traffic into the epilogue of every tile.

Reads the library build() makes (AM_GEMM_CODEGEN_LIB names another one) and runs nvcc.  Needs no GPU."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "audiomuse-ai_b200")
LIB = os.environ.get("AM_GEMM_CODEGEN_LIB") or os.path.join(PKG, "libaudiomuse_b200.so")


def _tool(name):
    for cand in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip(f"{name} not found")


def _dump(*flags):
    assert os.path.exists(LIB), f"{LIB} is not built"
    r = subprocess.run([_tool("cuobjdump"), *flags, LIB], capture_output=True, text=True, check=True)
    return r.stdout


def _resource_usage():
    """[(mangled name, resource line)] of every gemm_wgmma_kernel instantiation"""
    usage = re.findall(r"Function (\S*gemm_wgmma_kernel\S*):\s*\n\s*(REG:.*)", _dump("-res-usage"))
    assert usage, "no gemm_wgmma_kernel in the library"
    return usage


def _sass_bodies():
    sass = _dump("-sass", "-fun", ",".join(name for name, _ in _resource_usage()))
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    return [f.split("\n", 1) for f in funcs if "gemm_wgmma_kernel" in f.split("\n", 1)[0]]


def test_gemm_kernel_has_no_stack_frame():
    for name, res in _resource_usage():
        assert re.search(r"\bSTACK:0\b", res), f"{name}: {res}"


def test_gemm_kernel_sass_has_no_local_memory_access():
    bodies = _sass_bodies()
    assert len(bodies) == len(_resource_usage())
    for name, body in bodies:
        local = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not local, f"{name.strip()}: {len(local)} local-memory instructions"


def test_gemm_kernel_keeps_one_wgmma_group_in_flight():
    for name, body in _sass_bodies():
        assert re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x1\b", body), f"{name.strip()}: no wait_group 1"


def test_gemm_wgmma_is_not_serialised():
    spec = importlib.util.spec_from_file_location("_am_build_native", os.path.join(PKG, "build_native.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    nvcc = _tool("nvcc")
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, *mod.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(PKG, "csrc", "gemm.cu"), "-o",
                            os.path.join(tmp, "gemm.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    compiled = re.findall(r"Compiling entry function '(\S*gemm_wgmma_kernel\S*)'", r.stderr)
    assert compiled, "ptxas compiled no gemm_wgmma_kernel"
    serialised = [l for l in r.stderr.splitlines() if re.search(r"\((C7514|C7515|C7520)\)", l)]
    assert not serialised, "\n".join(serialised[:5])
    frames = re.findall(r"Function properties for (\S*gemm_wgmma_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(compiled)
    for name, *counts in frames:
        assert counts == ["0", "0", "0"], f"{name}: stack / spill stores / spill loads = {counts}"
