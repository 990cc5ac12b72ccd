"""Builds libaudiomuse_b200.so (sm_90a) in-tree with nvcc.  No JIT cache: the .so sits next
to this file so it travels to the GPU box with the repo snapshot."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
BUILD = os.path.join(PKG_DIR, "build")
LIB = os.path.join(PKG_DIR, "libaudiomuse_b200.so")
DEBUG_LIB = os.path.join(PKG_DIR, "libaudiomuse_b200_debug.so")   # product objects + csrc/debug/*.cu (probes, self tests)

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libaudiomuse_b200 cannot be built")


def _newest_header_mtime() -> float:
    m = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(PKG_DIR), "include")):
        for fn in os.listdir(root):
            if fn.endswith((".cuh", ".h")):
                m = max(m, os.path.getmtime(os.path.join(root, fn)))
    return m


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    dbg_dir = os.path.join(CSRC, "debug")
    dbg_srcs = sorted(f for f in os.listdir(dbg_dir) if f.endswith(".cu")) if os.path.isdir(dbg_dir) else []
    hdr_m = _newest_header_mtime()
    jobs = []
    objs, dbg_objs = [], []
    for d, names, out in ((CSRC, srcs, objs), (dbg_dir, dbg_srcs, dbg_objs)):
        for s in names:
            src = os.path.join(d, s)
            obj = os.path.join(BUILD, ("debug_" if d == dbg_dir else "") + s[:-3] + ".o")
            out.append(obj)
            if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m):
                jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        # AM_EXTRA_NVCC_FLAGS: extra flags for debug builds (e.g. -DNDEBUG=0 -G)
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("AM_EXTRA_NVCC_FLAGS", "").split(), "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for src, r in ex.map(compile_one, jobs):
                if verbose and r.stderr:
                    sys.stderr.write(r.stderr)
                if r.returncode != 0:
                    raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    stale = [o for o in os.listdir(BUILD) if o.endswith(".o") and os.path.join(BUILD, o) not in objs + dbg_objs]
    for o in stale:  # objects of sources that no longer exist must not be linked by accident
        os.remove(os.path.join(BUILD, o))
    for lib, members in ((LIB, objs), (DEBUG_LIB, objs + dbg_objs)):
        if jobs or stale or not os.path.exists(lib):
            cmd = [nvcc, "-shared", "-o", lib, *members, "-gencode", "arch=compute_90a,code=sm_90a",
                   "-Xcompiler", "-fPIC"]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
