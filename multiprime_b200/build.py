"""Build libmpb200.so in-tree with nvcc for sm_90a (H100).  The library lives next to this file, so the package is
importable and runnable straight from the source tree once this has run."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libmpb200.so")
SOURCES = ["mpb200.cu", "mpb_cscan.cu", "mpb_prefilter.cu", "mpb_walk_dev.cu", "mpb_peer.cu", "mpb_dimer.cu", "mpb_walk.cu",
           "mpb_products.cu", "mpb_pools.cu"]
HEADERS = [os.path.join(CSRC, h) for h in ("mpb_device.cuh", "mpb_host.h", "mpb_cscan.h", "mpb_walk_core.h")] + \
    [os.path.join(ROOT, "include", "mpb200.h")]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-Xptxas", "-v" if verbose else "-O3", "-shared", "-Xcompiler", "-fPIC", "-cudart", "static", "-t", "5",
           "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed: " + " ".join(cmd))
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
