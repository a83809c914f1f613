"""Builds the C-ABI shared library (csrc/*.cu -> lib/libsdetr_b200.so) with plain nvcc for sm_90a.

Deliberately NOT a torch C++ extension: the library has no torch/ATen symbols (that coupling is what
broke the reference's extension on a newer torch, SURVEY.md fact 2) and is loaded with ctypes.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libsdetr_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into one shared library; returns its path."""
    if not force and not is_stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [_nvcc(), *ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out.decode())
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    link = [_nvcc(), *ARCH, "-shared", "-cudart", "static", "-o", LIB, *objs]
    subprocess.run(link, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
