"""In-tree build of libngp_b200.so (nvcc, sm_90a only: the MLP kernels use Hopper wgmma).

No torch dependency: the library is a plain C-ABI shared object (include/ngp_b200.h) that the
Python host code reaches through ctypes.  The built file lives at taichi_nerfs_b200/lib/ (git-ignored), so the
package is importable straight from the source tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

_PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_PKG, "csrc")
LIBDIR = os.path.join(_PKG, "lib")
LIB = os.path.join(LIBDIR, "libngp_b200.so")
INCLUDE = os.path.join(os.path.dirname(_PKG), "include")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O2",
    "--expt-relaxed-constexpr",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libngp_b200.so")
    return nvcc


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(INCLUDE, "ngp_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    host_cc = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else None
    ccbin = ["-ccbin", host_cc] if host_cc else []
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
        hdrs.append(os.path.join(INCLUDE, "ngp_b200.h"))
        newest = max(os.path.getmtime(p) for p in [src] + hdrs)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > newest:
            continue
        cmd = [nvcc] + ccbin + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"nvcc failed for {src}:\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("nvcc compilation failed")
    cmd = [nvcc] + ccbin + ["-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
