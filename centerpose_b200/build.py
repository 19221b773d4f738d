"""In-tree build of the C-ABI shared library (nvcc, sm_90a only: the kernels use wgmma, Hopper's warpgroup MMA).

``python -m centerpose_b200.build`` or ``__graft_entry__.build()``.  nvcc cross-compiles
without a GPU; the resulting ``centerpose_b200/lib/libcenterpose_b200.so`` is git-ignored
but travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import glob
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBPATH = os.path.join(LIBDIR, "libcenterpose_b200.so")
STAMP = os.path.join(LIBDIR, "build.stamp")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-Xcompiler", "-fPIC", "-std=c++17", "-O3", "-lineinfo"] + ARCH
# NVVM's -O3 pipeline for sm_90 takes tens of minutes on the CUDA-core kernels of net_simt.cu (seconds for other targets);
# -O1 compiles them in under half a minute
FILE_FLAGS = {"net_simt.cu": ["-Xcicc", "-O1"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build centerpose_b200's CUDA library")


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _digest() -> str:
    h = hashlib.sha256()
    for p in _sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + \
            [os.path.join(HERE, "..", "include", "centerpose_b200.h")]:
        with open(p, "rb") as f:
            h.update(p.encode()); h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode()); h.update(repr(sorted(FILE_FLAGS.items())).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    dig = _digest()
    if not force and os.path.exists(LIBPATH) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIBPATH
    objs = []
    nvcc = _nvcc()
    # compile each translation unit separately (parallel-friendly, faster rebuilds)
    procs = []
    for src in _sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, "-c"] + NVCC_FLAGS + FILE_FLAGS.get(os.path.basename(src), []) + ["-o", obj, src]
        if verbose:
            cmd.insert(1, "-Xptxas"); cmd.insert(2, "-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, pr in procs:
        out, _ = pr.communicate()
        if verbose and out:
            print(out)
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
    link = [nvcc, "-shared"] + ARCH + ["-o", LIBPATH] + objs
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIBPATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
