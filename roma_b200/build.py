"""Builds libromab200.so (all CUDA kernels + the C ABI) in-tree with nvcc for sm_90a (H100).

    python -m roma_b200.build [--force]

The shared library lands in roma_b200/lib/ (git-ignored build output).
nvcc cross-compiles without a GPU, so the library can be built on a machine that has none.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIB = os.path.join(LIBDIR, "libromab200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I", INCLUDE,
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    h.update(" ".join(NVCC_FLAGS).encode())
    for dep in [path] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cuh")] + \
            [os.path.join(INCLUDE, "romab200.h")]:
        with open(dep, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _compile(src, verbose):
    obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
    stamp = obj + ".sha1"
    dig = _digest(src)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False
    cmd = ["nvcc", *NVCC_FLAGS, "-c", src, "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(res.stderr)
    with open(stamp, "w") as f:
        f.write(dig)
    return obj, True


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJDIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJDIR):
            os.remove(os.path.join(OBJDIR, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    objs = [o for o, _ in results]
    if any(changed for _, changed in results) or not os.path.exists(LIB):
        cmd = ["nvcc", "-shared", *ARCH, "-o", LIB, *objs, "-lcudart"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
