"""Compile the CUDA sources under csrc/ into fastspeech2_b200/libfs2b200.so for the H100 (sm_90a), next to the Python package.

Each .cu is compiled to an object in parallel (build/obj/, git-ignored) and the objects are linked with nvcc --shared.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "libfs2b200.so")
OBJ = os.path.join(ROOT, "build", "obj")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include")]


def sources():
    return sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")))


def _headers():
    return glob.glob(os.path.join(HERE, "csrc", "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h"))


def _newer(deps, target) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src: str, verbose: bool):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    r = subprocess.run([NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj], capture_output=True, text=True)
    return src, obj, r


def build(force: bool = False, verbose: bool = False) -> str:
    srcs, hdrs = sources(), _headers()
    if not force and not _newer(srcs + hdrs, LIB):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    todo = [s for s in srcs if force or verbose or _newer([s] + hdrs, os.path.join(OBJ, os.path.basename(s)[:-3] + ".o"))]
    with ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 1))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), todo))
    for src, _, r in results:
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"nvcc failed compiling {os.path.basename(src)}")
        if verbose:
            print(f"== {os.path.basename(src)}\n{r.stdout}{r.stderr}")
    objs = [os.path.join(OBJ, os.path.basename(s)[:-3] + ".o") for s in srcs]
    r = subprocess.run([NVCC, "--shared"] + ARCH + objs + ["-o", LIB], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed linking libfs2b200.so")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
