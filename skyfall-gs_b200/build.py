"""Build recipe for libsfgs.so (sm_90a only).

Plain nvcc, in-tree output (skyfall-gs_b200/lib/libsfgs.so) so the built
library travels with the repository snapshot to the GPU box.  No torch headers
are involved: the library exposes the C ABI of include/sfgs.h and the Python
side binds it with ctypes.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libsfgs.so")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newer(src_paths, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(p) > t for p in src_paths)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "sfgs.h"))
    srcs = sources()
    objs = []
    jobs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJDIR, s[:-3] + ".o")
        objs.append(obj)
        if force or _newer([src] + headers, obj):
            jobs.append([nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    for stale in os.listdir(OBJDIR):   # objects whose source was removed must not be linked
        if stale.endswith(".o") and os.path.join(OBJDIR, stale) not in objs:
            os.remove(os.path.join(OBJDIR, stale))
    if jobs or force or _newer(objs, LIB):
        run([nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
