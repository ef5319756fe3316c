"""Compile the UNMODIFIED reference rasterizer + simple-knn into oracle/_ref/ (test infrastructure).

Sources are compiled where they lie under /root/reference (read-only); nothing
is copied.  Flags follow the reference's own build (torch CUDAExtension defaults:
no fast-math, default FMA contraction, --expt-relaxed-constexpr) plus the two
fixes needed under gcc 13 / nvcc 12.9 that SURVEY.md §8c documents:
`-include cstdint` and `--expt-relaxed-constexpr` (without the latter nvcc
silently emits empty backward-preprocess kernels), plus the force-included
oracle/ref_glm_fix.h (see its header: without it nvcc 12.9 drops the SH colour
stores of the reference's preprocess kernel because glm's TMax functor is
host-only).

Run here (container with /root/reference); the resulting .so travels to the GPU
box with the repository snapshot (oracle/_ref/ is git-ignored, not gpurun-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("SFGS_REFERENCE", "/root/reference")
RAST = os.path.join(REF, "submodules", "diff-gaussian-rasterization-depth")
KNN = os.path.join(REF, "submodules", "simple-knn")
LIB = os.path.join(OUT, "libref_rasterizer.so")

FLAGS = ["-std=c++17", "-O3", "-include", "cstdint", "-include", os.path.join(HERE, "ref_glm_fix.h"),
         "--expt-relaxed-constexpr", "-w",
         "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
         "-I", os.path.join(RAST, "third_party", "glm"), "-I", os.path.join(RAST, "cuda_rasterizer"), "-I", KNN]


def available() -> bool:
    return os.path.isdir(RAST)


def build(force: bool = False) -> str | None:
    if not available():
        return LIB if os.path.exists(LIB) else None
    if os.path.exists(LIB) and not force:
        return LIB
    os.makedirs(OUT, exist_ok=True)
    srcs = {
        "forward": os.path.join(RAST, "cuda_rasterizer", "forward.cu"),
        "backward": os.path.join(RAST, "cuda_rasterizer", "backward.cu"),
        "rasterizer_impl": os.path.join(RAST, "cuda_rasterizer", "rasterizer_impl.cu"),
        "simple_knn": os.path.join(KNN, "simple_knn.cu"),
        "ref_shim": os.path.join(HERE, "ref_shim.cu"),
    }
    nvcc = os.environ.get("NVCC", "nvcc")

    def cc(item):
        name, src = item
        obj = os.path.join(OUT, name + ".o")
        extra = ["-include", "cfloat"] if name == "simple_knn" else []   # FLT_MAX, same class of fix as cstdint
        r = subprocess.run([nvcc] + FLAGS + extra + ["-c", src, "-o", obj], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"reference build failed for {src}:\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=5) as ex:
        objs = list(ex.map(cc, srcs.items()))
    r = subprocess.run([nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("reference link failed:\n" + r.stderr)
    for o in objs:
        os.remove(o)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
