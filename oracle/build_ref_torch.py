"""Build and install the reference's OWN torch extensions into oracle/_ref/ (test infrastructure).

What `pip install submodules/diff-gaussian-rasterization-depth` and `pip install submodules/fused-ssim` would put
into site-packages, put into the git-ignored oracle/_ref/ instead (it travels to the GPU box with the snapshot):

  oracle/_ref/diff_gauss/__init__.py   the reference's autograd wrapper, installed from RAST/diff_gauss/__init__.py
  oracle/_ref/diff_gauss/_C.so         its pybind module: RAST/{ext.cpp, rasterize_points.cu, cuda_rasterizer/*.cu}
  oracle/_ref/fused_ssim/__init__.py   the reference's fused-ssim wrapper, installed from SSIM/fused_ssim/__init__.py
  oracle/_ref/fused_ssim_cuda.so       its pybind module: SSIM/{ext.cpp, ssim.cu}

Sources are compiled where they lie under /root/reference (read-only) with torch.utils.cpp_extension — the same
toolchain path the reference's setup.py uses (CUDAExtension defaults, --expt-relaxed-constexpr included) — plus the
fixes SURVEY.md 8c / oracle/build_ref.py document for gcc 13 / nvcc 12.9 (`-include cstdint`, oracle/ref_glm_fix.h).
fused-ssim's setup.py flags (`--use_fast_math`, `--maxrregcount=32`; SSIM/setup.py) are reproduced.

Nothing here is committed: oracle/_ref/ is in .gitignore.  bench.py --impl reference drives these modules through
the reference's public API (diff_gauss.GaussianRasterizer + autograd; fused_ssim.fused_ssim); the parity tests use
them as the oracle for fused-ssim.
"""
from __future__ import annotations

import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("SFGS_REFERENCE", "/root/reference")
RAST = os.path.join(REF, "submodules", "diff-gaussian-rasterization-depth")
SSIM = os.path.join(REF, "submodules", "fused-ssim")


def available() -> bool:
    return os.path.isdir(RAST)


def built() -> bool:
    return os.path.exists(os.path.join(OUT, "diff_gauss", "_C.so")) and os.path.exists(os.path.join(OUT, "fused_ssim_cuda.so"))


def _load(name, sources, build_dir, extra_cuda, include):
    from torch.utils import cpp_extension
    os.makedirs(build_dir, exist_ok=True)
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    cpp_extension.load(name=name, sources=sources, extra_include_paths=include, extra_cuda_cflags=extra_cuda,
                       extra_cflags=["-include", "cstdint"], build_directory=build_dir, is_python_module=False,
                       verbose=False)
    return os.path.join(build_dir, name + ".so")


def build(force: bool = False) -> bool:
    if not available():
        return built()
    if built() and not force:
        return True
    fix = os.path.join(HERE, "ref_glm_fix.h")
    # --- diff_gauss._C ---------------------------------------------------------------------------------------
    srcs = [os.path.join(RAST, "cuda_rasterizer", f) for f in ("rasterizer_impl.cu", "forward.cu", "backward.cu")]
    srcs += [os.path.join(RAST, "rasterize_points.cu"), os.path.join(RAST, "ext.cpp")]
    so = _load("_C", srcs, os.path.join(OUT, "_build_diff_gauss"), ["-include", "cstdint", "-include", fix, "-w"],
               [os.path.join(RAST, "third_party", "glm")])
    pkg = os.path.join(OUT, "diff_gauss")
    os.makedirs(pkg, exist_ok=True)
    shutil.copyfile(so, os.path.join(pkg, "_C.so"))
    shutil.copyfile(os.path.join(RAST, "diff_gauss", "__init__.py"), os.path.join(pkg, "__init__.py"))   # the install step
    # --- fused_ssim_cuda -------------------------------------------------------------------------------------
    so = _load("fused_ssim_cuda", [os.path.join(SSIM, "ssim.cu"), os.path.join(SSIM, "ext.cpp")],
               os.path.join(OUT, "_build_fused_ssim"), ["--use_fast_math", "--maxrregcount=32", "-w"], [SSIM])
    shutil.copyfile(so, os.path.join(OUT, "fused_ssim_cuda.so"))
    pkg = os.path.join(OUT, "fused_ssim")
    os.makedirs(pkg, exist_ok=True)
    shutil.copyfile(os.path.join(SSIM, "fused_ssim", "__init__.py"), os.path.join(pkg, "__init__.py"))
    for d in ("_build_diff_gauss", "_build_fused_ssim"):
        shutil.rmtree(os.path.join(OUT, d), ignore_errors=True)
    return True


def import_reference_packages():
    """Import the installed reference packages under private names (the product's own `diff_gauss` / `fused_ssim`
    packages keep those names): returns (ref_diff_gauss, ref_fused_ssim)."""
    import importlib.util
    if not built():
        raise ImportError("oracle/_ref torch extensions missing: run `python oracle/build_ref_torch.py` where /root/reference exists")
    import torch  # noqa: F401  (libtorch must be loaded before the extension modules)

    def load_pkg(name, path, submods):
        spec = importlib.util.spec_from_file_location(name, os.path.join(path, "__init__.py"),
                                                      submodule_search_locations=[path])
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        for sub_name, sub_path in submods.items():      # pre-register compiled submodules / top-level extension modules
            sspec = importlib.util.spec_from_file_location(sub_name, sub_path)
            smod = importlib.util.module_from_spec(sspec)
            sys.modules[sub_name] = smod
            sspec.loader.exec_module(smod)
        spec.loader.exec_module(mod)
        return mod

    dg = load_pkg("ref_diff_gauss", os.path.join(OUT, "diff_gauss"), {"ref_diff_gauss._C": os.path.join(OUT, "diff_gauss", "_C.so")})
    fs = load_pkg("ref_fused_ssim", os.path.join(OUT, "fused_ssim"), {"fused_ssim_cuda": os.path.join(OUT, "fused_ssim_cuda.so")})
    return dg, fs


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
