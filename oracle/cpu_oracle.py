"""numpy/ctypes driver of oracle/sfgs_oracle.c — the CPU restatement of the reference rasterizer.

TEST INFRASTRUCTURE.  Imported only by tests/, __graft_entry__.smoke() and
bench.py (cpu_baseline / --impl reference legs).  See the header of
sfgs_oracle.c for the reference file:line each routine follows and for how the
oracle itself is pinned (tests/golden/, generated from the unmodified reference
CUDA code).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "sfgs_oracle.c")
OUT_DIR = os.path.join(HERE, "_build")
LIB = os.path.join(OUT_DIR, "libsfgs_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        cmd = ["gcc", "-O2", "-std=c11", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-shared", "-fPIC",
               SRC, "-o", LIB, "-lm"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle build failed:\n" + r.stderr)
    return LIB


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.oracle_preprocess.restype = C.c_longlong
        L.oracle_binning.restype = C.c_int
        L.oracle_num_threads.restype = C.c_int
        _lib = L
    return _lib


def _f(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def num_threads() -> int:
    return int(lib().oracle_num_threads())


def forward(means3D, scales, rotations, opacities, shs, sh_degree, viewmatrix, projmatrix, campos, W, H, tan_fovx,
            tan_fovy, bg, kernel_size=0.1, scale_modifier=1.0, colors_precomp=None, cov3D_precomp=None,
            norm3D_precomp=None, extras=None):
    """Full forward. Returns a dict with outputs and every intermediate the parity tests compare."""
    L = lib()
    means3D, scales, rotations = _f(means3D), _f(scales), _f(rotations)
    opac = _f(opacities).reshape(-1)
    shs = _f(shs) if colors_precomp is None else None
    colors_precomp, cov3D_precomp, norm3D_precomp = _f(colors_precomp), _f(cov3D_precomp), _f(norm3D_precomp)
    extras = _f(extras)
    vm, pm, cam, bg = _f(viewmatrix).reshape(-1), _f(projmatrix).reshape(-1), _f(campos), _f(bg)
    P = means3D.shape[0]
    M = 0 if shs is None else shs.shape[1]
    ED = 0 if extras is None else extras.shape[1]
    o = dict(radii=np.zeros(P, np.int32), means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
             cov3D=np.zeros((P, 6), np.float32), norm3D=np.zeros((P, 3), np.float32), rgb=np.zeros((P, 3), np.float32),
             conic_opacity=np.zeros((P, 4), np.float32), clamped=np.zeros((P, 3), np.uint8),
             tiles_touched=np.zeros(P, np.uint32), point_offsets=np.zeros(P, np.uint32))
    R = L.oracle_preprocess(C.c_int(P), C.c_int(int(sh_degree)), C.c_int(M), _p(means3D), _p(scales),
                            C.c_float(scale_modifier), _p(rotations), _p(opac), _p(shs), _p(cov3D_precomp),
                            _p(norm3D_precomp), _p(colors_precomp), _p(vm), _p(pm), _p(cam), C.c_int(W), C.c_int(H),
                            C.c_float(tan_fovx), C.c_float(tan_fovy), C.c_float(kernel_size), _p(o["radii"]),
                            _p(o["means2D"]), _p(o["depths"]), _p(o["cov3D"]), _p(o["norm3D"]), _p(o["rgb"]),
                            _p(o["conic_opacity"]), _p(o["clamped"]), _p(o["tiles_touched"]), _p(o["point_offsets"]))
    R = int(R)
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    o["num_rendered"] = R
    o["keys"] = np.zeros(max(R, 1), np.uint64)[:R]
    o["point_list"] = np.zeros(max(R, 1), np.uint32)[:R]
    keys_buf = np.zeros(max(R, 1), np.uint64); list_buf = np.zeros(max(R, 1), np.uint32)
    o["ranges"] = np.zeros((tiles, 2), np.uint32)
    rc = L.oracle_binning(C.c_int(P), C.c_int(W), C.c_int(H), _p(o["radii"]), _p(o["means2D"]), _p(o["depths"]),
                          _p(o["point_offsets"]), C.c_longlong(R), _p(keys_buf), _p(list_buf), _p(o["ranges"]))
    if rc != 0:
        raise MemoryError("oracle_binning")
    o["keys"], o["point_list"] = keys_buf[:R], list_buf[:R]
    colors = colors_precomp if colors_precomp is not None else o["rgb"]
    norms = norm3D_precomp if norm3D_precomp is not None else o["norm3D"]
    o["color"] = np.zeros((3, H, W), np.float32); o["depth"] = np.zeros((1, H, W), np.float32)
    o["norm"] = np.zeros((3, H, W), np.float32); o["alpha"] = np.zeros((1, H, W), np.float32)
    o["extra"] = np.zeros((ED, H, W), np.float32)
    o["n_contrib"] = np.zeros(H * W, np.uint32)
    L.oracle_render(C.c_int(W), C.c_int(H), C.c_int(ED), _p(o["ranges"]), _p(list_buf), _p(o["means2D"]), _p(colors),
                    _p(norms), _p(o["depths"]), _p(extras), _p(o["conic_opacity"]), _p(bg), _p(o["color"]),
                    _p(o["depth"]), _p(o["norm"]), _p(o["alpha"]), _p(o["extra"]), _p(o["n_contrib"]))
    o["_inputs"] = dict(means3D=means3D, scales=scales, rotations=rotations, shs=shs, vm=vm, pm=pm, cam=cam, bg=bg,
                        colors_precomp=colors_precomp, cov3D_precomp=cov3D_precomp, norm3D_precomp=norm3D_precomp,
                        extras=extras, W=W, H=H, tan_fovx=tan_fovx, tan_fovy=tan_fovy, kernel_size=kernel_size,
                        scale_modifier=scale_modifier, sh_degree=int(sh_degree), M=M, ED=ED)
    return o


def blend_backward(fwd, dL_color, dL_depth, dL_norm, dL_alpha, dL_extra=None):
    """The blend adjoint of `forward` for the given pixel cotangents: the screen-space sums means2D [P,3], conic [P,4],
    opacity [P], colors [P,3], depths [P], norm3D [P,3] and extra [P,ED] the per-Gaussian stage starts from."""
    L = lib()
    I = fwd["_inputs"]
    P = I["means3D"].shape[0]
    W, H, ED = I["W"], I["H"], I["ED"]
    dL_color, dL_depth, dL_norm, dL_alpha, dL_extra = _f(dL_color), _f(dL_depth), _f(dL_norm), _f(dL_alpha), _f(dL_extra)
    colors = I["colors_precomp"] if I["colors_precomp"] is not None else fwd["rgb"]
    norms = I["norm3D_precomp"] if I["norm3D_precomp"] is not None else fwd["norm3D"]
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    g = dict(means2D=z(P, 3), conic=z(P, 4), opacity=z(P), colors=z(P, 3), depths=z(P), norm3D=z(P, 3),
             extra=z(P, max(ED, 0)))
    plist = np.ascontiguousarray(fwd["point_list"])
    L.oracle_render_backward(C.c_int(W), C.c_int(H), C.c_int(ED), _p(fwd["ranges"]), _p(plist), _p(I["bg"]),
                             _p(fwd["means2D"]), _p(fwd["conic_opacity"]), _p(colors), _p(fwd["depths"]), _p(norms),
                             _p(I["extras"]), _p(fwd["alpha"]), _p(fwd["n_contrib"]), _p(dL_color), _p(dL_depth),
                             _p(dL_norm), _p(dL_alpha), _p(dL_extra), _p(g["means2D"]), _p(g["conic"]),
                             _p(g["opacity"]), _p(g["colors"]), _p(g["depths"]), _p(g["norm3D"]), _p(g["extra"]))
    return g


def backward(fwd, dL_color, dL_depth, dL_norm, dL_alpha, dL_extra=None):
    """Backward of `forward` for the given pixel cotangents. Returns the 10 gradient arrays of the reference."""
    L = lib()
    I = fwd["_inputs"]
    P = I["means3D"].shape[0]
    W, H, M = I["W"], I["H"], I["M"]
    norms = I["norm3D_precomp"] if I["norm3D_precomp"] is not None else fwd["norm3D"]
    cov3D = I["cov3D_precomp"] if I["cov3D_precomp"] is not None else fwd["cov3D"]
    s = blend_backward(fwd, dL_color, dL_depth, dL_norm, dL_alpha, dL_extra)
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    g = dict(means2D=s["means2D"], conic=s["conic"], opacity=s["opacity"], colors=s["colors"], depths=s["depths"],
             means3D=z(P, 3), cov3D=z(P, 6), norm3D=s["norm3D"], sh=z(P, M, 3), scales=z(P, 3), rot=z(P, 4),
             extra=s["extra"])
    L.oracle_gauss_backward(C.c_int(P), C.c_int(I["sh_degree"]), C.c_int(M), _p(I["means3D"]), _p(fwd["radii"]),
                            _p(I["shs"]), _p(fwd["clamped"]), _p(I["scales"]), _p(I["rotations"]),
                            C.c_float(I["scale_modifier"]), _p(cov3D), _p(norms),
                            C.c_int(1 if I["norm3D_precomp"] is not None else 0), _p(I["vm"]), _p(I["pm"]),
                            C.c_int(W), C.c_int(H), C.c_float(I["tan_fovx"]), C.c_float(I["tan_fovy"]),
                            C.c_float(I["kernel_size"]), _p(I["cam"]), _p(fwd["conic_opacity"]), _p(g["means2D"]),
                            _p(g["conic"]), _p(g["opacity"]), _p(g["colors"]), _p(g["depths"]), _p(g["means3D"]),
                            _p(g["cov3D"]), _p(g["norm3D"]), _p(g["sh"]), _p(g["scales"]), _p(g["rot"]))
    g["opacity"] = g["opacity"].reshape(P, 1)
    return g


def mark_visible(means3D, viewmatrix):
    L = lib()
    means3D = _f(means3D)
    vm = _f(viewmatrix).reshape(-1)
    out = np.zeros(means3D.shape[0], np.uint8)
    L.oracle_mark_visible(C.c_int(means3D.shape[0]), _p(means3D), _p(vm), _p(out))
    return out.astype(bool)
