"""The oracles of the parity tests for a forward with subpixel offsets — test infrastructure for test_subpixel_offset.py.

tests/subpixel_oracle.c and tests/subpixel_adjudicator_f64.cu include the unchanged oracles (oracle/sfgs_oracle.c,
oracle/adjudicator_f64.cu) and add their per-pixel blend / blend adjoint with the sample position moved by the offset.
Both are compiled on first use into a directory under the system's temporary directory (the tree may be read-only).

    cpu_forward(..., subpixel_offset)    oracle.cpu_oracle.forward, then the blend again at the offset positions
    cpu_backward(fwd, dL_color, ...)     oracle.cpu_oracle.backward for that forward
    backward_f64(I, ..., subpixel_offset)  oracle.adjudicator.backward_f64 for a forward with offsets
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import torch

from oracle import cpu_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
_libs = {}


def _build(src, deps, cmd):
    """Compile `src` (cmd with {src} / {out} placeholders) once per content of src + deps into the temporary
    directory; returns the loaded library."""
    h = hashlib.sha256()
    for p in [src] + deps:
        with open(p, "rb") as fh:
            h.update(fh.read())
    out_dir = os.path.join(tempfile.gettempdir(), f"sfgs_subpixel_oracle_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    lib = os.path.join(out_dir, f"{os.path.basename(src)}.{h.hexdigest()[:16]}.so")
    if not os.path.exists(lib):
        tmp = f"{lib}.{os.getpid()}.tmp"
        r = subprocess.run([a.format(src=src, out=tmp) for a in cmd], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"building {src} failed:\n" + r.stderr)
        os.replace(tmp, lib)
    return C.CDLL(lib)


def cpu_lib():
    if "cpu" not in _libs:
        # the oracle's own flags (oracle/cpu_oracle.py)
        _libs["cpu"] = _build(os.path.join(HERE, "subpixel_oracle.c"), [cpu_oracle.SRC],
                              ["gcc", "-O2", "-std=c11", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-mfma",
                               "-shared", "-fPIC", "{src}", "-o", "{out}", "-lm"])
    return _libs["cpu"]


def adj_lib():
    if "adj" not in _libs:
        from oracle import adjudicator
        L = _build(os.path.join(HERE, "subpixel_adjudicator_f64.cu"), [adjudicator.SRC],
                   [os.environ.get("NVCC", "nvcc"), "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-Xcompiler", "-fPIC", "-shared", "{src}", "-o", "{out}"])
        L.adj_backward_f64_subpixel.restype = C.c_int
        _libs["adj"] = L
    return _libs["adj"]


_f, _p = cpu_oracle._f, cpu_oracle._p


def cpu_forward(*args, subpixel_offset, **kw):
    """cpu_oracle.forward (same arguments) with pixel (x, y) sampled at (x + off[y,x,0], y + off[y,x,1])."""
    o = cpu_oracle.forward(*args, **kw)
    I = o["_inputs"]
    W, H, ED = I["W"], I["H"], I["ED"]
    off = _f(subpixel_offset).reshape(H, W, 2)
    colors = I["colors_precomp"] if I["colors_precomp"] is not None else o["rgb"]
    norms = I["norm3D_precomp"] if I["norm3D_precomp"] is not None else o["norm3D"]
    plist = np.ascontiguousarray(o["point_list"])
    cpu_lib().oracle_render_subpixel(
        C.c_int(W), C.c_int(H), C.c_int(ED), _p(o["ranges"]), _p(plist), _p(o["means2D"]), _p(colors), _p(norms),
        _p(o["depths"]), _p(I["extras"]), _p(o["conic_opacity"]), _p(I["bg"]), _p(o["color"]), _p(o["depth"]),
        _p(o["norm"]), _p(o["alpha"]), _p(o["extra"]), _p(o["n_contrib"]), _p(off))
    o["_subpixel_offset"] = off
    return o


def cpu_backward(fwd, dL_color, dL_depth, dL_norm, dL_alpha, dL_extra=None):
    """cpu_oracle.backward for a forward of cpu_forward."""
    L = cpu_lib()
    I = fwd["_inputs"]
    P = I["means3D"].shape[0]
    W, H, M, ED = I["W"], I["H"], I["M"], I["ED"]
    dL_color, dL_depth, dL_norm, dL_alpha, dL_extra = _f(dL_color), _f(dL_depth), _f(dL_norm), _f(dL_alpha), _f(dL_extra)
    colors = I["colors_precomp"] if I["colors_precomp"] is not None else fwd["rgb"]
    norms = I["norm3D_precomp"] if I["norm3D_precomp"] is not None else fwd["norm3D"]
    cov3D = I["cov3D_precomp"] if I["cov3D_precomp"] is not None else fwd["cov3D"]
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    g = dict(means2D=z(P, 3), conic=z(P, 4), opacity=z(P), colors=z(P, 3), depths=z(P), means3D=z(P, 3), cov3D=z(P, 6),
             norm3D=z(P, 3), sh=z(P, M, 3), scales=z(P, 3), rot=z(P, 4), extra=z(P, max(ED, 0)))
    plist = np.ascontiguousarray(fwd["point_list"])
    L.oracle_render_backward_subpixel(
        C.c_int(W), C.c_int(H), C.c_int(ED), _p(fwd["ranges"]), _p(plist), _p(I["bg"]), _p(fwd["means2D"]),
        _p(fwd["conic_opacity"]), _p(colors), _p(fwd["depths"]), _p(norms), _p(I["extras"]), _p(fwd["alpha"]),
        _p(fwd["n_contrib"]), _p(dL_color), _p(dL_depth), _p(dL_norm), _p(dL_alpha), _p(dL_extra), _p(g["means2D"]),
        _p(g["conic"]), _p(g["opacity"]), _p(g["colors"]), _p(g["depths"]), _p(g["norm3D"]), _p(g["extra"]),
        _p(fwd["_subpixel_offset"]))
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


def _tp(t):
    return None if (t is None or t.numel() == 0) else C.c_void_p(t.data_ptr())


def backward_f64(I, means3D, radii, shs, scales, rotations, scale_modifier, viewmatrix, projmatrix, campos, tan_fovx,
                 tan_fovy, kernel_size, sh_degree, bg, out_alpha, cot, subpixel_offset):
    """oracle.adjudicator.backward_f64 (same arguments, SH colours) for a forward with the [H,W,2] offsets given."""
    L = adj_lib()
    dev = means3D.device
    P = int(means3D.shape[0])
    H, W = int(cot[0].shape[1]), int(cot[0].shape[2])
    M = int(shs.shape[1])
    f32 = lambda t: t.contiguous().float()  # noqa: E731
    clamped = I["clamped"]
    if clamped.ndim == 1:      # this library packs the three flags into bits 0..2
        clamped = torch.stack([(clamped >> k) & 1 for k in range(3)], 1)
    clamped = clamped.to(torch.uint8).contiguous()
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)  # noqa: E731
    g = dict(means2D=z(P, 3), conic=z(P, 4), opacity=z(P), colors=z(P, 3), depths=z(P), norm3D=z(P, 3),
             means3D=z(P, 3), cov3D=z(P, 6), sh=z(P, M, 3), scales=z(P, 3), rot=z(P, 4))
    keep = [f32(I["means2D"]), f32(I["conic_opacity"]), f32(I["rgb"]), f32(I["depths"]), f32(I["norm3D"]),
            f32(I["cov3D"]), I["ranges"].contiguous().to(torch.int32), I["point_list"].contiguous().to(torch.int32),
            I["n_contrib"].contiguous().to(torch.int32), f32(out_alpha), [f32(c) for c in cot], f32(bg),
            f32(means3D), radii.contiguous().to(torch.int32), f32(shs), f32(scales), f32(rotations), f32(viewmatrix),
            f32(projmatrix), f32(campos), f32(subpixel_offset)]
    (m2d, con, col, dep, nrm, cov, ranges, plist, ncon, alpha, c4, bgf, m3d, rad, shf, sc, rot, vm, pm, cam,
     off) = keep
    torch.cuda.synchronize(dev)
    with torch.cuda.device(dev):
        rc = L.adj_backward_f64_subpixel(
            C.c_int(P), C.c_int(int(sh_degree)), C.c_int(M), C.c_int(W), C.c_int(H), _tp(ranges), _tp(plist),
            _tp(bgf), _tp(m2d), _tp(con), _tp(col), _tp(dep), _tp(nrm), _tp(alpha), _tp(ncon), _tp(c4[0]),
            _tp(c4[1]), _tp(c4[2]), _tp(c4[3]), _tp(m3d), _tp(rad), _tp(shf), _tp(clamped), _tp(sc), _tp(rot),
            C.c_float(float(scale_modifier)), _tp(cov), _tp(vm), _tp(pm), C.c_float(float(tan_fovx)),
            C.c_float(float(tan_fovy)), C.c_float(float(kernel_size)), _tp(cam), _tp(g["means2D"]), _tp(g["conic"]),
            _tp(g["opacity"]), _tp(g["colors"]), _tp(g["depths"]), _tp(g["norm3D"]), _tp(g["means3D"]),
            _tp(g["cov3D"]), _tp(g["sh"]), _tp(g["scales"]), _tp(g["rot"]),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), _tp(off))
    if rc != 0:
        raise RuntimeError(f"adjudicator: CUDA error {rc}")
    g["opacity"] = g["opacity"].view(P, 1)
    return g
