"""The rejection matrix of the rasterizer's 13 C entry points: every argument combination below that an entry refuses
before any CUDA work, with the code it returns, the entry named in its message and the text of the check that wins.

The entries share their checks, so the table pins the order in which they run as well as the set they make.  It runs
in a child process with no visible device: a case that a change wrongly lets through then fails with SFGS_E_CUDA (or
reaches an allocator that returns NULL) instead of launching a kernel on host pointers.  Cases the entries accept,
and the camera entries' P == 0 (answered with a memset), are left out of the table."""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4


def _ptr(buf, offset=0):
    return C.addressof(buf) + offset


def _matrix():
    """{case id: [return code, message]} for every case; run with no visible device."""
    for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from sfgs import native as N
    L = N.lib()
    buf = (C.c_double * 4096)()            # host memory standing in for every device buffer; 16-byte aligned
    ptr, odd = _ptr(buf), _ptr(buf, 4)
    peer_tab = (C.c_void_p * 9)(*([ptr] * 9))
    peers = C.cast(peer_tab, C.POINTER(C.c_void_p))
    alloc = N.ALLOC_FN(lambda _u, _n: None)  # accepted calls stop at their first allocation
    none = N.ALLOC_FN()

    def fwd_base(graph):
        a = N.ForwardArgs()
        a.geom_alloc = a.binning_alloc = a.image_alloc = alloc
        a.P, a.D, a.M, a.width, a.height = 8, 3, 16, 32, 32
        for f in ("background", "means3D", "shs", "opacities", "scales", "rotations", "viewmatrix", "projmatrix",
                  "cam_pos", "out_color", "out_depth", "out_norm", "out_alpha", "radii"):
            setattr(a, f, ptr)
        a.tan_fovx = a.tan_fovy = 0.5
        a.capacity_hint = 4096 if graph else 0
        return a

    def bwd_base(kind):
        b = N.BackwardArgs()
        b.P, b.D, b.M, b.R, b.width, b.height = 8, 3, 16, 64, 32, 32
        for f in ("background", "means3D", "shs", "scales", "rotations", "viewmatrix", "projmatrix", "cam_pos",
                  "radii", "geom_buffer", "binning_buffer", "image_buffer", "accum_alphas", "dL_dpix",
                  "dL_dpix_depth", "dL_dpix_norm", "dL_dpix_alpha", "dL_dmean2D", "dL_dconic", "dL_dopacity",
                  "dL_dcolor", "dL_ddepth", "dL_dmean3D", "dL_dcov3D", "dL_dnorm3D", "dL_dsh", "dL_dscale",
                  "dL_drot"):
            setattr(b, f, ptr)
        b.tan_fovx = b.tan_fovy = 0.5
        b.scratch_alloc = alloc
        if kind == "partial":
            b.phase, b.acc, b.gauss_begin, b.gauss_end = 2, ptr, 0, 8
        return b

    def extras_fwd(a):
        a.ED, a.extra_attrs, a.out_extra = 2, ptr, ptr

    def extras_bwd(b):
        b.ED, b.extra_attrs, b.dL_dextra, b.dL_dpix_extra = 2, ptr, ptr, ptr

    def acc_peers(b, n=1, per=8, phase=1):
        b.acc_peers, b.n_peers, b.peer_slice, b.phase, b.acc = peers, n, per, phase, ptr

    def sets(**kw):
        return lambda x: [setattr(x, k, v) for k, v in kw.items()]

    # perturbations of a valid call; "entry" ones change the entry's own parameters (dict keys below)
    fwd_cases = {
        "base": sets(), "null args": None, "P<0": sets(P=-1), "P=0": sets(P=0), "width=0": sets(width=0),
        "height=0": sets(height=0), "ED<0": sets(ED=-1), "ED>max": sets(ED=35), "ED=2": extras_fwd,
        "ED=2 missing": sets(ED=2), "band<0": sets(tile_row_begin=-1), "band inverted": sets(tile_row_begin=2),
        "band": sets(tile_row_begin=1, tile_row_end=2), "out_peers": sets(out_peers=peers, n_out_peers=1),
        "out_peers n=0": sets(out_peers=peers, n_out_peers=0), "out_peers n=9": sets(out_peers=peers, n_out_peers=9),
        "out_peers no local": sets(out_peers=peers, n_out_peers=1, out_color=None),
        "null out_color": sets(out_color=None), "null radii": sets(radii=None),
        "null allocator": sets(geom_alloc=none), "null means3D": sets(means3D=None),
        "no colours": sets(shs=None), "colours precomp": sets(shs=None, colors_precomp=ptr, M=0),
        "M<(D+1)^2": sets(M=4), "D>3": sets(D=4, M=25), "no scales": sets(scales=None),
        "no scales, cov3D": sets(scales=None, cov3D_precomp=ptr), "rotations misaligned": sets(rotations=odd),
        "debug": sets(debug=1), "capacity_hint=0": sets(capacity_hint=0), "null status": "entry",
    }
    bwd_cases = {
        "base": sets(), "null args": None, "P<0": sets(P=-1), "P=0": sets(P=0), "width=0": sets(width=0),
        "ED<0": sets(ED=-1), "ED>max": sets(ED=35), "ED=2": extras_bwd, "ED=2 missing": sets(ED=2),
        "ED=2 phase 1": lambda b: (extras_bwd(b), sets(phase=1, acc=ptr)(b)),
        "acc_peers": acc_peers, "acc_peers phase 0": lambda b: acc_peers(b, phase=0),
        "acc_peers n=9": lambda b: acc_peers(b, n=9), "acc_peers short": lambda b: acc_peers(b, per=4),
        "acc_peers ED=2": lambda b: (acc_peers(b), extras_bwd(b)),
        "phase 0": sets(phase=0, acc=None), "phase 1": sets(phase=1, acc=ptr),
        "phase 2": sets(phase=2, acc=ptr, gauss_begin=0, gauss_end=8), "phase 3": sets(phase=3, acc=ptr),
        "phase -1": sets(phase=-1), "phase 1 no acc": sets(phase=1, acc=None),
        "phase 2 no acc": sets(phase=2, acc=None, gauss_begin=0, gauss_end=8),
        "phase 2 bad range": sets(phase=2, acc=ptr, gauss_begin=0, gauss_end=9),
        "null scratch buffer": sets(geom_buffer=None), "null pixel gradient": sets(dL_dpix=None),
        "null accum_alphas": sets(accum_alphas=None), "null output": sets(dL_dmean2D=None),
        "null radii": sets(radii=None), "null dL_dsh": sets(dL_dsh=None), "band<0": sets(tile_row_begin=-1),
        "band": sets(tile_row_begin=1, tile_row_end=2), "acc misaligned": sets(acc=odd),
        "rotations misaligned": sets(rotations=odd), "null scratch_alloc": sets(scratch_alloc=none),
        "null scratch_alloc, acc": sets(scratch_alloc=none, acc=ptr), "debug": sets(debug=1), "R=0": sets(R=0),
        "null camera output": "entry", "ncam=0": "entry", "ncam=35": "entry", "ncam=37": "entry", "ncam=36": "entry",
    }

    def fwd_plain(a, off, det, e):
        return L.sfgs_rasterize_forward(a)

    def fwd_off(fn):
        return lambda a, off, det, e: fn(a, off)

    def fwd_graph(a, off, det, e):
        return L.sfgs_rasterize_forward_graph(a, off, None, None if e == "null status" else ptr)

    def bwd_plain(fn):
        return lambda b, off, det, e: fn(b)

    def bwd_off(fn):
        return lambda b, off, det, e: fn(b, off)

    def bwd_camera(fn):
        return lambda b, off, det, e: fn(b, off, det, None if e == "null camera output" else ptr)

    def bwd_partial(b, off, det, e):
        ncam = int(e[5:]) if e.startswith("ncam=") else 35
        return L.sfgs_rasterize_backward_camera_partial(b, off, det, ncam, None if e == "null camera output" else ptr)

    def bwd_graph(b, off, det, e):
        ncam = int(e[5:]) if e.startswith("ncam=") else (35 if e == "null camera output" else 0)
        return L.sfgs_rasterize_backward_graph(b, off, det, None, None if e == "null camera output" else ptr, ncam)

    # entry: (call, direction, kind, takes offsets, takes deterministic)
    entries = {
        "sfgs_rasterize_forward": (fwd_plain, "fwd", "eager", False, False),
        "sfgs_rasterize_forward_subpixel": (fwd_off(L.sfgs_rasterize_forward_subpixel), "fwd", "eager", True, False),
        "sfgs_rasterize_forward_subpixel_peers": (fwd_off(L.sfgs_rasterize_forward_subpixel_peers), "fwd", "eager",
                                                  True, False),
        "sfgs_rasterize_forward_graph": (fwd_graph, "fwd", "graph", True, False),
        "sfgs_rasterize_backward": (bwd_plain(L.sfgs_rasterize_backward), "bwd", "eager", False, False),
        "sfgs_rasterize_backward_deterministic": (bwd_plain(L.sfgs_rasterize_backward_deterministic), "bwd", "eager",
                                                  False, False),
        "sfgs_rasterize_backward_subpixel": (bwd_off(L.sfgs_rasterize_backward_subpixel), "bwd", "eager", True, False),
        "sfgs_rasterize_backward_subpixel_peers": (bwd_off(L.sfgs_rasterize_backward_subpixel_peers), "bwd", "eager",
                                                   True, False),
        "sfgs_rasterize_backward_deterministic_subpixel": (bwd_off(L.sfgs_rasterize_backward_deterministic_subpixel),
                                                           "bwd", "eager", True, False),
        "sfgs_rasterize_backward_camera": (bwd_camera(L.sfgs_rasterize_backward_camera), "bwd", "camera", True, True),
        "sfgs_rasterize_backward_camera_intrinsics": (bwd_camera(L.sfgs_rasterize_backward_camera_intrinsics), "bwd",
                                                      "camera", True, True),
        "sfgs_rasterize_backward_camera_partial": (bwd_partial, "bwd", "partial", True, True),
        "sfgs_rasterize_backward_graph": (bwd_graph, "bwd", "graph", True, True),
    }
    entry_cases = {"graph": {"null status", "null camera output", "ncam=0", "ncam=35", "ncam=37", "ncam=36"},
                   "camera": {"null camera output"},
                   "partial": {"null camera output", "ncam=0", "ncam=35", "ncam=37", "ncam=36"}}
    out = {}
    for name, (call, dirn, kind, takes_off, takes_det) in entries.items():
        cases = fwd_cases if dirn == "fwd" else bwd_cases
        for case, change in cases.items():
            if change == "entry" and case not in entry_cases.get(kind, ()):
                continue
            if dirn == "fwd" and case == "null status" and kind != "graph":
                continue
            for off in ((None, ptr) if takes_off else (None,)):
                for det in ((0, 1) if takes_det else (0,)):
                    args = fwd_base(kind == "graph") if dirn == "fwd" else bwd_base(kind)
                    if callable(change):
                        change(args)
                    rc = call(None if change is None else C.byref(args), off, det, case)
                    key = f"{name[len('sfgs_rasterize_'):]} | off={int(off is not None)} det={det} | {case}"
                    out[key] = [rc, N.last_error()]
    return out


# Each outcome: (code, a substring naming the entry, the text of the winning check).
OUTCOMES = [
    (SFGS_E_BADARG, "forward", "null args"),
    (SFGS_E_BADARG, "forward", "bad sizes"),
    (SFGS_E_BADARG, "forward", "ED out of range"),
    (SFGS_E_BADARG, "forward", "extra attrs missing"),
    (SFGS_E_BADARG, "forward", "bad tile-row band"),
    (SFGS_E_BADARG, "forward", "at most 8 out_peers"),
    (SFGS_E_BADARG, "forward", "null output"),
    (SFGS_E_BADARG, "forward", "null allocator"),
    (SFGS_E_BADARG, "forward", "null input"),
    (SFGS_E_BADARG, "forward", "need shs or colors_precomp"),
    (SFGS_E_BADARG, "forward", "SH degree/M mismatch"),
    (SFGS_E_BADARG, "forward", "need scales+rotations or cov3D_precomp"),
    (SFGS_E_BADARG, "forward", "need scales+rotations or norm3D_precomp"),
    (SFGS_E_BADARG, "forward", "rotations must be 16-byte aligned"),
    (SFGS_E_UNSUPPORTED, "forward_subpixel", "extra_attrs are not supported with subpixel offsets"),
    (SFGS_E_UNSUPPORTED, "forward_subpixel",
     "out_peers are not supported by this entry; use sfgs_rasterize_forward_subpixel_peers"),
    (SFGS_E_BADARG, "forward_graph", "null args"),
    (SFGS_E_UNSUPPORTED, "forward_graph", "extra_attrs are not supported with subpixel offsets"),
    (SFGS_E_UNSUPPORTED, "forward_graph", "tile-row bands are not supported under graph capture"),
    (SFGS_E_UNSUPPORTED, "forward_graph", "out_peers are not supported under graph capture"),
    (SFGS_E_BADARG, "forward_graph", "debug synchronises after every stage and cannot be captured"),
    (SFGS_E_BADARG, "forward_graph", "capacity_hint must be > 0 (the binning capacity of the captured frame)"),
    (SFGS_E_BADARG, "forward_graph", "null status word"),
    (SFGS_E_BADARG, "backward", "null args"),
    (SFGS_E_BADARG, "backward", "bad sizes"),
    (SFGS_E_BADARG, "backward", "ED out of range"),
    (SFGS_E_BADARG, "backward", "extra attrs missing"),
    (SFGS_E_UNSUPPORTED, "backward", "extra_attrs are not supported by the two-phase backward"),
    (SFGS_E_BADARG, "backward", "acc_peers needs phase 1, 1..8 peers and n_peers*peer_slice >= P"),
    (SFGS_E_BADARG, "backward", "phase must be 0, 1 or 2"),
    (SFGS_E_BADARG, "backward", "phases 1 and 2 need the caller's acc buffer"),
    (SFGS_E_BADARG, "backward", "bad Gaussian range"),
    (SFGS_E_BADARG, "backward", "null scratch buffer"),
    (SFGS_E_BADARG, "backward", "null pixel gradient"),
    (SFGS_E_BADARG, "backward", "null output"),
    (SFGS_E_BADARG, "backward", "radii missing"),
    (SFGS_E_BADARG, "backward", "dL_dsh missing"),
    (SFGS_E_BADARG, "backward", "bad tile-row band"),
    (SFGS_E_BADARG, "backward", "acc must be 16-byte aligned"),
    (SFGS_E_BADARG, "backward", "rotations must be 16-byte aligned"),
    (SFGS_E_BADARG, "backward", "null scratch allocator"),
    (SFGS_E_UNSUPPORTED, "backward_deterministic", "extra_attrs have no deterministic implementation"),
    (SFGS_E_UNSUPPORTED, "backward_deterministic",
     "acc_peers (system-scope reductions) have no deterministic implementation"),
    (SFGS_E_BADARG, "backward_deterministic", "null scratch allocator"),
    (SFGS_E_UNSUPPORTED, "backward_subpixel", "extra_attrs are not supported with subpixel offsets"),
    (SFGS_E_UNSUPPORTED, "backward_subpixel",
     "acc_peers are not supported by this entry; use sfgs_rasterize_backward_subpixel_peers"),
    (SFGS_E_UNSUPPORTED, "backward", "extra_attrs are not supported with subpixel offsets"),
    (SFGS_E_UNSUPPORTED, "backward",
     "acc_peers are not supported by this entry; use sfgs_rasterize_backward_subpixel_peers"),
    (SFGS_E_BADARG, "backward_camera", "null args"),
    (SFGS_E_UNSUPPORTED, "backward", "extra_attrs have no deterministic implementation"),
    (SFGS_E_UNSUPPORTED, "backward_camera", "camera gradients are formed by the one-call backward (phase 0) only"),
    (SFGS_E_UNSUPPORTED, "backward_camera", "acc_peers (the multi-GPU backward) have no camera gradients"),
    (SFGS_E_BADARG, "backward_camera", "null scratch allocator"),
    (SFGS_E_BADARG, "backward_camera", "null dL_dcamera"),
    (SFGS_E_BADARG, "backward_camera_intrinsics", "null args"),
    (SFGS_E_UNSUPPORTED, "backward_camera_intrinsics",
     "camera gradients are formed by the one-call backward (phase 0) only"),
    (SFGS_E_UNSUPPORTED, "backward_camera_intrinsics", "acc_peers (the multi-GPU backward) have no camera gradients"),
    (SFGS_E_BADARG, "backward_camera_intrinsics", "null scratch allocator"),
    (SFGS_E_BADARG, "backward_camera_intrinsics", "null dL_dcamera"),
    (SFGS_E_BADARG, "backward_camera_partial", "null args"),
    (SFGS_E_UNSUPPORTED, "backward_camera_partial", "extra_attrs are not supported by the two-phase backward"),
    (SFGS_E_UNSUPPORTED, "backward_camera_partial", "camera partials are formed by phase 2 only"),
    (SFGS_E_BADARG, "backward_camera_partial", "null scratch allocator"),
    (SFGS_E_BADARG, "backward_camera_partial", "null dL_dcamera_partial"),
    (SFGS_E_BADARG, "backward_camera_partial", "ncam must be 35 or 37"),
    (SFGS_E_BADARG, "backward_graph", "null args"),
    (SFGS_E_UNSUPPORTED, "backward_graph", "extra_attrs are not supported with subpixel offsets"),
    (SFGS_E_UNSUPPORTED, "backward_graph",
     "phases 1 and 2 (the two-phase backward) are not supported under graph capture"),
    (SFGS_E_UNSUPPORTED, "backward_graph", "acc_peers are not supported under graph capture"),
    (SFGS_E_UNSUPPORTED, "backward_graph", "tile-row bands are not supported under graph capture"),
    (SFGS_E_BADARG, "backward_graph", "debug synchronises after every stage and cannot be captured"),
    (SFGS_E_BADARG, "backward_graph", "R must be the forward's binning capacity (> 0)"),
    (SFGS_E_BADARG, "backward_graph", "null dL_dcamera"),
    (SFGS_E_BADARG, "backward_graph", "ncam must be 0, 35 or 37"),
]
# {entry | offsets given, deterministic argument: {case: outcome}}, taken from the entry points as they were
# before their checks moved into one function per direction
REJECTED = {
    "forward | off=0 det=0": {
        "null args": 0, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 2, "ED=2 missing": 3, "band<0": 4,
        "band inverted": 4, "out_peers n=9": 5, "null out_color": 6, "null radii": 6, "null allocator": 7,
        "null means3D": 8, "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11, "no scales, cov3D": 12,
        "rotations misaligned": 13,
    },
    "forward_subpixel | off=0 det=0": {
        "null args": 0, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 2, "ED=2 missing": 3, "band<0": 4,
        "band inverted": 4, "out_peers n=9": 5, "null out_color": 6, "null radii": 6, "null allocator": 7,
        "null means3D": 8, "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11, "no scales, cov3D": 12,
        "rotations misaligned": 13,
    },
    "forward_subpixel | off=1 det=0": {
        "null args": 0, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 14, "ED=2": 14,
        "ED=2 missing": 14, "band<0": 4, "band inverted": 4, "out_peers": 15, "out_peers n=0": 15,
        "out_peers n=9": 15, "out_peers no local": 15, "null out_color": 6, "null radii": 6, "null allocator": 7,
        "null means3D": 8, "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11, "no scales, cov3D": 12,
        "rotations misaligned": 13,
    },
    "forward_subpixel_peers | off=0 det=0": {
        "null args": 0, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 2, "ED=2 missing": 3, "band<0": 4,
        "band inverted": 4, "out_peers n=9": 5, "null out_color": 6, "null radii": 6, "null allocator": 7,
        "null means3D": 8, "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11, "no scales, cov3D": 12,
        "rotations misaligned": 13,
    },
    "forward_subpixel_peers | off=1 det=0": {
        "null args": 0, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 14, "ED=2": 14,
        "ED=2 missing": 14, "band<0": 4, "band inverted": 4, "out_peers n=9": 5, "null out_color": 6, "null radii": 6,
        "null allocator": 7, "null means3D": 8, "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11,
        "no scales, cov3D": 12, "rotations misaligned": 13,
    },
    "forward_graph | off=0 det=0": {
        "null args": 16, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 2, "ED=2 missing": 3,
        "band<0": 18, "band inverted": 18, "band": 18, "out_peers": 19, "out_peers n=0": 19, "out_peers n=9": 19,
        "out_peers no local": 19, "null out_color": 6, "null radii": 6, "null allocator": 7, "null means3D": 8,
        "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11, "no scales, cov3D": 12,
        "rotations misaligned": 13, "debug": 20, "capacity_hint=0": 21, "null status": 22,
    },
    "forward_graph | off=1 det=0": {
        "null args": 16, "P<0": 1, "width=0": 1, "height=0": 1, "ED<0": 2, "ED>max": 17, "ED=2": 17,
        "ED=2 missing": 17, "band<0": 18, "band inverted": 18, "band": 18, "out_peers": 19, "out_peers n=0": 19,
        "out_peers n=9": 19, "out_peers no local": 19, "null out_color": 6, "null radii": 6, "null allocator": 7,
        "null means3D": 8, "no colours": 9, "M<(D+1)^2": 10, "D>3": 10, "no scales": 11, "no scales, cov3D": 12,
        "rotations misaligned": 13, "debug": 20, "capacity_hint=0": 21, "null status": 22,
    },
    "backward | off=0 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 25, "ED=2 missing": 26, "ED=2 phase 1": 27,
        "acc_peers phase 0": 28, "acc_peers n=9": 28, "acc_peers short": 28, "acc_peers ED=2": 27, "phase 3": 29,
        "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30, "phase 2 bad range": 31,
        "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33, "null output": 34,
        "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39,
        "null scratch_alloc": 40,
    },
    "backward_deterministic | off=0 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 41, "ED=2": 41, "ED=2 missing": 41,
        "ED=2 phase 1": 41, "acc_peers": 42, "acc_peers phase 0": 42, "acc_peers n=9": 42, "acc_peers short": 42,
        "acc_peers ED=2": 42, "phase 3": 29, "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30,
        "phase 2 bad range": 31, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 40, "null scratch_alloc, acc": 43,
    },
    "backward_subpixel | off=0 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 25, "ED=2 missing": 26, "ED=2 phase 1": 27,
        "acc_peers phase 0": 28, "acc_peers n=9": 28, "acc_peers short": 28, "acc_peers ED=2": 27, "phase 3": 29,
        "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30, "phase 2 bad range": 31,
        "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33, "null output": 34,
        "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39,
        "null scratch_alloc": 40,
    },
    "backward_subpixel | off=1 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 44, "ED=2": 44, "ED=2 missing": 44,
        "ED=2 phase 1": 44, "acc_peers": 45, "acc_peers phase 0": 45, "acc_peers n=9": 45, "acc_peers short": 45,
        "acc_peers ED=2": 44, "phase 3": 29, "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30,
        "phase 2 bad range": 31, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 40,
    },
    "backward_subpixel_peers | off=0 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 25, "ED=2 missing": 26, "ED=2 phase 1": 27,
        "acc_peers phase 0": 28, "acc_peers n=9": 28, "acc_peers short": 28, "acc_peers ED=2": 27, "phase 3": 29,
        "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30, "phase 2 bad range": 31,
        "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33, "null output": 34,
        "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39,
        "null scratch_alloc": 40,
    },
    "backward_subpixel_peers | off=1 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 44, "ED=2": 44, "ED=2 missing": 44,
        "ED=2 phase 1": 44, "acc_peers phase 0": 28, "acc_peers n=9": 28, "acc_peers short": 28, "acc_peers ED=2": 44,
        "phase 3": 29, "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30, "phase 2 bad range": 31,
        "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33, "null output": 34,
        "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39,
        "null scratch_alloc": 40,
    },
    "backward_deterministic_subpixel | off=0 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 41, "ED=2": 41, "ED=2 missing": 41,
        "ED=2 phase 1": 41, "acc_peers": 42, "acc_peers phase 0": 42, "acc_peers n=9": 42, "acc_peers short": 42,
        "acc_peers ED=2": 42, "phase 3": 29, "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30,
        "phase 2 bad range": 31, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 40, "null scratch_alloc, acc": 43,
    },
    "backward_deterministic_subpixel | off=1 det=0": {
        "null args": 23, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 46, "ED=2": 46, "ED=2 missing": 46,
        "ED=2 phase 1": 46, "acc_peers": 47, "acc_peers phase 0": 47, "acc_peers n=9": 47, "acc_peers short": 47,
        "acc_peers ED=2": 46, "phase 3": 29, "phase -1": 29, "phase 1 no acc": 30, "phase 2 no acc": 30,
        "phase 2 bad range": 31, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 40, "null scratch_alloc, acc": 43,
    },
    "backward_camera | off=0 det=0": {
        "null args": 48, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 25, "ED=2 missing": 26, "ED=2 phase 1": 50,
        "acc_peers": 50, "acc_peers phase 0": 51, "acc_peers n=9": 50, "acc_peers short": 50, "acc_peers ED=2": 50,
        "phase 1": 50, "phase 2": 50, "phase 3": 50, "phase -1": 50, "phase 1 no acc": 50, "phase 2 no acc": 50,
        "phase 2 bad range": 50, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 52, "null scratch_alloc, acc": 52, "null camera output": 53,
    },
    "backward_camera | off=0 det=1": {
        "null args": 48, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 49, "ED=2": 49, "ED=2 missing": 49,
        "ED=2 phase 1": 50, "acc_peers": 50, "acc_peers phase 0": 51, "acc_peers n=9": 50, "acc_peers short": 50,
        "acc_peers ED=2": 50, "phase 1": 50, "phase 2": 50, "phase 3": 50, "phase -1": 50, "phase 1 no acc": 50,
        "phase 2 no acc": 50, "phase 2 bad range": 50, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 52, "null scratch_alloc, acc": 52,
        "null camera output": 53,
    },
    "backward_camera | off=1 det=0": {
        "null args": 48, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 46, "ED=2": 46, "ED=2 missing": 46,
        "ED=2 phase 1": 50, "acc_peers": 50, "acc_peers phase 0": 51, "acc_peers n=9": 50, "acc_peers short": 50,
        "acc_peers ED=2": 50, "phase 1": 50, "phase 2": 50, "phase 3": 50, "phase -1": 50, "phase 1 no acc": 50,
        "phase 2 no acc": 50, "phase 2 bad range": 50, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 52, "null scratch_alloc, acc": 52,
        "null camera output": 53,
    },
    "backward_camera | off=1 det=1": {
        "null args": 48, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 46, "ED=2": 46, "ED=2 missing": 46,
        "ED=2 phase 1": 50, "acc_peers": 50, "acc_peers phase 0": 51, "acc_peers n=9": 50, "acc_peers short": 50,
        "acc_peers ED=2": 50, "phase 1": 50, "phase 2": 50, "phase 3": 50, "phase -1": 50, "phase 1 no acc": 50,
        "phase 2 no acc": 50, "phase 2 bad range": 50, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 52, "null scratch_alloc, acc": 52,
        "null camera output": 53,
    },
    "backward_camera_intrinsics | off=0 det=0": {
        "null args": 54, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 25, "ED=2 missing": 26, "ED=2 phase 1": 55,
        "acc_peers": 55, "acc_peers phase 0": 56, "acc_peers n=9": 55, "acc_peers short": 55, "acc_peers ED=2": 55,
        "phase 1": 55, "phase 2": 55, "phase 3": 55, "phase -1": 55, "phase 1 no acc": 55, "phase 2 no acc": 55,
        "phase 2 bad range": 55, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 57, "null scratch_alloc, acc": 57, "null camera output": 58,
    },
    "backward_camera_intrinsics | off=0 det=1": {
        "null args": 54, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 49, "ED=2": 49, "ED=2 missing": 49,
        "ED=2 phase 1": 55, "acc_peers": 55, "acc_peers phase 0": 56, "acc_peers n=9": 55, "acc_peers short": 55,
        "acc_peers ED=2": 55, "phase 1": 55, "phase 2": 55, "phase 3": 55, "phase -1": 55, "phase 1 no acc": 55,
        "phase 2 no acc": 55, "phase 2 bad range": 55, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 57, "null scratch_alloc, acc": 57,
        "null camera output": 58,
    },
    "backward_camera_intrinsics | off=1 det=0": {
        "null args": 54, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 46, "ED=2": 46, "ED=2 missing": 46,
        "ED=2 phase 1": 55, "acc_peers": 55, "acc_peers phase 0": 56, "acc_peers n=9": 55, "acc_peers short": 55,
        "acc_peers ED=2": 55, "phase 1": 55, "phase 2": 55, "phase 3": 55, "phase -1": 55, "phase 1 no acc": 55,
        "phase 2 no acc": 55, "phase 2 bad range": 55, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 57, "null scratch_alloc, acc": 57,
        "null camera output": 58,
    },
    "backward_camera_intrinsics | off=1 det=1": {
        "null args": 54, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 46, "ED=2": 46, "ED=2 missing": 46,
        "ED=2 phase 1": 55, "acc_peers": 55, "acc_peers phase 0": 56, "acc_peers n=9": 55, "acc_peers short": 55,
        "acc_peers ED=2": 55, "phase 1": 55, "phase 2": 55, "phase 3": 55, "phase -1": 55, "phase 1 no acc": 55,
        "phase 2 no acc": 55, "phase 2 bad range": 55, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 37,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 57, "null scratch_alloc, acc": 57,
        "null camera output": 58,
    },
    "backward_camera_partial | off=0 det=0": {
        "null args": 59, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 60, "ED=2": 60, "ED=2 missing": 60,
        "ED=2 phase 1": 61, "acc_peers": 61, "acc_peers phase 0": 61, "acc_peers n=9": 61, "acc_peers short": 61,
        "acc_peers ED=2": 61, "phase 0": 61, "phase 1": 61, "phase 3": 61, "phase -1": 61, "phase 1 no acc": 61,
        "phase 2 no acc": 30, "phase 2 bad range": 31, "null scratch buffer": 32, "null output": 34, "null radii": 35,
        "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 62,
        "null scratch_alloc, acc": 62, "null camera output": 63, "ncam=0": 64, "ncam=36": 64,
    },
    "backward_camera_partial | off=0 det=1": {
        "null args": 59, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 60, "ED=2": 60, "ED=2 missing": 60,
        "ED=2 phase 1": 61, "acc_peers": 61, "acc_peers phase 0": 61, "acc_peers n=9": 61, "acc_peers short": 61,
        "acc_peers ED=2": 61, "phase 0": 61, "phase 1": 61, "phase 3": 61, "phase -1": 61, "phase 1 no acc": 61,
        "phase 2 no acc": 30, "phase 2 bad range": 31, "null scratch buffer": 32, "null output": 34, "null radii": 35,
        "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 62,
        "null scratch_alloc, acc": 62, "null camera output": 63, "ncam=0": 64, "ncam=36": 64,
    },
    "backward_camera_partial | off=1 det=0": {
        "null args": 59, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 60, "ED=2": 60, "ED=2 missing": 60,
        "ED=2 phase 1": 61, "acc_peers": 61, "acc_peers phase 0": 61, "acc_peers n=9": 61, "acc_peers short": 61,
        "acc_peers ED=2": 61, "phase 0": 61, "phase 1": 61, "phase 3": 61, "phase -1": 61, "phase 1 no acc": 61,
        "phase 2 no acc": 30, "phase 2 bad range": 31, "null scratch buffer": 32, "null output": 34, "null radii": 35,
        "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 62,
        "null scratch_alloc, acc": 62, "null camera output": 63, "ncam=0": 64, "ncam=36": 64,
    },
    "backward_camera_partial | off=1 det=1": {
        "null args": 59, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 60, "ED=2": 60, "ED=2 missing": 60,
        "ED=2 phase 1": 61, "acc_peers": 61, "acc_peers phase 0": 61, "acc_peers n=9": 61, "acc_peers short": 61,
        "acc_peers ED=2": 61, "phase 0": 61, "phase 1": 61, "phase 3": 61, "phase -1": 61, "phase 1 no acc": 61,
        "phase 2 no acc": 30, "phase 2 bad range": 31, "null scratch buffer": 32, "null output": 34, "null radii": 35,
        "null dL_dsh": 36, "band<0": 37, "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 62,
        "null scratch_alloc, acc": 62, "null camera output": 63, "ncam=0": 64, "ncam=36": 64,
    },
    "backward_graph | off=0 det=0": {
        "null args": 65, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 25, "ED=2 missing": 26, "ED=2 phase 1": 67,
        "acc_peers": 67, "acc_peers phase 0": 68, "acc_peers n=9": 67, "acc_peers short": 67, "acc_peers ED=2": 67,
        "phase 1": 67, "phase 2": 67, "phase 3": 67, "phase -1": 67, "phase 1 no acc": 67, "phase 2 no acc": 67,
        "phase 2 bad range": 67, "null scratch buffer": 32, "null pixel gradient": 33, "null accum_alphas": 33,
        "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 69, "band": 69, "acc misaligned": 38,
        "rotations misaligned": 39, "null scratch_alloc": 40, "debug": 70, "R=0": 71, "null camera output": 72,
        "ncam=36": 73,
    },
    "backward_graph | off=0 det=1": {
        "null args": 65, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 49, "ED=2": 49, "ED=2 missing": 49,
        "ED=2 phase 1": 67, "acc_peers": 67, "acc_peers phase 0": 68, "acc_peers n=9": 67, "acc_peers short": 67,
        "acc_peers ED=2": 67, "phase 1": 67, "phase 2": 67, "phase 3": 67, "phase -1": 67, "phase 1 no acc": 67,
        "phase 2 no acc": 67, "phase 2 bad range": 67, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 69, "band": 69,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 40, "null scratch_alloc, acc": 40,
        "debug": 70, "R=0": 71, "null camera output": 72, "ncam=36": 73,
    },
    "backward_graph | off=1 det=0": {
        "null args": 65, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 66, "ED=2": 66, "ED=2 missing": 66,
        "ED=2 phase 1": 67, "acc_peers": 67, "acc_peers phase 0": 68, "acc_peers n=9": 67, "acc_peers short": 67,
        "acc_peers ED=2": 67, "phase 1": 67, "phase 2": 67, "phase 3": 67, "phase -1": 67, "phase 1 no acc": 67,
        "phase 2 no acc": 67, "phase 2 bad range": 67, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 69, "band": 69,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 40, "debug": 70, "R=0": 71,
        "null camera output": 72, "ncam=36": 73,
    },
    "backward_graph | off=1 det=1": {
        "null args": 65, "P<0": 24, "width=0": 24, "ED<0": 25, "ED>max": 66, "ED=2": 66, "ED=2 missing": 66,
        "ED=2 phase 1": 67, "acc_peers": 67, "acc_peers phase 0": 68, "acc_peers n=9": 67, "acc_peers short": 67,
        "acc_peers ED=2": 67, "phase 1": 67, "phase 2": 67, "phase 3": 67, "phase -1": 67, "phase 1 no acc": 67,
        "phase 2 no acc": 67, "phase 2 bad range": 67, "null scratch buffer": 32, "null pixel gradient": 33,
        "null accum_alphas": 33, "null output": 34, "null radii": 35, "null dL_dsh": 36, "band<0": 69, "band": 69,
        "acc misaligned": 38, "rotations misaligned": 39, "null scratch_alloc": 40, "null scratch_alloc, acc": 40,
        "debug": 70, "R=0": 71, "null camera output": 72, "ncam=36": 73,
    },
}
EXPECTED = {f"{g} | {case}": i for g, cases in REJECTED.items() for case, i in cases.items()}


def test_entry_rejection_matrix():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout)
    rejected = {k for k, (rc, _) in got.items() if rc in (SFGS_E_BADARG, SFGS_E_UNSUPPORTED)}
    assert sorted(rejected - set(EXPECTED)) == [], "newly rejected"
    assert sorted(set(EXPECTED) - rejected) == [], [(k, got.get(k)) for k in sorted(set(EXPECTED) - rejected)]
    for key, i in EXPECTED.items():
        code, entry, what = OUTCOMES[i]
        rc, msg = got[key]
        assert rc == code and entry in msg and what in msg, (key, rc, msg, OUTCOMES[i])


if __name__ == "__main__":
    print(json.dumps(_matrix()))
