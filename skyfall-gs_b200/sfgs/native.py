"""ctypes binding of libsfgs.so (the C ABI declared in include/sfgs.h).

The structures below mirror `sfgs_forward_args` / `sfgs_backward_args` field
for field.  Nothing here falls back to another implementation: if the shared
library is missing or does not load, importing the ops raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libsfgs.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)

c_float_p = C.c_void_p  # raw device pointers travel as integers
c_int_p = C.c_void_p


class ForwardArgs(C.Structure):
    _fields_ = [
        ("geom_alloc", ALLOC_FN), ("geom_user", C.c_void_p),
        ("binning_alloc", ALLOC_FN), ("binning_user", C.c_void_p),
        ("image_alloc", ALLOC_FN), ("image_user", C.c_void_p),
        ("P", C.c_int), ("D", C.c_int), ("M", C.c_int), ("ED", C.c_int),
        ("width", C.c_int), ("height", C.c_int),
        ("background", c_float_p), ("means3D", c_float_p), ("shs", c_float_p),
        ("colors_precomp", c_float_p), ("opacities", c_float_p), ("scales", c_float_p),
        ("scale_modifier", C.c_float),
        ("rotations", c_float_p), ("cov3D_precomp", c_float_p), ("norm3D_precomp", c_float_p),
        ("extra_attrs", c_float_p), ("viewmatrix", c_float_p), ("projmatrix", c_float_p),
        ("cam_pos", c_float_p),
        ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("kernel_size", C.c_float),
        ("prefiltered", C.c_int),
        ("out_color", c_float_p), ("out_depth", c_float_p), ("out_norm", c_float_p),
        ("out_alpha", c_float_p), ("out_extra", c_float_p), ("radii", c_int_p),
        ("debug", C.c_int), ("stream", C.c_void_p), ("capacity_hint", C.c_longlong),
        ("tile_row_begin", C.c_int), ("tile_row_end", C.c_int),
        ("out_norm_raw", c_float_p),
        ("out_peers", C.POINTER(C.c_void_p)), ("n_out_peers", C.c_int),
    ]


class BackwardArgs(C.Structure):
    _fields_ = [
        ("P", C.c_int), ("D", C.c_int), ("M", C.c_int), ("R", C.c_int), ("ED", C.c_int),
        ("width", C.c_int), ("height", C.c_int),
        ("background", c_float_p), ("means3D", c_float_p), ("shs", c_float_p),
        ("colors_precomp", c_float_p), ("scales", c_float_p),
        ("scale_modifier", C.c_float),
        ("rotations", c_float_p), ("cov3D_precomp", c_float_p), ("norm3D_precomp", c_float_p),
        ("extra_attrs", c_float_p), ("viewmatrix", c_float_p), ("projmatrix", c_float_p),
        ("cam_pos", c_float_p),
        ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("kernel_size", C.c_float),
        ("radii", c_int_p),
        ("geom_buffer", C.c_void_p), ("binning_buffer", C.c_void_p), ("image_buffer", C.c_void_p),
        ("accum_alphas", c_float_p), ("dL_dpix", c_float_p), ("dL_dpix_depth", c_float_p),
        ("dL_dpix_norm", c_float_p), ("dL_dpix_alpha", c_float_p), ("dL_dpix_extra", c_float_p),
        ("dL_dmean2D", c_float_p), ("dL_dconic", c_float_p), ("dL_dopacity", c_float_p),
        ("dL_dcolor", c_float_p), ("dL_ddepth", c_float_p), ("dL_dmean3D", c_float_p),
        ("dL_dcov3D", c_float_p), ("dL_dnorm3D", c_float_p), ("dL_dsh", c_float_p),
        ("dL_dscale", c_float_p), ("dL_drot", c_float_p), ("dL_dextra", c_float_p),
        ("scratch_alloc", ALLOC_FN), ("scratch_user", C.c_void_p),
        ("debug", C.c_int), ("stream", C.c_void_p),
        ("tile_row_begin", C.c_int), ("tile_row_end", C.c_int),
        ("norm_raw", c_float_p),
        ("phase", C.c_int), ("acc", c_float_p), ("gauss_begin", C.c_int), ("gauss_end", C.c_int),
        ("acc_peers", C.POINTER(C.c_void_p)), ("n_peers", C.c_int), ("peer_slice", C.c_int),
    ]


class GeomView(C.Structure):
    _fields_ = [("rec", C.c_void_p), ("cov3D", C.c_void_p), ("clamped", C.c_void_p), ("tiles_touched", C.c_void_p)]


class ImageView(C.Structure):
    _fields_ = [("n_contrib", C.c_void_p), ("ranges", C.c_void_p), ("tile_count", C.c_void_p)]


class BinningView(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("point_list", C.c_void_p)]


# every symbol include/sfgs.h declares
ABI_VERSION = 4   # SFGS_VERSION of include/sfgs.h these struct mirrors were written for

EXPORTS = [
    "sfgs_rasterize_forward", "sfgs_rasterize_backward", "sfgs_rasterize_backward_deterministic", "sfgs_mark_visible",
    "sfgs_rasterize_forward_subpixel", "sfgs_rasterize_backward_subpixel", "sfgs_rasterize_backward_deterministic_subpixel",
    "sfgs_rasterize_forward_subpixel_peers", "sfgs_rasterize_backward_subpixel_peers",
    "sfgs_rasterize_backward_camera", "sfgs_rasterize_backward_camera_intrinsics", "sfgs_rasterize_backward_camera_partial",
    "sfgs_geom_bytes", "sfgs_image_bytes", "sfgs_binning_bytes",
    "sfgs_geom_layout", "sfgs_image_layout", "sfgs_binning_layout", "sfgs_last_capacity",
    "sfgs_fusedssim_forward", "sfgs_fusedssim_backward", "sfgs_dist2_knn3",
    "sfgs_activations_forward", "sfgs_activations_backward",
    "sfgs_last_error", "sfgs_version", "sfgs_launch_count", "sfgs_profile_enable", "sfgs_profile_read", "sfgs_sizeof", "sfgs_sm_clock_probe",
    "sfgs_selftest_expf", "sfgs_overflow_reruns", "sfgs_appearance_forward", "sfgs_appearance_backward",
    "sfgs_appearance_backward_scratch_bytes", "sfgs_compute_3d_filter",
    "sfgs_densification_stats", "sfgs_densify_plan_blocks", "sfgs_densify_plan", "sfgs_densify_apply",
]
STAGE_NAMES = ["fwd_zero", "preprocess", "tile_scan", "emit_keys", "tile_sort", "render_fwd", "bwd_zero", "render_bwd",
               "gauss_bwd", "bwd_order"]

_lib = None


def lib() -> C.CDLL:
    """Load libsfgs.so (once). Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python skyfall-gs_b200/build.py` "
            "(or __graft_entry__.build()). There is no fallback implementation.")
    L = C.CDLL(LIB_PATH)
    L.sfgs_rasterize_forward.argtypes = [C.POINTER(ForwardArgs)]
    L.sfgs_rasterize_forward.restype = C.c_int
    L.sfgs_rasterize_backward.argtypes = [C.POINTER(BackwardArgs)]
    L.sfgs_rasterize_backward.restype = C.c_int
    L.sfgs_rasterize_backward_deterministic.argtypes = [C.POINTER(BackwardArgs)]
    L.sfgs_rasterize_backward_deterministic.restype = C.c_int
    L.sfgs_rasterize_forward_subpixel.argtypes = [C.POINTER(ForwardArgs), C.c_void_p]
    L.sfgs_rasterize_forward_subpixel.restype = C.c_int
    L.sfgs_rasterize_backward_subpixel.argtypes = [C.POINTER(BackwardArgs), C.c_void_p]
    L.sfgs_rasterize_backward_subpixel.restype = C.c_int
    L.sfgs_rasterize_backward_deterministic_subpixel.argtypes = [C.POINTER(BackwardArgs), C.c_void_p]
    L.sfgs_rasterize_backward_deterministic_subpixel.restype = C.c_int
    L.sfgs_rasterize_forward_subpixel_peers.argtypes = [C.POINTER(ForwardArgs), C.c_void_p]
    L.sfgs_rasterize_forward_subpixel_peers.restype = C.c_int
    L.sfgs_rasterize_backward_subpixel_peers.argtypes = [C.POINTER(BackwardArgs), C.c_void_p]
    L.sfgs_rasterize_backward_subpixel_peers.restype = C.c_int
    L.sfgs_rasterize_backward_camera.argtypes = [C.POINTER(BackwardArgs), C.c_void_p, C.c_int, C.c_void_p]
    L.sfgs_rasterize_backward_camera.restype = C.c_int
    L.sfgs_rasterize_backward_camera_intrinsics.argtypes = [C.POINTER(BackwardArgs), C.c_void_p, C.c_int, C.c_void_p]
    L.sfgs_rasterize_backward_camera_intrinsics.restype = C.c_int
    L.sfgs_rasterize_backward_camera_partial.argtypes = [C.POINTER(BackwardArgs), C.c_void_p, C.c_int, C.c_int,
                                                         C.c_void_p]
    L.sfgs_rasterize_backward_camera_partial.restype = C.c_int
    L.sfgs_mark_visible.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.sfgs_mark_visible.restype = C.c_int
    L.sfgs_geom_bytes.argtypes = [C.c_int]; L.sfgs_geom_bytes.restype = C.c_size_t
    L.sfgs_image_bytes.argtypes = [C.c_int, C.c_int]; L.sfgs_image_bytes.restype = C.c_size_t
    L.sfgs_binning_bytes.argtypes = [C.c_longlong]; L.sfgs_binning_bytes.restype = C.c_size_t
    L.sfgs_geom_layout.argtypes = [C.c_void_p, C.c_int, C.POINTER(GeomView)]; L.sfgs_geom_layout.restype = C.c_int
    L.sfgs_image_layout.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(ImageView)]; L.sfgs_image_layout.restype = C.c_int
    L.sfgs_binning_layout.argtypes = [C.c_void_p, C.c_longlong, C.POINTER(BinningView)]; L.sfgs_binning_layout.restype = C.c_int
    L.sfgs_last_capacity.argtypes = []; L.sfgs_last_capacity.restype = C.c_longlong
    L.sfgs_overflow_reruns.argtypes = []; L.sfgs_overflow_reruns.restype = C.c_longlong
    L.sfgs_fusedssim_forward.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.sfgs_fusedssim_forward.restype = C.c_int
    L.sfgs_fusedssim_backward.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.sfgs_fusedssim_backward.restype = C.c_int
    L.sfgs_dist2_knn3.argtypes = [C.c_int, C.c_void_p, C.c_void_p, ALLOC_FN, C.c_void_p, C.c_void_p]
    L.sfgs_dist2_knn3.restype = C.c_int
    L.sfgs_activations_forward.argtypes = [C.c_int] + [C.c_void_p] * 8
    L.sfgs_activations_forward.restype = C.c_int
    L.sfgs_activations_backward.argtypes = [C.c_int] + [C.c_void_p] * 11
    L.sfgs_activations_backward.restype = C.c_int
    L.sfgs_last_error.argtypes = []; L.sfgs_last_error.restype = C.c_char_p
    L.sfgs_version.argtypes = []; L.sfgs_version.restype = C.c_int
    if L.sfgs_version() != ABI_VERSION:
        raise ImportError(f"{LIB_PATH} has ABI v{L.sfgs_version()}, these bindings expect v{ABI_VERSION}: rebuild it")
    L.sfgs_launch_count.argtypes = []; L.sfgs_launch_count.restype = C.c_longlong
    L.sfgs_sizeof.argtypes = [C.c_int]; L.sfgs_sizeof.restype = C.c_size_t
    L.sfgs_sm_clock_probe.argtypes = [C.c_void_p, C.c_void_p]; L.sfgs_sm_clock_probe.restype = C.c_int
    L.sfgs_appearance_forward.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 10
    L.sfgs_appearance_forward.restype = C.c_int
    L.sfgs_appearance_backward.argtypes = ([C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
                                           + [C.c_void_p] * 20 + [ALLOC_FN, C.c_void_p, C.c_void_p])
    L.sfgs_appearance_backward.restype = C.c_int
    L.sfgs_appearance_backward_scratch_bytes.argtypes = [C.c_int]
    L.sfgs_appearance_backward_scratch_bytes.restype = C.c_size_t
    L.sfgs_compute_3d_filter.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    L.sfgs_compute_3d_filter.restype = C.c_int
    L.sfgs_densification_stats.argtypes = [C.c_int] + [C.c_void_p] * 8
    L.sfgs_densification_stats.restype = C.c_int
    L.sfgs_densify_plan_blocks.argtypes = [C.c_int]; L.sfgs_densify_plan_blocks.restype = C.c_int
    L.sfgs_densify_plan.argtypes = ([C.c_int] + [C.c_void_p] * 5 + [C.c_float, C.c_void_p, C.c_float, C.c_float, C.c_int,
                                    C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p])
    L.sfgs_densify_plan.restype = C.c_int
    L.sfgs_densify_apply.argtypes = ([C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_int, C.POINTER(C.c_int)]
                                     + [C.POINTER(C.c_void_p)] * 6 + [C.c_void_p])
    L.sfgs_densify_apply.restype = C.c_int
    L.sfgs_selftest_expf.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.sfgs_selftest_expf.restype = C.c_int
    L.sfgs_profile_enable.argtypes = [C.c_int]; L.sfgs_profile_enable.restype = C.c_int
    L.sfgs_profile_read.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.c_int]
    L.sfgs_profile_read.restype = C.c_int
    for which, st in enumerate((ForwardArgs, BackwardArgs, GeomView, ImageView, BinningView)):
        if L.sfgs_sizeof(which) != C.sizeof(st):
            raise ImportError(f"ABI mismatch: {st.__name__} is {C.sizeof(st)} bytes here, {L.sfgs_sizeof(which)} in {LIB_PATH}")
    _lib = L
    return L


def profile_enable(on: bool) -> None:
    lib().sfgs_profile_enable(1 if on else 0)


def profile_read() -> dict:
    """{stage: (total_ms, launches)} accumulated since profile_enable(True)."""
    ms = (C.c_double * len(STAGE_NAMES))()
    cnt = (C.c_longlong * len(STAGE_NAMES))()
    lib().sfgs_profile_read(ms, cnt, len(STAGE_NAMES))
    return {name: (ms[i], cnt[i]) for i, name in enumerate(STAGE_NAMES)}


def last_error() -> str:
    return lib().sfgs_last_error().decode("utf-8", "replace")


class SfgsError(RuntimeError):
    pass


def check(code: int, what: str) -> int:
    if code < 0:
        raise SfgsError(f"{what} failed with code {code}: {last_error()}")
    return code
