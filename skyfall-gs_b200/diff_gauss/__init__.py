"""diff_gauss — drop-in for the reference's autograd wrapper package.

Public surface (what gaussian_renderer/__init__.py:14 imports and what
RAST/diff_gauss/__init__.py:182-254 defines):

    GaussianRasterizationSettings   NamedTuple, same 14 fields in the same order
    GaussianRasterizer(settings)    nn.Module; .forward(...) and .markVisible(positions)
    rasterize_gaussians(...)        functional form

Returned tuple: (color[3,H,W], depth[1,H,W], unit normal[3,H,W], alpha[1,H,W],
radii[P] int32, extra[F,H,W] | empty), and with GaussianRasterizer(settings, depth_quantile=q) a 7th output,
depth_q[1,H,W]: the depth at which the pixel's accumulated opacity crosses q (q = 0.5: the median depth), 0 where
it never does, differentiable like the others; with GaussianRasterizer(settings, depth_distortion=True) a 7th output,
distortion[1,H,W]: sum_{i<j} w_i w_j (m_i - m_j)^2 over the pixel's blended splats, the distortion loss of Mip-NeRF
360 / 2DGS, differentiable like the others.  With GaussianRasterizer(settings, ray_depth=True) the outputs are the
same, but each splat's depth is taken where the pixel's ray meets it rather than at its centre (in depth and in
depth_q), so the depth's gradient also reaches rotations and scales; GaussianRasterizer(settings, ray_depth=True,
plane_normals=True) also replaces each splat's shortest-axis normal by the normal of its ray-depth plane, so the
normal map describes the surface the depth map renders.  `means2D` is a dummy [P,3] leaf whose
.grad receives (dL/dx_ndc * W/2, dL/dy_ndc * H/2, sum |.|) — the densification
statistics consumed by scene/gaussian_model.py:744-749.
"""
from __future__ import annotations

import functools
import os
import sys
from typing import NamedTuple

import torch
import torch.nn as nn

_pkg_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _pkg_root not in sys.path:  # make the sibling `sfgs` package importable when only this dir is on sys.path
    sys.path.insert(0, _pkg_root)

from . import _C  # noqa: E402
from sfgs import graphs as _graphs  # noqa: E402

MAX_EXTRA_DIMS = 34  # RAST/cuda_rasterizer/auxiliary.h:20

# The reference normalises the blended normal map with torch ops inside the autograd graph
# (RAST/diff_gauss/__init__.py:48: ~4 elementwise kernels forward, ~8 backward, three passes over 3·H·W floats).
# Here the blend kernel writes the unit normals itself and the blend adjoint applies the normalize adjoint while
# it loads each pixel's cotangent (SURVEY.md 8f rank 1).  Set SFGS_FUSE_NORMALIZE=0 to get the torch post-op back.
FUSE_NORMALIZE = os.environ.get("SFGS_FUSE_NORMALIZE", "1") != "0"

# GaussianRasterizationSettings.subpixel_offset (Mip-Splatting's ray jitter: Skyfall-GS's train.py --ray_jitter draws
# U(-0.5, 0.5) per pixel, and --resample_gt_image resamples the target at the same positions).  The reference's
# rasterizer drops it; with SFGS_SUBPIXEL_OFFSET=1 a [H,W,2] tensor is honoured: pixel (x, y) samples the splats at
# (x + off[y,x,0], y + off[y,x,1]).  Placeholders with numel() <= 1 are ignored.  Off by default, so the default
# keeps the reference's semantics exactly.
SUBPIXEL_OFFSET = os.environ.get("SFGS_SUBPIXEL_OFFSET", "0") == "1"


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float      # or a 0-d tensor: one that requires grad gets dL/dtanfovx (focal refinement)
    tanfovy: float
    kernel_size: float
    subpixel_offset: torch.Tensor  # ignored (as by the reference) unless SUBPIXEL_OFFSET is on
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _snapshot(args):
    return tuple(a.detach().cpu().clone() if isinstance(a, torch.Tensor) else a for a in args)


def _guarded(fn, args, debug, dump_name, label):
    """Run a native call; in debug mode keep a CPU copy of the inputs and dump it if the call throws
    (same contract as the reference's snapshot_fw.dump / snapshot_bw.dump)."""
    if not debug:
        return fn(*args)
    saved = _snapshot(args)
    try:
        return fn(*args)
    except Exception:
        torch.save(saved, dump_name)
        print(f"\nAn error occured in {label}. Writing {dump_name} for debugging.\n")
        raise


def _subpixel_offset(rs):
    """The offsets to honour: None unless SUBPIXEL_OFFSET is on and the settings carry a [H,W,2] tensor."""
    off = rs.subpixel_offset
    if not SUBPIXEL_OFFSET or not isinstance(off, torch.Tensor) or off.numel() <= 1:
        return None
    if tuple(off.shape) != (int(rs.image_height), int(rs.image_width), 2):
        raise ValueError(f"subpixel_offset must have shape ({int(rs.image_height)}, {int(rs.image_width)}, 2), "
                         f"got {tuple(off.shape)}")
    return off.detach()


def _with_offset(fn):
    """fn with the subpixel offsets taken from its last positional argument."""
    return lambda *a, **kw: fn(*a[:-1], subpixel_offset=a[-1], **kw)


def _checked_inputs(shs, colors_precomp, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, extra_attrs):
    """The reference's four argument checks (RAST/diff_gauss/__init__.py:209-230), then the optional inputs with the
    empty tensor the native layer takes for None: (shs, colors_precomp, cov3Ds_precomp, norm3Ds_precomp,
    extra_attrs)."""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    has_sr = scales is not None or rotations is not None
    if ((scales is None or rotations is None) and cov3Ds_precomp is None) or (has_sr and cov3Ds_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    if scales is None:
        raise ValueError('To support norm and depth prediction, scales == None is not allowed')
    if rotations is None:
        raise ValueError('To support norm and depth prediction, rotations == None is not allowed')
    return tuple(torch.Tensor([]) if t is None else t
                 for t in (shs, colors_precomp, cov3Ds_precomp, norm3Ds_precomp, extra_attrs))


class _RasterizeGaussians(torch.autograd.Function):
    """The rasterizer for the pinhole camera (diff_gauss) and the orthographic one (sfgs.ortho).  Every input slot is
    always passed: the callers resolve the options `fuse_normalize`, `depth_quantile` (q or None), `depth_distortion`,
    `subpixel_offset` (a [H,W,2] tensor or None), `ortho`, `ray_depth` and `plane_normals` (the last three slots have
    defaults).  With a quantile the outputs end with (depth_q, depth_q_pos); with the distortion, with distortion."""
    # viewmatrix, projmatrix and campos are inputs of their own (the settings tuple is not tracked by autograd), so a
    # camera built from parameters that require grad (scene/cameras.py: Camera(..., optimizing=True)) gets gradients
    CAMERA_INPUTS = slice(12, 15)
    # tanfovx and tanfovy likewise: a 0-d tensor that requires grad gets dL/dtanfovx (focal refinement).  The native
    # layer reads them with float(), which for a CUDA tensor is a host sync each forward and backward, so keep the
    # leaves of a focal refinement on the CPU
    INTRINSICS_INPUTS = slice(15, 17)

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                norm3Ds_precomp, extra_attrs, raster_settings, fuse_normalize, viewmatrix, projmatrix, campos, tanfovx,
                tanfovy, depth_quantile, depth_distortion, subpixel_offset=None, ortho=False, ray_depth=False,
                plane_normals=False):
        rs = raster_settings
        ctx.depth_q, ctx.dist, ctx.ray_depth = depth_quantile is not None, bool(depth_distortion), bool(ray_depth)
        ctx.plane_normals = bool(plane_normals)
        n_extra = extra_attrs.shape[1] if extra_attrs.shape[0] != 0 else 0
        assert n_extra <= MAX_EXTRA_DIMS
        # under stream capture (torch.cuda.graph) the capture-safe entries run: no host wait, intrinsics that are 0-d
        # CUDA tensors read at replay time, a capacity fixed at capture (sfgs.graphs)
        ctx.graph = means3D.is_cuda and torch.cuda.is_current_stream_capturing()
        capacity = 0
        opts = {}
        if ctx.graph:
            for on, what in ((ctx.depth_q, "the depth quantile"), (ctx.dist, "the depth distortion"),
                             (ortho, "the orthographic camera"), (ctx.plane_normals, "plane normals"),
                             (ctx.ray_depth, "ray depth")):
                if on:
                    raise _C.SfgsError(f"diff_gauss: {what} cannot be captured in a CUDA graph")
            if rs.debug:
                raise _C.SfgsError("diff_gauss: debug=True synchronises after every stage and cannot be captured in a "
                                   "CUDA graph")
            P = int(means3D.shape[0])
            capacity = _graphs.resolve_capacity(means3D.device, P, rs.image_width, rs.image_height) if P > 0 else 1
            opts.update(capacity_hint=capacity, graph=True)
        if ortho:
            opts["ortho"] = True
        if ctx.depth_q:
            opts["depth_quantile"] = depth_quantile
        if ctx.dist:
            opts["depth_distortion"] = True
        if ctx.ray_depth:
            opts["ray_depth"] = True
        if ctx.plane_normals:
            opts["plane_normals"] = True
        native_args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
                       cov3Ds_precomp, norm3Ds_precomp, extra_attrs, n_extra, viewmatrix, projmatrix,
                       tanfovx, tanfovy, rs.kernel_size, rs.image_height, rs.image_width, sh, rs.sh_degree,
                       campos, rs.prefiltered, rs.debug)
        ctx.fused = bool(fuse_normalize)
        fwd = functools.partial(_C.rasterize_gaussians_fused if ctx.fused else _C.rasterize_gaussians, **opts)
        if subpixel_offset is not None:
            # the offsets travel as the last argument, so that the debug snapshot holds them too
            fwd, native_args = _with_offset(fwd), native_args + (subpixel_offset,)
        out = _guarded(fwd, native_args, rs.debug, "snapshot_fw.dump", "forward")
        (num_rendered, color, depth, norm, alpha, radii, extra, geom_buf, binning_buf, img_buf) = out[:10]
        norm_raw = out[10] if ctx.fused else torch.empty(0, device=means3D.device)
        # the 7th output and the state its backward reads: (depth_q, depth_q_pos) or (distortion, distortion_state)
        side, side_state = out[-2:] if ctx.depth_q or ctx.dist else (None, torch.empty(0, device=means3D.device))
        ctx.raster_settings, ctx.subpixel_offset, ctx.ortho = rs, subpixel_offset, bool(ortho)
        ctx.camera, ctx.intrinsics = (viewmatrix, projmatrix, campos), (tanfovx, tanfovy)
        # the graph backward is given the capacity in place of num_rendered (not known on the host under capture)
        ctx.num_rendered = capacity if ctx.graph else num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, radii,
                              extra_attrs, sh, geom_buf, binning_buf, img_buf, alpha, norm_raw, side_state)
        ctx.mark_non_differentiable(radii)
        if ctx.depth_q:
            # depth_q_pos: which splat each pixel selected (0: none), for render_height_map's mask
            ctx.mark_non_differentiable(radii, side_state)
            return color, depth, norm, alpha, radii, extra, side, side_state
        return (color, depth, norm, alpha, radii, extra) + ((side,) if ctx.dist else ())

    @staticmethod
    def backward(ctx, g_color, g_depth, g_norm, g_alpha, _g_radii, g_extra, g_side=None, _g_depth_q_pos=None):
        rs = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, radii, extra_attrs, sh,
         geom_buf, binning_buf, img_buf, alpha, norm_raw, side_state) = ctx.saved_tensors
        viewmatrix, projmatrix, campos = ctx.camera
        native_args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, extra_attrs, rs.scale_modifier,
                       cov3Ds_precomp, norm3Ds_precomp, viewmatrix, projmatrix, *ctx.intrinsics,
                       rs.kernel_size, g_color, g_depth, g_norm, g_alpha, g_extra, sh, rs.sh_degree, campos,
                       geom_buf, ctx.num_rendered, binning_buf, img_buf, alpha, rs.debug)
        need_camera = ctx.needs_input_grad[_RasterizeGaussians.CAMERA_INPUTS]
        need_intrinsics = ctx.needs_input_grad[_RasterizeGaussians.INTRINSICS_INPUTS]
        opts = dict(norm_raw=norm_raw) if ctx.fused else {}
        # only when asked for: a camera without requires_grad keeps the default native call, and the focal-length
        # gradients come with the camera gradients, from one native call
        if any(need_intrinsics):
            opts.update(camera_grad=True, intrinsics_grad=True)
        elif any(need_camera):
            opts.update(camera_grad=True)
        if ctx.graph:
            opts["graph"] = True
        if ctx.ortho:
            opts["ortho"] = True
        if ctx.depth_q:
            opts.update(depth_q_pos=side_state, dL_dout_depth_q=g_side.contiguous())
        if ctx.dist:
            opts.update(distortion_state=side_state, dL_dout_distortion=g_side.contiguous())
        if ctx.ray_depth:
            opts["ray_depth"] = True
        if ctx.plane_normals:
            opts["plane_normals"] = True
        bwd = functools.partial(_C.rasterize_gaussians_backward_fused if ctx.fused else
                                _C.rasterize_gaussians_backward, **opts)
        if ctx.subpixel_offset is not None:
            bwd, native_args = _with_offset(bwd), native_args + (ctx.subpixel_offset,)
        grads = _guarded(bwd, native_args, rs.debug, "snapshot_bw.dump", "backward")

        def cast(gs, inputs, need):
            return tuple(g.to(dtype=t.dtype, device=t.device) if n else None for g, t, n in zip(gs, inputs, need))
        g_camera = cast(grads[10:13], ctx.camera, need_camera) if opts.get("camera_grad") else (None,) * 3
        g_intrinsics = cast(grads[13:15], ctx.intrinsics, need_intrinsics) if any(need_intrinsics) else (None,) * 2
        (g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_norm3D, g_sh, g_scales, g_rot, g_extra_attrs) = grads[:10]
        # order of forward's inputs; the settings tuple and the options get no gradient
        return ((g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rot, g_cov3D, g_norm3D, g_extra_attrs)
                + (None, None) + g_camera + g_intrinsics + (None,) * 6)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        norm3Ds_precomp, extra_attrs, raster_settings, depth_quantile=None, depth_distortion=False,
                        ray_depth=False, plane_normals=False):
    rs = raster_settings
    if depth_distortion and depth_quantile is not None:
        raise _C.SfgsError("diff_gauss: depth_distortion and depth_quantile in one call are not supported; render "
                           "them in two calls")
    if plane_normals and not ray_depth:
        raise _C.SfgsError("diff_gauss: plane_normals are the normals of the ray-depth plane and need ray_depth=True")
    if depth_distortion and plane_normals:
        raise _C.SfgsError("diff_gauss: depth_distortion together with plane_normals is not supported")
    if depth_distortion and ray_depth:
        raise _C.SfgsError("diff_gauss: depth_distortion together with ray_depth is not supported")
    out = _RasterizeGaussians.apply(
        means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, norm3Ds_precomp,
        extra_attrs, rs, FUSE_NORMALIZE, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy,
        None if depth_quantile is None else float(depth_quantile), bool(depth_distortion), _subpixel_offset(rs), False,
        bool(ray_depth), bool(plane_normals))
    color, depth, norm, alpha, radii, extra = out[:6]
    if not FUSE_NORMALIZE:
        # the reference normalises the blended normal map in torch, inside the autograd graph (diff_gauss/__init__.py:48)
        norm = torch.nn.functional.normalize(norm, p=2, dim=0)
    return (color, depth, norm, alpha, radii, extra) + tuple(out[6:7])


class GaussianRasterizer(nn.Module):
    """depth_quantile=q (0 < q < 1): forward() also returns depth_q [1,H,W], the depth at which each pixel's accumulated
    opacity crosses q (include/sfgs.h, sfgs_rasterize_forward_depth_quantile).  depth_distortion=True: forward() also
    returns distortion [1,H,W], sum_{i<j} w_i w_j (m_i - m_j)^2 over each pixel's blended splats in units of depth^2
    (include/sfgs.h, sfgs_rasterize_forward_distortion).  Not under CUDA-graph capture, and not both in one call.
    ray_depth=True: the same outputs, with each splat's depth taken where the pixel's ray meets it, z + g . (p - mu),
    not at its centre (include/sfgs.h, sfgs_rasterize_forward_ray_depth); combines with depth_quantile, not with
    depth_distortion or CUDA-graph capture.  plane_normals=True (with ray_depth=True): the same outputs, with each
    splat's normal that of its ray-depth plane rather than its shortest axis (include/sfgs.h,
    sfgs_rasterize_forward_plane_normals); norm3Ds_precomp raises with it."""

    def __init__(self, raster_settings, depth_quantile=None, depth_distortion=False, ray_depth=False,
                 plane_normals=False):
        super().__init__()
        self.raster_settings = raster_settings
        self.depth_quantile = depth_quantile
        self.depth_distortion = depth_distortion
        self.ray_depth = ray_depth
        self.plane_normals = plane_normals

    def markVisible(self, positions):
        """Boolean mask of the points in front of the near plane (view depth > 0.2)."""
        rs = self.raster_settings
        with torch.no_grad():
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3Ds_precomp=None, norm3Ds_precomp=None, extra_attrs=None):
        shs, colors_precomp, cov3Ds_precomp, norm3Ds_precomp, extra_attrs = _checked_inputs(
            shs, colors_precomp, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, extra_attrs)
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                   norm3Ds_precomp, extra_attrs, self.raster_settings, self.depth_quantile,
                                   self.depth_distortion, self.ray_depth, self.plane_normals)
