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
360 / 2DGS, differentiable like the others.  `means2D` is a dummy [P,3] leaf whose
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


def _requires_grad(x):
    return isinstance(x, torch.Tensor) and x.requires_grad


class _RasterizeGaussians(torch.autograd.Function):
    # viewmatrix, projmatrix and campos are inputs of their own (the settings tuple is not tracked by autograd), so a
    # camera built from parameters that require grad (scene/cameras.py: Camera(..., optimizing=True)) gets gradients.
    CAMERA_INPUTS = slice(12, 15)
    # tanfovx and tanfovy likewise, passed only when one of them is a tensor that requires grad (focal refinement);
    # otherwise the settings' values are used, as they always were
    INTRINSICS_INPUTS = slice(15, 17)

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                norm3Ds_precomp, extra_attrs, raster_settings, fuse_normalize=False, viewmatrix=None, projmatrix=None,
                campos=None, tanfovx=None, tanfovy=None, depth_quantile=None, depth_distortion=False):
        rs = raster_settings
        ctx.depth_q = depth_quantile is not None
        ctx.dist = bool(depth_distortion)
        # the option inputs after the intrinsics slots: none, the quantile, or the quantile slot and the distortion flag
        ctx.n_options = 2 if ctx.dist else int(ctx.depth_q)
        ctx.intrinsics = None if tanfovx is None else (tanfovx, tanfovy)
        viewmatrix = rs.viewmatrix if viewmatrix is None else viewmatrix
        projmatrix = rs.projmatrix if projmatrix is None else projmatrix
        campos = rs.campos if campos is None else campos
        n_extra = extra_attrs.shape[1] if extra_attrs.shape[0] != 0 else 0
        assert n_extra <= MAX_EXTRA_DIMS
        native_args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
                       cov3Ds_precomp, norm3Ds_precomp, extra_attrs, n_extra, viewmatrix, projmatrix,
                       rs.tanfovx, rs.tanfovy, rs.kernel_size, rs.image_height, rs.image_width, sh, rs.sh_degree,
                       campos, rs.prefiltered, rs.debug)
        ctx.fused = bool(fuse_normalize)
        off = _subpixel_offset(rs)
        fwd = _C.rasterize_gaussians_fused if ctx.fused else _C.rasterize_gaussians
        # under stream capture (torch.cuda.graph) the capture-safe entries run: no host wait, intrinsics that are 0-d
        # CUDA tensors read at replay time, a capacity fixed at capture (sfgs.graphs)
        ctx.graph = means3D.is_cuda and torch.cuda.is_current_stream_capturing()
        capacity = 0
        if ctx.graph:
            if ctx.depth_q:
                raise _C.SfgsError("diff_gauss: the depth quantile cannot be captured in a CUDA graph")
            if ctx.dist:
                raise _C.SfgsError("diff_gauss: the depth distortion cannot be captured in a CUDA graph")
            if rs.debug:
                raise _C.SfgsError("diff_gauss: debug=True synchronises after every stage and cannot be captured in a "
                                   "CUDA graph")
            P = int(means3D.shape[0])
            capacity = _graphs.resolve_capacity(means3D.device, P, rs.image_width, rs.image_height) if P > 0 else 1
            fwd = functools.partial(fwd, capacity_hint=capacity, graph=True)
        if ctx.depth_q:
            fwd = functools.partial(fwd, depth_quantile=depth_quantile)
        if ctx.dist:
            fwd = functools.partial(fwd, depth_distortion=True)
        if off is not None:
            # the offsets travel as the last argument, so that the debug snapshot holds them too
            fwd, native_args = _with_offset(fwd), native_args + (off,)
        out = _guarded(fwd, native_args, rs.debug, "snapshot_fw.dump", "forward")
        # the 7th output and the state its backward reads: (depth_q, depth_q_pos) or (distortion, distortion_state)
        side, side_state = out[-2:] if ctx.n_options else (None, torch.empty(0, device=means3D.device))
        if ctx.fused:
            (num_rendered, color, depth, norm, alpha, radii, extra, geom_buf, binning_buf, img_buf,
             norm_raw) = out[:11]
        else:
            (num_rendered, color, depth, norm, alpha, radii, extra,
             geom_buf, binning_buf, img_buf) = out[:10]
            norm_raw = torch.empty(0, device=means3D.device)
        ctx.subpixel_offset = off
        ctx.raster_settings = rs
        ctx.camera = (viewmatrix, projmatrix, campos)
        # the graph backward is given the capacity in place of num_rendered (not known on the host under capture)
        ctx.num_rendered = capacity if ctx.graph else num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, radii,
                              extra_attrs, sh, geom_buf, binning_buf, img_buf, alpha, norm_raw, side_state)
        ctx.mark_non_differentiable(radii)
        if ctx.n_options:
            return color, depth, norm, alpha, radii, extra, side
        return color, depth, norm, alpha, radii, extra

    @staticmethod
    def backward(ctx, g_color, g_depth, g_norm, g_alpha, _g_radii, g_extra, g_side=None):
        rs = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, radii, extra_attrs, sh,
         geom_buf, binning_buf, img_buf, alpha, norm_raw, side_state) = ctx.saved_tensors
        viewmatrix, projmatrix, campos = ctx.camera
        native_args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, extra_attrs, rs.scale_modifier,
                       cov3Ds_precomp, norm3Ds_precomp, viewmatrix, projmatrix, rs.tanfovx, rs.tanfovy,
                       rs.kernel_size, g_color, g_depth, g_norm, g_alpha, g_extra, sh, rs.sh_degree, campos,
                       geom_buf, ctx.num_rendered, binning_buf, img_buf, alpha, rs.debug)
        bwd = _C.rasterize_gaussians_backward
        if ctx.fused:
            bwd = lambda *a, **kw: _C.rasterize_gaussians_backward_fused(*a, norm_raw=norm_raw, **kw)  # noqa: E731
        camera_grad = any(ctx.needs_input_grad[_RasterizeGaussians.CAMERA_INPUTS])
        intrinsics_grad = ctx.intrinsics is not None and any(
            ctx.needs_input_grad[_RasterizeGaussians.INTRINSICS_INPUTS])
        if intrinsics_grad:
            # the focal-length gradients come with the camera gradients, from one native call
            bwd = functools.partial(bwd, camera_grad=True, intrinsics_grad=True)
        elif camera_grad:
            # only when asked for: a camera without requires_grad keeps the default native call
            bwd = functools.partial(bwd, camera_grad=True)
        if ctx.graph:
            bwd = functools.partial(bwd, graph=True)
        if ctx.depth_q:
            bwd = functools.partial(bwd, depth_q_pos=side_state, dL_dout_depth_q=g_side.contiguous())
        if ctx.dist:
            bwd = functools.partial(bwd, distortion_state=side_state, dL_dout_distortion=g_side.contiguous())
        if ctx.subpixel_offset is not None:
            bwd, native_args = _with_offset(bwd), native_args + (ctx.subpixel_offset,)
        grads = _guarded(bwd, native_args, rs.debug, "snapshot_bw.dump", "backward")
        (g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_norm3D, g_sh, g_scales, g_rot, g_extra_attrs) = grads[:10]
        g_camera = (None, None, None)
        if camera_grad or intrinsics_grad:
            g_camera = tuple(g.to(dtype=t.dtype, device=t.device) if need else None for g, t, need in
                             zip(grads[10:13], ctx.camera, ctx.needs_input_grad[_RasterizeGaussians.CAMERA_INPUTS]))
        g_intrinsics = ()
        if ctx.intrinsics is not None or ctx.n_options:
            g_intrinsics = (None, None)
            if intrinsics_grad:
                g_intrinsics = tuple(
                    g.to(dtype=t.dtype, device=t.device) if need else None for g, t, need in
                    zip(grads[13:15], ctx.intrinsics, ctx.needs_input_grad[_RasterizeGaussians.INTRINSICS_INPUTS]))
        # order of forward's inputs; the settings tuple, the fusion flag and the options get no gradient
        return (g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rot, g_cov3D, g_norm3D, g_extra_attrs,
                None, None) + g_camera + g_intrinsics + (None,) * ctx.n_options


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        norm3Ds_precomp, extra_attrs, raster_settings, depth_quantile=None, depth_distortion=False):
    rs = raster_settings
    # tanfovx / tanfovy may be 0-d tensors; the native layer reads them with float(), which for a CUDA tensor is a
    # host sync each forward and backward, so keep the leaves of a focal refinement on the CPU
    intrinsics = (rs.tanfovx, rs.tanfovy) if _requires_grad(rs.tanfovx) or _requires_grad(rs.tanfovy) else ()
    if depth_distortion and depth_quantile is not None:
        raise _C.SfgsError("diff_gauss: depth_distortion and depth_quantile in one call are not supported; render "
                           "them in two calls")
    # the quantile, then the distortion flag, follow the two intrinsics slots (None: the settings' values)
    options = ()
    if depth_distortion:
        options = (intrinsics or (None, None)) + (None, True)
    elif depth_quantile is not None:
        options = (intrinsics or (None, None)) + (float(depth_quantile),)
    out = _RasterizeGaussians.apply(
        means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, norm3Ds_precomp,
        extra_attrs, raster_settings, FUSE_NORMALIZE, rs.viewmatrix, rs.projmatrix, rs.campos,
        *(options or intrinsics))
    color, depth, norm, alpha, radii, extra = out[:6]
    if not FUSE_NORMALIZE:
        # the reference normalises the blended normal map in torch, inside the autograd graph (diff_gauss/__init__.py:48)
        norm = torch.nn.functional.normalize(norm, p=2, dim=0)
    return (color, depth, norm, alpha, radii, extra) + tuple(out[6:])


class GaussianRasterizer(nn.Module):
    """depth_quantile=q (0 < q < 1): forward() also returns depth_q [1,H,W], the depth at which each pixel's accumulated
    opacity crosses q (include/sfgs.h, sfgs_rasterize_forward_depth_quantile).  depth_distortion=True: forward() also
    returns distortion [1,H,W], sum_{i<j} w_i w_j (m_i - m_j)^2 over each pixel's blended splats in units of depth^2
    (include/sfgs.h, sfgs_rasterize_forward_distortion).  Not under CUDA-graph capture, and not both in one call."""

    def __init__(self, raster_settings, depth_quantile=None, depth_distortion=False):
        super().__init__()
        self.raster_settings = raster_settings
        self.depth_quantile = depth_quantile
        self.depth_distortion = depth_distortion

    def markVisible(self, positions):
        """Boolean mask of the points in front of the near plane (view depth > 0.2)."""
        rs = self.raster_settings
        with torch.no_grad():
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3Ds_precomp=None, norm3Ds_precomp=None, extra_attrs=None):
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        has_sr = scales is not None or rotations is not None
        if ((scales is None or rotations is None) and cov3Ds_precomp is None) or (has_sr and cov3Ds_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if scales is None:
            raise ValueError('To support norm and depth prediction, scales == None is not allowed')
        if rotations is None:
            raise ValueError('To support norm and depth prediction, rotations == None is not allowed')

        def _or_empty(t):
            return torch.Tensor([]) if t is None else t

        return rasterize_gaussians(means3D, means2D, _or_empty(shs), _or_empty(colors_precomp), opacities, scales,
                                   rotations, _or_empty(cov3Ds_precomp), _or_empty(norm3Ds_precomp),
                                   _or_empty(extra_attrs), self.raster_settings, self.depth_quantile,
                                   self.depth_distortion)
