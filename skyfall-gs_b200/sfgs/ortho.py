"""Orthographic views: render and differentiate nadir height maps of a satellite scene.

The rasterizer's orthographic camera (sfgs_rasterize_forward_ortho / sfgs_rasterize_backward_ortho, include/sfgs.h)
behind a module shaped like diff_gauss.GaussianRasterizer:

    OrthoRasterizationSettings   NamedTuple; half_width / half_height (s_x, s_y) replace tanfovx / tanfovy, no campos
    OrthoRasterizer(settings)    nn.Module; same call signature, validation and 6-tuple as GaussianRasterizer
    projection_matrix(...)       the orthographic projection, transposed (row vectors) like getProjectionMatrix
    nadir_camera(...)            a camera looking straight down (-z) on an axis-aligned box of a z-up scene
    render_height_map(...)       the scene's height map (a DSM) in one rasterizer call, differentiable

The view is t = [m, 1]·viewmatrix.  A Gaussian's pixel position is ndc = ([m, 1]·projmatrix).xy (no divide), its depth
t_z, and its 2D covariance J W Sigma W^T J^T with the constant J = diag(W / (2 s_x), H / (2 s_y)).  SH colours and the
normals' orientation use the view's +z axis, one direction for the whole frame.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch
import torch.nn as nn

import diff_gauss

from . import native as N
from . import rasterizer as R


class OrthoRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    half_width: float       # s_x: half the view volume's width, in view-space units
    half_height: float      # s_y
    kernel_size: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    prefiltered: bool
    debug: bool
    subpixel_offset: Optional[torch.Tensor] = None   # [H,W,2] CUDA float32, or None


def projection_matrix(s_x, s_y, znear, zfar, cx=0.0, cy=0.0):
    """The orthographic projection of the box |x| <= s_x, |y| <= s_y, znear <= z <= zfar of view space, as the
    transposed (row-vector) [4,4] float32 matrix, like getProjectionMatrix: projmatrix = viewmatrix @ this.

    x and y map to ndc x / s_x + cx and y / s_y + cy, so (cx, cy) is the principal point's offset in ndc (0: the
    image centre); z maps to [0, 1] (the rasterizer does not read it) and w is 1."""
    O = torch.zeros((4, 4), dtype=torch.float64)
    O[0, 0], O[0, 3] = 1.0 / float(s_x), float(cx)
    O[1, 1], O[1, 3] = 1.0 / float(s_y), float(cy)
    O[2, 2], O[2, 3] = 1.0 / (float(zfar) - float(znear)), -float(znear) / (float(zfar) - float(znear))
    O[3, 3] = 1.0
    return O.t().contiguous().float()


class NadirCamera(NamedTuple):
    image_height: int
    image_width: int
    half_width: float
    half_height: float
    viewmatrix: torch.Tensor    # [4,4] float32, row vectors (world_view_transform)
    projmatrix: torch.Tensor    # [4,4] float32, viewmatrix @ projection_matrix
    z_top: float                # the camera plane; a pixel's height is z_top - its depth
    xmin: float                 # world x of the image's left edge
    ymax: float                 # world y of the image's top edge
    resolution: float           # world units per pixel


def nadir_camera(xmin, xmax, ymin, ymax, resolution, z_top):
    """An orthographic camera at height z_top looking down (-z) on the box [xmin, xmax] x [ymin, ymax] of a scene
    whose up axis is +z (Skyfall-GS's normalised scenes).  Image columns run along +x and rows along -y (north up);
    pixel (i, j) covers x in [xmin + i r, xmin + (i+1) r], y in [ymax - (j+1) r, ymax - j r] for r = resolution.
    The image is round((xmax - xmin) / r) x round((ymax - ymin) / r) pixels, so the box is grown or shrunk on its right
    and bottom edges by less than half a pixel.  View depth is z_top - z: the scene must lie at least 0.2 below z_top,
    as for any camera (the near cull)."""
    r = float(resolution)
    if not r > 0.0:
        raise ValueError(f"resolution must be > 0, got {resolution}")
    W = max(1, int(round((float(xmax) - float(xmin)) / r)))
    H = max(1, int(round((float(ymax) - float(ymin)) / r)))
    s_x, s_y = 0.5 * W * r, 0.5 * H * r
    c = (float(xmin) + s_x, float(ymax) - s_y, float(z_top))
    # view axes in world space: x_v = +x, y_v = -y, z_v = -z (a proper rotation); t = R (m - c)
    Rm = torch.tensor([[1.0, 0.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, -1.0]], dtype=torch.float64)
    V = torch.zeros((4, 4), dtype=torch.float64)
    V[:3, :3] = Rm.t()
    V[3, :3] = -(Rm @ torch.tensor(c, dtype=torch.float64))
    V[3, 3] = 1.0
    view = V.float()
    proj = (V @ projection_matrix(s_x, s_y, 0.01, max(2.0 * abs(float(z_top)), 1.0) + 1e4).double()).float()
    return NadirCamera(H, W, s_x, s_y, view, proj, float(z_top), float(xmin), float(ymax), r)


class OrthoRasterizer(nn.Module):
    """diff_gauss.GaussianRasterizer for an orthographic camera: same call, same checks, same returned
    (color [3,H,W], depth [1,H,W], unit normal [3,H,W], alpha [1,H,W], radii [P], extra [F,H,W] | empty).  `means2D`'s
    .grad receives (dL/dx_ndc W/2, dL/dy_ndc H/2, sum |.|), the densification statistics.  There are no camera
    gradients: a viewmatrix or projmatrix that requires grad raises.  With depth_quantile=q (0 < q < 1) a 7th output,
    depth_q [1,H,W], as for diff_gauss.GaussianRasterizer; with depth_distortion=True a 7th output, distortion [1,H,W],
    likewise (not both in one call).  ray_depth=True: the same outputs with each splat's depth taken where the pixel's
    ray meets it (as for diff_gauss.GaussianRasterizer); with depth_quantile, not with depth_distortion.
    plane_normals=True (with ray_depth=True): each splat's normal is that of its ray-depth plane (as for
    diff_gauss.GaussianRasterizer); norm3Ds_precomp raises with it."""

    def __init__(self, raster_settings: OrthoRasterizationSettings, depth_quantile=None, depth_distortion=False,
                 ray_depth=False, plane_normals=False):
        super().__init__()
        self.raster_settings = raster_settings
        self.depth_quantile = depth_quantile
        self.depth_distortion = depth_distortion
        self.ray_depth = ray_depth
        self.plane_normals = plane_normals

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3Ds_precomp=None, norm3Ds_precomp=None, extra_attrs=None):
        out = self._rasterize(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3Ds_precomp,
                              norm3Ds_precomp, extra_attrs)
        return out[:7] if self.depth_quantile is not None else out

    def _rasterize(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                   cov3Ds_precomp=None, norm3Ds_precomp=None, extra_attrs=None):
        """forward()'s checks and call; with a quantile the tuple also ends with depth_q_pos [H,W]."""
        rs = self.raster_settings
        shs, colors_precomp, cov3Ds_precomp, norm3Ds_precomp, extra_attrs = diff_gauss._checked_inputs(
            shs, colors_precomp, scales, rotations, cov3Ds_precomp, norm3Ds_precomp, extra_attrs)
        if any(isinstance(m, torch.Tensor) and m.requires_grad for m in (rs.viewmatrix, rs.projmatrix)):
            raise ValueError("OrthoRasterizer forms no camera gradients: viewmatrix and projmatrix must not require "
                             "grad (detach them)")
        if rs.subpixel_offset is not None:
            R.check_subpixel_offset(rs.subpixel_offset, int(rs.image_height), int(rs.image_width))
        if self.depth_distortion and self.depth_quantile is not None:
            raise N.SfgsError("OrthoRasterizer: depth_distortion and depth_quantile in one call are not supported; "
                              "render them in two calls")
        if self.plane_normals and not self.ray_depth:
            raise N.SfgsError("OrthoRasterizer: plane_normals are the normals of the ray-depth plane and need "
                              "ray_depth=True")
        if self.depth_distortion and self.plane_normals:
            raise N.SfgsError("OrthoRasterizer: depth_distortion together with plane_normals is not supported")
        if self.depth_distortion and self.ray_depth:
            raise N.SfgsError("OrthoRasterizer: depth_distortion together with ray_depth is not supported")
        # the half-extents travel in the tan_fov fields (as numbers: they get no gradient), and campos is not read
        s_x, s_y = float(rs.half_width), float(rs.half_height)
        campos = torch.zeros(3, dtype=torch.float32, device=means3D.device)
        settings = diff_gauss.GaussianRasterizationSettings(
            rs.image_height, rs.image_width, s_x, s_y, rs.kernel_size, rs.subpixel_offset, rs.bg, rs.scale_modifier,
            rs.viewmatrix, rs.projmatrix, rs.sh_degree, campos, rs.prefiltered, rs.debug)
        # deterministic under torch.use_deterministic_algorithms(True), as for the perspective backward
        return diff_gauss._RasterizeGaussians.apply(
            means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, norm3Ds_precomp,
            extra_attrs, settings, True, rs.viewmatrix, rs.projmatrix, campos, s_x, s_y,
            None if self.depth_quantile is None else float(self.depth_quantile), bool(self.depth_distortion),
            rs.subpixel_offset, True, bool(self.ray_depth), bool(self.plane_normals))


def render_height_map(camera: NadirCamera, means3D, opacities, scales, rotations, shs=None, colors_precomp=None,
                      sh_degree=0, alpha_min=0.5, kernel_size=0.1, scale_modifier=1.0, surface_quantile=None,
                      ray_depth=False):
    """The scene's height map [H, W] seen by `camera` (nadir_camera): z_top - depth / alpha where the accumulated
    alpha is >= alpha_min, NaN elsewhere.  depth / alpha is the alpha-normalised expected view depth of the pixel.
    Differentiable with respect to the Gaussians (e.g. an L1 against a DSM over the finite pixels).

    surface_quantile=q (0 < q < 1): z_top - depth_q instead, the depth of the one splat at which the pixel's
    accumulated opacity crosses q (q = 0.5: the median depth), where a splat was selected and alpha >= alpha_min.  It
    does not blend a roof edge with the ground below it; a lower q reports the first surface seen from above.

    ray_depth=True: each splat reports its depth where the pixel's ray meets it, not its centre's depth, so a sloped
    roof of flat splats is rendered as a slope instead of terraces (in both maps), and the map's gradient reaches the
    splats' rotations and scales."""
    dev = means3D.device
    if shs is None and colors_precomp is None:
        colors_precomp = torch.zeros((means3D.shape[0], 3), dtype=torch.float32, device=dev)
    rs = OrthoRasterizationSettings(camera.image_height, camera.image_width, camera.half_width, camera.half_height,
                                    kernel_size, torch.zeros(3, device=dev), scale_modifier,
                                    camera.viewmatrix.to(dev), camera.projmatrix.to(dev), sh_degree, False, False)
    means2D = torch.zeros_like(means3D)
    out = OrthoRasterizer(rs, depth_quantile=surface_quantile, ray_depth=ray_depth)._rasterize(
        means3D, means2D, opacities, shs=shs, colors_precomp=colors_precomp, scales=scales, rotations=rotations)
    depth, alpha = out[1][0], out[3][0]
    if surface_quantile is not None:
        depth_q, depth_q_pos = out[6][0], out[7]
        valid = (depth_q_pos > 0) & (alpha >= alpha_min)
        return torch.where(valid, camera.z_top - depth_q, torch.full_like(depth_q, float("nan")))
    valid = alpha >= alpha_min
    safe = torch.where(valid, alpha, torch.ones_like(alpha))       # no 0/0 in the masked branch's gradient
    return torch.where(valid, camera.z_top - depth / safe, torch.full_like(depth, float("nan")))
