"""The `diff_gauss._C` surface on top of libsfgs.so.

rasterize_gaussians          <- RasterizeGaussiansCUDA          (RAST/rasterize_points.cu:35-135)
rasterize_gaussians_backward <- RasterizeGaussiansBackwardCUDA  (RAST/rasterize_points.cu:137-243)
mark_visible                 <- markVisible                     (RAST/rasterize_points.cu:245-264)

Same positional arguments, same return tuples, same error behaviour (a bad
means3D shape raises; CUDA errors surface as exceptions).  Differences that a
caller cannot observe: outputs are allocated uninitialised because every
element is written by the kernels (the reference zero-fills 6 + 12 tensors per
iteration), and the scratch byte tensors have this library's layout.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import warnings

import torch

from . import native as N

NUM_CHANNELS = 3


def _ptr(t, keep):
    """Device pointer of a tensor, or None for `None` / empty tensors (the reference passes nullptr)."""
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32 and t.dtype != torch.int32 and t.dtype != torch.uint8 and t.dtype != torch.bool:
        raise TypeError(f"unsupported dtype {t.dtype}")
    if not t.is_cuda:
        raise ValueError("tensor must live on a CUDA device")
    tc = t.contiguous()
    if tc.data_ptr() % 16:          # offset views: the kernels use 128-bit loads on [P,4] / [P,16,3] rows
        tc = tc.clone()
    keep.append(tc)
    return tc.data_ptr()


def _band(tile_rows):
    """(begin, end) of a tile-row band for the C ABI, where (0, 0) means "whole image": an EMPTY band that happens to
    start at row 0 (a rank without rows when there are fewer tile rows than ranks) is passed as an empty band past the
    grid instead."""
    b0, b1 = int(tile_rows[0]), int(tile_rows[1])
    if b1 <= b0:
        return 1 << 20, 1 << 20
    return b0, b1


class _Arena:
    """Allocator callback target: the last tensor handed out is the live buffer."""

    def __init__(self, device):
        self.device = device
        self.tensor = torch.empty(0, dtype=torch.uint8, device=device)
        self.cb = N.ALLOC_FN(self._alloc)

    def _alloc(self, _user, nbytes):
        try:
            self.tensor = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
            return self.tensor.data_ptr()
        except Exception:  # noqa: BLE001 - must not raise through the C ABI
            return None


def check_subpixel_offset(subpixel_offset, H, W):
    """Validate a per-pixel offset tensor: CUDA float32 of shape (H, W, 2).  Raises ValueError otherwise."""
    t = subpixel_offset
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or tuple(t.shape) != (H, W, 2):
        what = (f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__)
        raise ValueError(f"subpixel_offset must be a CUDA float32 tensor of shape ({H}, {W}, 2), got {what}")


def _tan_fov(tan_fovx, tan_fovy, dev):
    """(host floats, device [2] tensor or None) for the graph entries: 0-d CUDA tensors are read by the kernels at run
    time (never with float(), which would synchronise); with two Python numbers they are baked in as launch
    parameters."""
    tensors = [isinstance(t, torch.Tensor) for t in (tan_fovx, tan_fovy)]
    if not any(tensors):
        return float(tan_fovx), float(tan_fovy), None
    parts = []
    for t, is_t in zip((tan_fovx, tan_fovy), tensors):
        if is_t:
            if not t.is_cuda or t.numel() != 1:
                raise ValueError("under graph capture tanfovx / tanfovy must be Python numbers or 0-d CUDA tensors")
            parts.append(t.detach().reshape(()).to(device=dev, dtype=torch.float32))
        else:
            parts.append(torch.full((), float(t), dtype=torch.float32, device=dev))
    return 1.0, 1.0, torch.stack(parts)


GRAPH = "cannot be captured in a CUDA graph"
ORTHO = "not supported with an orthographic camera"
DEPTH_Q = "not supported with the depth quantile"
DISTORTION = "not supported with the depth distortion"
RAY_DEPTH = "not supported with ray depth"
PLANE_NORMALS = "not supported with plane normals"


def _check_plane_normals(where, ray_depth, norm3Ds_precomp, **opts):
    """plane_normals=True: it needs ray_depth=True, and norm3Ds_precomp and each option of `opts` that is set raise
    SfgsError, before any native call."""
    if not ray_depth:
        raise N.SfgsError(f"{where}: plane normals are the normals of the ray-depth plane and need ray_depth=True")
    _reject(where, PLANE_NORMALS, **opts,
            norm3Ds_precomp=norm3Ds_precomp is not None and norm3Ds_precomp.numel() != 0)


def _reject(where, tail, **opts):
    """The options of `opts` that are set (truthy values, in order) as one SfgsError, raised before any native call:
    "<where>: <names> <tail>"."""
    what = [k for k, v in opts.items() if v]
    if what:
        raise N.SfgsError(f"{where}: {', '.join(what)} {tail}")


def _given_together(a_name, a, b_name, b):
    """Whether the pair of a per-pixel output's backward inputs is given; one without the other raises ValueError."""
    if (a is None) != (b is None):
        raise ValueError(f"{a_name} and {b_name} come together")
    return a is not None


def _check_pixel_inputs(state_name, state, dtype, shape, cot_name, cot, H, W, dev):
    """A per-pixel output's backward inputs: the forward's `state` (`dtype`, `shape`) and a float32 [1,H,W] (or [H,W])
    cotangent `cot`, on the rasterizer's device.  Raises ValueError otherwise."""
    for name, t, dt, shapes in ((state_name, state, dtype, (shape,)),
                                (cot_name, cot, torch.float32, ((1, H, W), (H, W)))):
        if not isinstance(t, torch.Tensor) or t.dtype != dt or t.device != dev or tuple(t.shape) not in shapes:
            what = f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{name} must be a {dt} tensor of shape {shapes[0]} on {dev}, got {what}")


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier,
                        cov3Ds_precomp, norm3Ds_precomp, extra_attrs, attr_degree, viewmatrix, projmatrix,
                        tan_fovx, tan_fovy, kernel_size, image_height, image_width, sh, degree, campos,
                        prefiltered, debug, capacity_hint=0, tile_rows=None, fuse_normalize=False, out_planes=None,
                        out_peers=None, subpixel_offset=None, graph=False, *, ortho=False, depth_quantile=None,
                        depth_distortion=False, ray_depth=False, plane_normals=False):
    """Same positional signature and return tuple as the reference's `_C.rasterize_gaussians`.  With
    `fuse_normalize=True` the returned normal map is already F.normalize(., dim=0) (the reference's torch post-op,
    diff_gauss/__init__.py:48) and the un-normalised blend is appended to the tuple for the backward.

    `subpixel_offset` ([H,W,2] CUDA float32, or None): pixel (x, y) samples the splats at (x + off[y,x,0],
    y + off[y,x,1]) (sfgs_rasterize_forward_subpixel); the backward must be given the same tensor.  Offsets must be
    finite; a NaN or Inf raises.  They combine with `tile_rows` and `out_peers`: every rank passes the whole frame's
    offsets, and the bands reassemble the one-call frame bit for bit (with `out_peers` through
    sfgs_rasterize_forward_subpixel_peers).

    `graph=True`: the capture-safe forward (sfgs_rasterize_forward_graph) for torch.cuda.graph.  `capacity_hint` (> 0)
    is the binning capacity; `tan_fovx` / `tan_fovy` may be 0-d CUDA tensors, read on the device at every replay; the
    frame's error flags go to the sticky status word of sfgs.graphs instead of raising, and the first element of the
    tuple is -1 (num_rendered is not known on the host).  debug, tile_rows and out_peers raise.

    `ortho=True`: an orthographic view (sfgs_rasterize_forward_ortho, include/sfgs.h; sfgs.ortho builds its matrices):
    `tan_fovx` / `tan_fovy` are the half-extents s_x, s_y of the view volume, the projected centre is
    [m, 1]·projmatrix without a divide, and SH and normals see the view's +z axis.  Offsets combine with it; graph,
    tile_rows and out_peers raise SfgsError.

    `depth_quantile=q` (0 < q < 1; sfgs_rasterize_forward_depth_quantile, include/sfgs.h): also the surface depth at
    crossing level q, the depth of the splat at which the pixel's accumulated opacity crosses q (q = 0.5: the median
    depth), or 0 where none does.  The tuple ends with (depth_q [1,H,W], depth_q_pos [H,W] int32); the backward takes
    depth_q_pos back.  It combines with `ortho` and offsets; graph, tile_rows, out_peers and extra_attrs raise SfgsError.
    Every other output is bit-identical to the call without it.

    `depth_distortion=True` (sfgs_rasterize_forward_distortion, include/sfgs.h): also the depth distortion
    R = sum_{i<j} w_i w_j (m_i - m_j)^2 over the pixel's blended splats (w = alpha T, m the view depth), the distortion
    loss of Mip-NeRF 360 / 2DGS, in units of depth^2.  The tuple ends with (distortion [1,H,W], distortion_state
    [2,H,W]); the backward takes distortion_state back.  It combines with `ortho` and offsets; depth_quantile, graph,
    tile_rows, out_peers and extra_attrs raise SfgsError.  Every other output is bit-identical to the call without it.

    `ray_depth=True` (sfgs_rasterize_forward_ray_depth, include/sfgs.h): each splat's depth is taken where the pixel's
    ray meets it, d(p) = z + g . (p - mu) with g its depth slope, not its centre's depth z, in out_depth and (with
    `depth_quantile`) in depth_q.  The backward must be given `ray_depth=True` too.  It combines with `ortho`, offsets
    and `depth_quantile`; depth_distortion, graph, tile_rows, out_peers and extra_attrs raise SfgsError.  Every other
    output is bit-identical to the call without it.

    `plane_normals=True` (with `ray_depth=True`; sfgs_rasterize_forward_plane_normals, include/sfgs.h): the normal
    map blends the normal of each splat's ray-depth plane, u = w3 - g_x T0 - g_y T1 flipped toward the camera, in place
    of its shortest axis, so the normals describe the surface the depth map renders.  The backward must be given
    `plane_normals=True` too.  Without ray_depth it raises, and so do norm3Ds_precomp and everything ray depth rejects,
    naming plane normals.  Every other output is bit-identical to the `ray_depth=True` call."""
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    banded = dict(tile_rows=tile_rows is not None, out_peers=out_peers is not None)
    if plane_normals:
        _check_plane_normals("rasterize_gaussians(plane_normals=True)", ray_depth, norm3Ds_precomp,
                             depth_distortion=depth_distortion, graph=graph, **banded,
                             extra_attrs=int(attr_degree) > 0)
    if ray_depth:
        _reject("rasterize_gaussians(ray_depth=True)", RAY_DEPTH, depth_distortion=depth_distortion, graph=graph,
                **banded, extra_attrs=int(attr_degree) > 0)
    if depth_distortion:
        _reject("rasterize_gaussians(depth_distortion=True)", DISTORTION, depth_quantile=depth_quantile is not None,
                graph=graph, **banded, extra_attrs=int(attr_degree) > 0)
    if depth_quantile is not None:
        _reject("rasterize_gaussians(depth_quantile=...)", DEPTH_Q, graph=graph, **banded,
                extra_attrs=int(attr_degree) > 0)
    if ortho:
        _reject("rasterize_gaussians(ortho=True)", ORTHO, graph=graph, **banded)
    if graph:
        _reject("rasterize_gaussians(graph=True)", GRAPH, **{"debug=True (it synchronises after every stage)": debug},
                **banded)
        if int(capacity_hint) <= 0:
            raise N.SfgsError("rasterize_gaussians(graph=True) needs capacity_hint > 0 (see sfgs.graphs.capacity)")
    H, W, F = int(image_height), int(image_width), int(attr_degree)
    if subpixel_offset is not None:
        check_subpixel_offset(subpixel_offset, H, W)
    L = N.lib()
    P = int(means3D.shape[0])
    dev = means3D.device
    fopt = dict(dtype=torch.float32, device=dev)
    alloc = torch.zeros if P == 0 else torch.empty      # the reference returns zero images for P == 0
    # one allocation for the 8 image planes: colour(3) depth(1) alpha(1) normal(3)
    # multi-GPU tile-row mode: `out_planes` is this rank's symmetric [8,H,W] frame block and `out_peers` the
    # peer-mapped pointers of every rank's block; the blend kernel then stores the band into all of them
    if out_planes is not None and P > 0:
        planes = out_planes.view(8, H, W)
        norm_raw = torch.empty((3, H, W), **fopt) if fuse_normalize else None
    else:
        planes = alloc((11 if fuse_normalize else 8, H, W), **fopt)
        norm_raw = planes[8:11] if fuse_normalize else None
    out_color, out_depth, out_alpha, out_norm = planes[0:3], planes[3:4], planes[4:5], planes[5:8]
    radii = alloc((P,), dtype=torch.int32, device=dev)
    out_extra = alloc((F, H, W), **fopt) if F > 0 else torch.empty(0, **fopt)
    # the per-pixel output and the state its backward reads
    side = ()
    if depth_quantile is not None:
        side = (alloc((1, H, W), **fopt), alloc((H, W), dtype=torch.int32, device=dev))     # depth_q, depth_q_pos
    elif depth_distortion:
        side = (alloc((1, H, W), **fopt), alloc((2, H, W), **fopt))     # distortion, distortion_state

    if P == 0:
        # the reference short-circuits: zero images, empty scratch (rasterize_points.cu:94)
        empty = torch.empty(0, dtype=torch.uint8, device=dev)
        rendered, buffers = 0, (empty, empty.clone(), empty.clone())
    else:
        with torch.cuda.device(dev):
            geom, binning, img = _Arena(dev), _Arena(dev), _Arena(dev)
            keep = []
            M = int(sh.shape[1]) if (sh is not None and sh.numel() != 0) else 0
            a = N.ForwardArgs()
            a.geom_alloc, a.binning_alloc, a.image_alloc = geom.cb, binning.cb, img.cb
            a.P, a.D, a.M, a.ED = P, int(degree), M, F
            a.width, a.height = W, H
            a.background = _ptr(background, keep)
            a.means3D = _ptr(means3D, keep)
            a.shs = _ptr(sh, keep)
            a.colors_precomp = _ptr(colors, keep)
            a.opacities = _ptr(opacity, keep)
            a.scales = _ptr(scales, keep)
            a.scale_modifier = float(scale_modifier)
            a.rotations = _ptr(rotations, keep)
            a.cov3D_precomp = _ptr(cov3Ds_precomp, keep)
            a.norm3D_precomp = _ptr(norm3Ds_precomp, keep)
            a.extra_attrs = _ptr(extra_attrs, keep)
            a.viewmatrix = _ptr(viewmatrix, keep)
            a.projmatrix = _ptr(projmatrix, keep)
            a.cam_pos = _ptr(campos, keep)
            if graph:
                a.tan_fovx, a.tan_fovy, tan_fov = _tan_fov(tan_fovx, tan_fovy, dev)
                a.kernel_size = float(kernel_size)
            else:
                a.tan_fovx, a.tan_fovy, a.kernel_size = float(tan_fovx), float(tan_fovy), float(kernel_size)
            a.prefiltered = int(bool(prefiltered))
            a.out_color, a.out_depth = out_color.data_ptr(), out_depth.data_ptr()
            a.out_norm, a.out_alpha = out_norm.data_ptr(), out_alpha.data_ptr()
            a.out_extra = out_extra.data_ptr() if F > 0 else None
            a.out_norm_raw = norm_raw.data_ptr() if fuse_normalize else None
            if out_peers is not None:
                peer_arr = (C.c_void_p * len(out_peers))(*[int(p) for p in out_peers])
                keep.append(peer_arr)
                a.out_peers = C.cast(peer_arr, C.POINTER(C.c_void_p))
                a.n_out_peers = len(out_peers)
            a.radii = radii.data_ptr()
            a.debug = int(bool(debug))
            a.stream = torch.cuda.current_stream(dev).cuda_stream
            a.capacity_hint = int(capacity_hint)
            if tile_rows is not None:
                a.tile_row_begin, a.tile_row_end = _band(tile_rows)
            # the entry and its arguments after the struct, in the order of precedence of the options
            off = _ptr(subpixel_offset, keep)
            if ray_depth:
                q = depth_quantile is not None
                entry = "sfgs_rasterize_forward_plane_normals" if plane_normals else "sfgs_rasterize_forward_ray_depth"
                args = (off, int(bool(ortho)),
                        float(depth_quantile) if q else 0.0, side[0].data_ptr() if q else None,
                        side[1].data_ptr() if q else None)
            elif depth_quantile is not None:
                entry, args = "sfgs_rasterize_forward_depth_quantile", (off, int(bool(ortho)), float(depth_quantile),
                                                                        side[0].data_ptr(), side[1].data_ptr())
            elif depth_distortion:
                entry, args = "sfgs_rasterize_forward_distortion", (off, int(bool(ortho)), side[0].data_ptr(),
                                                                    side[1].data_ptr())
            elif graph:
                from . import graphs
                entry, args = "sfgs_rasterize_forward_graph", (off, tan_fov.data_ptr() if tan_fov is not None else None,
                                                               graphs.status_word(dev).data_ptr())
            elif ortho:
                entry, args = "sfgs_rasterize_forward_ortho", (off,)
            elif off is not None:
                entry, args = "sfgs_rasterize_forward_subpixel" + ("_peers" if out_peers is not None else ""), (off,)
            else:
                entry, args = "sfgs_rasterize_forward", ()
            rendered = N.check(getattr(L, entry)(C.byref(a), *args), entry)
        rendered, buffers = -1 if graph else rendered, (geom.tensor, binning.tensor, img.tensor)
    return ((rendered, out_color, out_depth, out_norm, out_alpha, radii, out_extra) + buffers +
            (norm_raw,) * bool(fuse_normalize) + side)


def _use_deterministic(has_extra, has_peers):
    """torch.are_deterministic_algorithms_enabled(), checked against the options the deterministic backward lacks:
    those raise as torch's own ops do, or warn under warn_only=True (and the default backward runs)."""
    if not torch.are_deterministic_algorithms_enabled():
        return False
    what = ["extra_attrs"] * has_extra + ["acc_peers"] * has_peers
    if not what:
        return True
    msg = (f"rasterize_gaussians_backward with {' and '.join(what)} does not have a deterministic implementation, but "
           "you set 'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, "
           "or you can use the 'warn_only=True' option, if that's acceptable for your application.")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
        return False
    raise RuntimeError(msg)


@contextlib.contextmanager
def _no_fill(on):
    """Deterministic mode makes torch.empty fill new memory (torch.utils.deterministic.fill_uninitialized_memory).
    Every buffer the backward allocates is written by its kernels before it is read, so with `on` that fill of the
    outputs and the scratch (about 1.2 GB for a 1080p frame of 1M Gaussians) is skipped."""
    fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.utils.deterministic.fill_uninitialized_memory = fill and not on
    try:
        yield
    finally:
        torch.utils.deterministic.fill_uninitialized_memory = fill


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, extra_attrs, scale_modifier,
                                 cov3Ds_precomp, norm3Ds_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                 kernel_size, dL_dout_color, dL_dout_depth, dL_dout_norm, dL_dout_alpha,
                                 dL_dout_extra, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer,
                                 out_alpha, debug, tile_rows=None, norm_raw=None, phase=0, acc=None,
                                 gauss_range=None, acc_peers=None, peer_slice=0, subpixel_offset=None,
                                 camera_grad=False, intrinsics_grad=False, graph=False, *, ortho=False,
                                 depth_q_pos=None, dL_dout_depth_q=None, distortion_state=None,
                                 dL_dout_distortion=None, ray_depth=False, plane_normals=False):
    """Same positional signature and return tuple as the reference's `_C.rasterize_gaussians_backward`.  With
    `norm_raw` (the extra tensor a `fuse_normalize=True` forward returned) `dL_dout_norm` is taken w.r.t. the unit
    normal map and the adjoint of F.normalize is applied inside the blend-adjoint kernel.

    Two-phase form for the tile-row sharded multi-GPU mode (include/sfgs.h): `phase=1` runs only the blend adjoint
    of this rank's band and returns the [P,16] sums (`acc`, allocated here unless given); `phase=2` runs only the
    per-Gaussian adjoint for `gauss_range=(begin, end)` from `acc`, whose row 0 is Gaussian `begin` (e.g. a
    reduce-scatter result), and returns the usual tuple with rows [begin, end) valid.

    Under `torch.use_deterministic_algorithms(True)` the call runs the deterministic backward
    (sfgs_rasterize_backward_deterministic): the same outputs up to the order of the sums, bit-identical from run to
    run.  `extra_attrs` and `acc_peers` have no deterministic implementation: they raise, or with `warn_only=True`
    warn and run the default backward.

    `subpixel_offset`: the tensor the forward was given (sfgs_rasterize_backward_subpixel and its deterministic form);
    no gradient is formed with respect to it.  It combines with both phases and with `acc_peers` (through
    sfgs_rasterize_backward_subpixel_peers).

    `camera_grad=True` (one-call backward only): the same call through sfgs_rasterize_backward_camera, which also forms
    the camera gradients; the tuple then ends with (dL_dviewmatrix [4,4], dL_dprojmatrix [4,4], dL_dcampos [3]), in the
    layout of the inputs.  Every other output is bit-identical to the call without it.

    `camera_grad=True, intrinsics_grad=True`: the same call through sfgs_rasterize_backward_camera_intrinsics, which
    also forms the gradients with respect to the focal lengths; the tuple then ends with the three camera tensors and
    (dL_dtanfovx, dL_dtanfovy), 0-d tensors.  Every other output, the camera tensors included, is bit-identical to the
    call without it.

    `phase=2, camera_grad=True[, intrinsics_grad=True]` (sfgs_rasterize_backward_camera_partial): the tuple ends with
    ONE float64 tensor of 35 [37] camera terms, the unrounded sums over the Gaussians of `gauss_range`.  The ranks of a
    sharded frame add these partials and round once (sfgs.multigpu.reduce_camera_gradients).  The gradient rows are
    bit-identical to the phase-2 call without it.

    `graph=True`: the capture-safe backward (sfgs_rasterize_backward_graph) of a `graph=True` forward; `R` is the
    capacity that forward was given, and `tan_fovx` / `tan_fovy` may be 0-d CUDA tensors.  Every option of the
    one-call backward is taken (offsets, deterministic mode, camera and focal gradients); phases 1 and 2, acc_peers,
    tile_rows and debug raise.

    `ortho=True`: the backward of an `ortho=True` forward (sfgs_rasterize_backward_ortho), with the same settings and
    offsets; the deterministic mode is taken as above.  graph, tile_rows, acc_peers, phases 1 and 2 and camera or
    focal gradients raise SfgsError.

    `depth_q_pos` (the forward's, with `depth_quantile`) and `dL_dout_depth_q` ([1,H,W]): the backward of a depth
    quantile forward (sfgs_rasterize_backward_depth_quantile), which adds dL/d depth_q to the depth gradient of the
    splat each pixel selected.  It takes offsets, `ortho`, the deterministic mode, phase 1, and camera and focal
    gradients (not with `ortho`); graph, tile_rows, acc_peers and extra_attrs raise SfgsError.

    `distortion_state` (the forward's, with `depth_distortion=True`) and `dL_dout_distortion` ([1,H,W]): the backward of
    a depth-distortion forward (sfgs_rasterize_backward_distortion), which adds dL/dR to the blend adjoint's alpha and
    depth terms.  It takes offsets, `ortho`, the deterministic mode, phase 1, and camera and focal gradients (not with
    `ortho`); depth_q_pos, graph, tile_rows, acc_peers and extra_attrs raise SfgsError.

    `ray_depth=True`: the backward of a `ray_depth=True` forward (sfgs_rasterize_backward_ray_depth), with or without
    its depth quantile's `depth_q_pos` / `dL_dout_depth_q`; the depth cotangents then also reach each splat's depth
    slope, and through it its rotation, scale and covariance.  It takes offsets, `ortho`, the deterministic mode,
    phase 1, and camera and focal gradients (not with `ortho`); distortion_state, graph, tile_rows, acc_peers and
    extra_attrs raise SfgsError.

    `plane_normals=True` (with `ray_depth=True`): the backward of a `plane_normals=True` forward
    (sfgs_rasterize_backward_plane_normals); the normal cotangent reaches each splat's plane normal, and through it its
    depth slope, covariance, rotation, scale, mean and the camera and focal terms.  dL_dnorm3D is 0.  It takes what
    `ray_depth=True` takes; without ray_depth it raises, and so do norm3Ds_precomp and everything ray depth rejects."""
    banded = dict(tile_rows=tile_rows is not None, acc_peers=acc_peers is not None)
    has_extra = extra_attrs is not None and extra_attrs.numel() != 0
    if plane_normals:
        _check_plane_normals("rasterize_gaussians_backward(plane_normals=True)", ray_depth, norm3Ds_precomp,
                             distortion_state=distortion_state is not None or dL_dout_distortion is not None,
                             graph=graph, **banded, extra_attrs=has_extra)
    if ray_depth:
        _reject("rasterize_gaussians_backward(ray_depth=True)", RAY_DEPTH,
                distortion_state=distortion_state is not None or dL_dout_distortion is not None, graph=graph, **banded,
                extra_attrs=has_extra)
    dist = _given_together("distortion_state", distortion_state, "dL_dout_distortion", dL_dout_distortion)
    if dist:
        _reject("rasterize_gaussians_backward(distortion_state=...)", DISTORTION,
                depth_q_pos=depth_q_pos is not None or dL_dout_depth_q is not None, graph=graph, **banded,
                extra_attrs=has_extra)
    depth_q = _given_together("depth_q_pos", depth_q_pos, "dL_dout_depth_q", dL_dout_depth_q)
    if depth_q:
        _reject("rasterize_gaussians_backward(depth_q_pos=...)", DEPTH_Q, graph=graph, **banded, extra_attrs=has_extra)
    if ortho:
        _reject("rasterize_gaussians_backward(ortho=True)", ORTHO, graph=graph, **banded,
                **{f"phase={int(phase)}": int(phase) != 0}, camera_grad=camera_grad, intrinsics_grad=intrinsics_grad)
    if intrinsics_grad and not camera_grad:
        raise ValueError("intrinsics_grad=True needs camera_grad=True")
    if graph:
        _reject("rasterize_gaussians_backward(graph=True)", GRAPH,
                **{"debug=True (it synchronises after every stage)": debug}, **banded,
                **{f"phase={int(phase)} (the two-phase backward)": int(phase) != 0})
    H, W = int(dL_dout_color.shape[1]), int(dL_dout_color.shape[2])
    dev = means3D.device
    if subpixel_offset is not None:
        check_subpixel_offset(subpixel_offset, H, W)
    if depth_q:
        _check_pixel_inputs("depth_q_pos", depth_q_pos, torch.int32, (H, W), "dL_dout_depth_q", dL_dout_depth_q,
                            H, W, dev)
    if dist:
        _check_pixel_inputs("distortion_state", distortion_state, torch.float32, (2, H, W), "dL_dout_distortion",
                            dL_dout_distortion, H, W, dev)
    F = int(extra_attrs.shape[1]) if has_extra else 0
    deterministic = _use_deterministic(F > 0, acc_peers is not None)
    L = N.lib()
    P = int(means3D.shape[0])
    M = int(sh.shape[1]) if (sh is not None and sh.numel() != 0) else 0
    fopt = dict(dtype=torch.float32, device=dev)
    ncam = (37 if intrinsics_grad else 35) if camera_grad else 0
    # phase 2 returns the camera terms as one float64 partial, formed by sfgs_rasterize_backward_camera_partial; the
    # quantile and distortion entries take float32 terms (and reject phase 2), and P == 0 returns zeros as a partial
    partial = camera_grad and phase == 2
    alloc = torch.zeros if P == 0 else torch.empty      # the reference returns zero gradients for P == 0

    with _no_fill(deterministic):
        # one allocation for all fixed-width per-Gaussian gradients (every element is written by the kernel)
        widths = dict(means3D=3, means2D=3, colors=3, depths=1, conic=4, opacity=1, cov3D=6, norm3D=3, scales=3, rot=4)
        pad = lambda n: (n + 3) & ~3                       # keep every sub-array 16-byte aligned  # noqa: E731
        flat = alloc((sum(pad(P * w) for w in widths.values()),), **fopt)
        outs, pos = {}, 0
        for k, w in widths.items():
            outs[k] = flat[pos:pos + P * w].view(P, w)
            pos += pad(P * w)
        dL_dsh = alloc((P, M, 3), **fopt)
        dL_dextra = alloc((P, F), **fopt) if F > 0 else torch.empty(0, **fopt)
        f64 = partial and (P == 0 or not (depth_q or dist or ray_depth))
        dL_dcamera = alloc((ncam,), dtype=torch.float64 if f64 else torch.float32, device=dev) if ncam else None
        if P > 0:
            with torch.cuda.device(dev):
                scratch = _Arena(dev)
                keep = []
                a = N.BackwardArgs()
                a.phase = int(phase)
                if acc_peers is not None:
                    # phase 1 with the reduce-scatter fused into the kernel: peer-mapped slice pointers, nothing
                    # allocated here
                    if phase != 1:
                        raise ValueError("acc_peers is a phase-1 option")
                    peer_arr = (C.c_void_p * len(acc_peers))(*[int(p) for p in acc_peers])
                    keep.append(peer_arr)                      # must outlive the call
                    a.acc_peers = C.cast(peer_arr, C.POINTER(C.c_void_p))
                    a.n_peers, a.peer_slice = len(acc_peers), int(peer_slice)
                elif phase == 1 and acc is None:
                    acc = torch.empty((P, 16), **fopt)
                if acc is not None:
                    a.acc = _ptr(acc, keep)
                if gauss_range is not None:
                    a.gauss_begin, a.gauss_end = int(gauss_range[0]), int(gauss_range[1])
                a.P, a.D, a.M, a.R, a.ED = P, int(degree), M, int(R), F
                a.width, a.height = W, H
                a.background = _ptr(background, keep)
                a.means3D = _ptr(means3D, keep)
                a.shs = _ptr(sh, keep)
                a.colors_precomp = _ptr(colors, keep)
                a.scales = _ptr(scales, keep)
                a.scale_modifier = float(scale_modifier)
                a.rotations = _ptr(rotations, keep)
                a.cov3D_precomp = _ptr(cov3Ds_precomp, keep)
                a.norm3D_precomp = _ptr(norm3Ds_precomp, keep)
                a.extra_attrs = _ptr(extra_attrs, keep)
                a.viewmatrix = _ptr(viewmatrix, keep)
                a.projmatrix = _ptr(projmatrix, keep)
                a.cam_pos = _ptr(campos, keep)
                if graph:
                    a.tan_fovx, a.tan_fovy, tan_fov = _tan_fov(tan_fovx, tan_fovy, dev)
                    a.kernel_size = float(kernel_size)
                else:
                    a.tan_fovx, a.tan_fovy, a.kernel_size = float(tan_fovx), float(tan_fovy), float(kernel_size)
                a.radii = _ptr(radii, keep)
                a.geom_buffer = _ptr(geomBuffer, keep)
                a.binning_buffer = _ptr(binningBuffer, keep)
                a.image_buffer = _ptr(imageBuffer, keep)
                a.accum_alphas = _ptr(out_alpha, keep)
                a.dL_dpix = _ptr(dL_dout_color, keep)
                a.dL_dpix_depth = _ptr(dL_dout_depth, keep)
                a.dL_dpix_norm = _ptr(dL_dout_norm, keep)
                a.dL_dpix_alpha = _ptr(dL_dout_alpha, keep)
                a.norm_raw = _ptr(norm_raw, keep) if norm_raw is not None else None
                a.dL_dpix_extra = _ptr(dL_dout_extra, keep) if F > 0 else None
                a.dL_dmean2D = outs["means2D"].data_ptr()
                a.dL_dconic = outs["conic"].data_ptr()
                a.dL_dopacity = outs["opacity"].data_ptr()
                a.dL_dcolor = outs["colors"].data_ptr()
                a.dL_ddepth = outs["depths"].data_ptr()
                a.dL_dmean3D = outs["means3D"].data_ptr()
                a.dL_dcov3D = outs["cov3D"].data_ptr()
                a.dL_dnorm3D = outs["norm3D"].data_ptr()
                a.dL_dsh = dL_dsh.data_ptr() if M > 0 else None
                a.dL_dscale = outs["scales"].data_ptr()
                a.dL_drot = outs["rot"].data_ptr()
                a.dL_dextra = dL_dextra.data_ptr() if F > 0 else None
                a.scratch_alloc = scratch.cb
                a.debug = int(bool(debug))
                a.stream = torch.cuda.current_stream(dev).cuda_stream
                if tile_rows is not None:
                    a.tile_row_begin, a.tile_row_end = _band(tile_rows)
                # the entry and its arguments after the struct, in the order of precedence of the options
                off = _ptr(subpixel_offset, keep)
                det = int(deterministic)
                cam = dL_dcamera.data_ptr() if ncam else None
                if ray_depth:
                    entry = ("sfgs_rasterize_backward_plane_normals" if plane_normals
                             else "sfgs_rasterize_backward_ray_depth")
                    args = (off, int(bool(ortho)), det, _ptr(depth_q_pos, keep) if depth_q else None,
                            _ptr(dL_dout_depth_q, keep) if depth_q else None, cam, ncam)
                elif depth_q:
                    entry, args = "sfgs_rasterize_backward_depth_quantile", (off, int(bool(ortho)), det,
                                                                             _ptr(depth_q_pos, keep),
                                                                             _ptr(dL_dout_depth_q, keep), cam, ncam)
                elif dist:
                    entry, args = "sfgs_rasterize_backward_distortion", (off, int(bool(ortho)), det,
                                                                         _ptr(distortion_state, keep),
                                                                         _ptr(dL_dout_distortion, keep), cam, ncam)
                elif graph:
                    entry, args = "sfgs_rasterize_backward_graph", (off, det, tan_fov.data_ptr() if tan_fov is not None
                                                                    else None, cam, ncam)
                elif ortho:
                    entry, args = "sfgs_rasterize_backward_ortho", (off, det)
                elif partial:
                    entry, args = "sfgs_rasterize_backward_camera_partial", (off, det, ncam, cam)
                elif camera_grad:
                    entry = "sfgs_rasterize_backward_camera" + ("_intrinsics" if intrinsics_grad else "")
                    args = (off, det, cam)
                elif off is not None:
                    entry = ("sfgs_rasterize_backward_deterministic_subpixel" if deterministic else
                             "sfgs_rasterize_backward_subpixel" + ("_peers" if acc_peers is not None else ""))
                    args = (off,)
                else:
                    entry, args = "sfgs_rasterize_backward" + ("_deterministic" if deterministic else ""), ()
                N.check(getattr(L, entry)(C.byref(a), *args), entry)
                # the arena and its callback form a reference cycle: drop the scratch now (stream-ordered, like any
                # freed tensor) instead of whenever the garbage collector runs — the deterministic path's scratch is
                # ~0.5 KB per tile instance
                scratch.tensor = None
            if phase == 1:
                return acc      # None when the sums went straight to the peers' slices
    ret = (outs["means2D"], outs["colors"], outs["opacity"], outs["means3D"], outs["cov3D"], outs["norm3D"],
           dL_dsh, outs["scales"], outs["rot"], dL_dextra)
    if not ncam:
        return ret
    if partial:
        return ret + (dL_dcamera,)
    ret += (dL_dcamera[0:16].view(4, 4), dL_dcamera[16:32].view(4, 4), dL_dcamera[32:35])
    return ret + (dL_dcamera[35], dL_dcamera[36]) if intrinsics_grad else ret


def mark_visible(means3D, viewmatrix, projmatrix):
    L = N.lib()
    P = int(means3D.shape[0])
    present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
    if P != 0:
        keep = []
        with torch.cuda.device(means3D.device):
            N.check(L.sfgs_mark_visible(P, _ptr(means3D, keep), _ptr(viewmatrix, keep), _ptr(projmatrix, keep),
                                        present.data_ptr(), torch.cuda.current_stream(means3D.device).cuda_stream),
                    "sfgs_mark_visible")
    return present
