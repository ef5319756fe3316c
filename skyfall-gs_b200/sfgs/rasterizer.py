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


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier,
                        cov3Ds_precomp, norm3Ds_precomp, extra_attrs, attr_degree, viewmatrix, projmatrix,
                        tan_fovx, tan_fovy, kernel_size, image_height, image_width, sh, degree, campos,
                        prefiltered, debug, capacity_hint=0, tile_rows=None, fuse_normalize=False, out_planes=None,
                        out_peers=None, subpixel_offset=None):
    """Same positional signature and return tuple as the reference's `_C.rasterize_gaussians`.  With
    `fuse_normalize=True` the returned normal map is already F.normalize(., dim=0) (the reference's torch post-op,
    diff_gauss/__init__.py:48) and the un-normalised blend is appended to the tuple for the backward.

    `subpixel_offset` ([H,W,2] CUDA float32, or None): pixel (x, y) samples the splats at (x + off[y,x,0],
    y + off[y,x,1]) (sfgs_rasterize_forward_subpixel); the backward must be given the same tensor.  Offsets must be
    finite; a NaN or Inf raises.  They combine with `tile_rows` and `out_peers`: every rank passes the whole frame's
    offsets, and the bands reassemble the one-call frame bit for bit (with `out_peers` through
    sfgs_rasterize_forward_subpixel_peers)."""
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    H, W, F = int(image_height), int(image_width), int(attr_degree)
    if subpixel_offset is not None:
        check_subpixel_offset(subpixel_offset, H, W)
    L = N.lib()
    P = int(means3D.shape[0])
    dev = means3D.device
    fopt = dict(dtype=torch.float32, device=dev)

    if P == 0:
        # the reference short-circuits: zero images, empty scratch (rasterize_points.cu:94)
        out_extra = torch.zeros((F, H, W), **fopt) if F > 0 else torch.empty(0, **fopt)
        empty = torch.empty(0, dtype=torch.uint8, device=dev)
        ret = (0, torch.zeros((NUM_CHANNELS, H, W), **fopt), torch.zeros((1, H, W), **fopt),
               torch.zeros((3, H, W), **fopt), torch.zeros((1, H, W), **fopt),
               torch.zeros((P,), dtype=torch.int32, device=dev), out_extra, empty, empty.clone(), empty.clone())
        return ret + (torch.zeros((3, H, W), **fopt),) if fuse_normalize else ret

    with torch.cuda.device(dev):
        # one allocation for the 8 image planes: colour(3) depth(1) alpha(1) normal(3)
        # multi-GPU tile-row mode: `out_planes` is this rank's symmetric [8,H,W] frame block and `out_peers` the
        # peer-mapped pointers of every rank's block; the blend kernel then stores the band into all of them
        if out_planes is not None:
            planes = out_planes.view(8, H, W)
            norm_raw = torch.empty((3, H, W), **fopt) if fuse_normalize else None
        else:
            planes = torch.empty((11 if fuse_normalize else 8, H, W), **fopt)
            norm_raw = planes[8:11] if fuse_normalize else None
        out_color, out_depth, out_alpha, out_norm = planes[0:3], planes[3:4], planes[4:5], planes[5:8]
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        out_extra = torch.empty((F, H, W), **fopt) if F > 0 else torch.empty(0, **fopt)

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
        if subpixel_offset is not None:
            entry = "sfgs_rasterize_forward_subpixel" + ("_peers" if out_peers is not None else "")
            rendered = N.check(getattr(L, entry)(C.byref(a), _ptr(subpixel_offset, keep)), entry)
        else:
            rendered = N.check(L.sfgs_rasterize_forward(C.byref(a)), "sfgs_rasterize_forward")
    ret = (rendered, out_color, out_depth, out_norm, out_alpha, radii, out_extra,
           geom.tensor, binning.tensor, img.tensor)
    return ret + (norm_raw,) if fuse_normalize else ret


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
                                 camera_grad=False, intrinsics_grad=False):
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
    bit-identical to the phase-2 call without it."""
    if intrinsics_grad and not camera_grad:
        raise ValueError("intrinsics_grad=True needs camera_grad=True")
    if subpixel_offset is not None:
        check_subpixel_offset(subpixel_offset, int(dL_dout_color.shape[1]), int(dL_dout_color.shape[2]))
    F = int(extra_attrs.shape[1]) if (extra_attrs is not None and extra_attrs.numel() != 0) else 0
    deterministic = _use_deterministic(F > 0, acc_peers is not None)
    L = N.lib()
    P = int(means3D.shape[0])
    H, W = int(dL_dout_color.shape[1]), int(dL_dout_color.shape[2])
    M = int(sh.shape[1]) if (sh is not None and sh.numel() != 0) else 0
    dev = means3D.device
    fopt = dict(dtype=torch.float32, device=dev)

    if P == 0:
        z = lambda *s: torch.zeros(s, **fopt)  # noqa: E731
        ret = (z(P, 3), z(P, 3), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, M, 3), z(P, 3), z(P, 4),
               z(P, F) if F > 0 else torch.empty(0, **fopt))
        if camera_grad and phase == 2:
            return ret + (torch.zeros((37 if intrinsics_grad else 35,), dtype=torch.float64, device=dev),)
        if camera_grad:
            ret += (z(4, 4), z(4, 4), z(3))
        return ret + (z(), z()) if intrinsics_grad else ret

    with torch.cuda.device(dev), _no_fill(deterministic):
        # one allocation for all fixed-width per-Gaussian gradients (every element is written by the kernel)
        widths = dict(means3D=3, means2D=3, colors=3, depths=1, conic=4, opacity=1, cov3D=6, norm3D=3, scales=3, rot=4)
        pad = lambda n: (n + 3) & ~3                       # keep every sub-array 16-byte aligned  # noqa: E731
        flat = torch.empty((sum(pad(P * w) for w in widths.values()),), **fopt)
        outs, off = {}, 0
        for k, w in widths.items():
            outs[k] = flat[off:off + P * w].view(P, w)
            off += pad(P * w)
        dL_dsh = torch.empty((P, M, 3), **fopt) if M > 0 else torch.zeros((P, 0, 3), **fopt)
        dL_dextra = torch.empty((P, F), **fopt) if F > 0 else torch.empty(0, **fopt)
        scratch = _Arena(dev)
        keep = []
        a = N.BackwardArgs()
        a.phase = int(phase)
        if acc_peers is not None:
            # phase 1 with the reduce-scatter fused into the kernel: peer-mapped slice pointers, nothing allocated here
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
        if camera_grad and phase == 2:
            ncam = 37 if intrinsics_grad else 35
            dL_dcamera = torch.empty((ncam,), dtype=torch.float64, device=dev)
            off = _ptr(subpixel_offset, keep) if subpixel_offset is not None else None
            N.check(L.sfgs_rasterize_backward_camera_partial(C.byref(a), off, int(deterministic), ncam,
                                                             dL_dcamera.data_ptr()),
                    "sfgs_rasterize_backward_camera_partial")
        elif camera_grad:
            dL_dcamera = torch.empty((37 if intrinsics_grad else 35,), **fopt)
            off = _ptr(subpixel_offset, keep) if subpixel_offset is not None else None
            entry = "sfgs_rasterize_backward_camera_intrinsics" if intrinsics_grad else "sfgs_rasterize_backward_camera"
            N.check(getattr(L, entry)(C.byref(a), off, int(deterministic), dL_dcamera.data_ptr()), entry)
        elif subpixel_offset is not None:
            off = _ptr(subpixel_offset, keep)
            if deterministic:
                N.check(L.sfgs_rasterize_backward_deterministic_subpixel(C.byref(a), off),
                        "sfgs_rasterize_backward_deterministic_subpixel")
            else:
                entry = "sfgs_rasterize_backward_subpixel" + ("_peers" if acc_peers is not None else "")
                N.check(getattr(L, entry)(C.byref(a), off), entry)
        elif deterministic:
            N.check(L.sfgs_rasterize_backward_deterministic(C.byref(a)), "sfgs_rasterize_backward_deterministic")
        else:
            N.check(L.sfgs_rasterize_backward(C.byref(a)), "sfgs_rasterize_backward")
        # the arena and its callback form a reference cycle: drop the scratch now (stream-ordered, like any freed
        # tensor) instead of whenever the garbage collector runs — the deterministic path's scratch is ~0.5 KB per
        # tile instance
        scratch.tensor = None
    if phase == 1:
        return acc      # None when the sums went straight to the peers' slices
    ret = (outs["means2D"], outs["colors"], outs["opacity"], outs["means3D"], outs["cov3D"], outs["norm3D"],
           dL_dsh, outs["scales"], outs["rot"], dL_dextra)
    if camera_grad and phase == 2:
        return ret + (dL_dcamera,)
    if camera_grad:
        ret += (dL_dcamera[0:16].view(4, 4), dL_dcamera[16:32].view(4, 4), dL_dcamera[32:35])
    if intrinsics_grad:
        ret += (dL_dcamera[35], dL_dcamera[36])
    return ret


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
