"""Stand-in for the reference's compiled module `diff_gauss._C` (RAST/ext.cpp:15-18).

Exposes the same three callables with the same positional signatures; the work
is done by libsfgs.so through the C ABI in include/sfgs.h.
"""
from sfgs import rasterizer as _R
from sfgs.rasterizer import mark_visible, rasterize_gaussians, rasterize_gaussians_backward  # noqa: F401
from sfgs.native import SfgsError  # noqa: F401
from sfgs.native import lib as _lib


def rasterize_gaussians_fused(*args, **kw):
    """`rasterize_gaussians` with the F.normalize post-op fused into the blend kernel; returns the reference's
    10-tuple (normal map already unit length) + the un-normalised blend needed by the backward.  The fused pair looks
    sfgs.rasterizer's functions up at each call, so sfgs.ortho, which runs through them, sees what that module holds."""
    return _R.rasterize_gaussians(*args, fuse_normalize=True, **kw)


def rasterize_gaussians_backward_fused(*args, norm_raw, **kw):
    return _R.rasterize_gaussians_backward(*args, norm_raw=norm_raw, **kw)


_lib()  # fail at import time if the CUDA library has not been built
