"""sfgs — Python host side of the H100-native splat rasterizer.

`sfgs.native` binds the C ABI (include/sfgs.h) with ctypes; `sfgs.rasterizer`
implements, on top of it, the three functions of the reference's pybind module
`diff_gauss._C` with identical names, argument orders and return tuples
(RAST/ext.cpp:15-18, RAST/rasterize_points.h:17-78).  PyTorch is used for
device memory and streams only.
"""
from . import native  # noqa: F401
