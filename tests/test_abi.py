"""The C-ABI library loads and exports every symbol include/sfgs.h declares (no GPU needed)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "sfgs.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(sfgs_[a-z0-9_]+)\s*\(", src))
    return sorted(n for n in names if not n.endswith("_fn"))


def test_header_symbols_exported():
    from sfgs import native
    L = native.lib()
    names = header_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/sfgs.h but not exported by libsfgs.so"
    assert set(native.EXPORTS) == set(names), set(native.EXPORTS) ^ set(names)


def test_struct_sizes_match_c():
    from sfgs import native
    L = native.lib()
    for which, st in enumerate((native.ForwardArgs, native.BackwardArgs, native.GeomView, native.ImageView,
                                native.BinningView)):
        assert L.sfgs_sizeof(which) == C.sizeof(st)


def test_version_and_layout_sizes():
    from sfgs import native
    L = native.lib()
    assert L.sfgs_version() == 4
    g1, g2 = L.sfgs_geom_bytes(1000), L.sfgs_geom_bytes(2000)
    assert 1000 * (64 + 24 + 1 + 4) <= g1 < g2
    assert L.sfgs_image_bytes(1920, 1080) >= 1920 * 1080 * 4 + 8160 * 12   # n_contrib + ranges + tile histogram
    assert L.sfgs_binning_bytes(1000) >= 1000 * (4 + 1 + 8 + 8)
    assert L.sfgs_geom_bytes(0) > 0


def test_error_paths_without_gpu():
    """Argument validation happens before any CUDA call."""
    from sfgs import native
    L = native.lib()
    assert L.sfgs_rasterize_forward(None) == -2
    assert L.sfgs_rasterize_backward(None) == -2
    a = native.ForwardArgs()
    a.P, a.width, a.height = 10, 0, 16
    assert L.sfgs_rasterize_forward(C.byref(a)) == -2
    assert "bad sizes" in native.last_error()
    assert L.sfgs_mark_visible(-1, None, None, None, None, None) == -2
    assert L.sfgs_mark_visible(0, None, None, None, None, None) == 0
    assert L.sfgs_fusedssim_forward(1e-4, 9e-4, 0, 3, 8, 8, None, None, 1, None, None, None, None, None) == 0
    assert L.sfgs_fusedssim_forward(1e-4, 9e-4, 1, 3, 8, 8, None, None, 1, None, None, None, None, None) == -2


def test_new_option_validation_without_gpu():
    """ABI v2 options are validated before any CUDA work: backward phases, peer tables, fused activations."""
    from sfgs import native
    L = native.lib()
    b = native.BackwardArgs()
    b.P, b.width, b.height = 8, 32, 32
    dummy = (C.c_float * 64)()
    ptr = C.cast(dummy, C.c_void_p)          # the struct mirrors declare raw pointers as c_void_p
    b.geom_buffer = b.binning_buffer = b.image_buffer = C.cast(dummy, C.c_void_p)
    b.phase = 3
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2 and "phase" in native.last_error()
    b.phase = 1                                   # phase 1 needs the pixel cotangents and a caller-owned acc (or peers)
    for f in ("dL_dpix", "dL_dpix_depth", "dL_dpix_norm", "dL_dpix_alpha", "accum_alphas"):
        setattr(b, f, ptr)
    b.ED = 35                                     # more extra channels than SFGS_MAX_EXTRA
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2 and "ED out of range" in native.last_error()
    b.ED = 0
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2 and "acc" in native.last_error()
    peers = (C.c_void_p * 2)(C.cast(dummy, C.c_void_p), C.cast(dummy, C.c_void_p))
    b.acc_peers, b.n_peers, b.peer_slice = C.cast(peers, C.POINTER(C.c_void_p)), 2, 3     # 2*3 < P
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2 and "acc_peers" in native.last_error()
    b.n_peers, b.peer_slice = 9, 4                                                          # more than 8 peers
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2
    b.phase, b.n_peers = 0, 2                                                               # peers are a phase-1 option
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2
    # forward: peer frame blocks are limited to 8
    a = native.ForwardArgs()
    a.P, a.width, a.height = 8, 32, 32
    a.out_peers, a.n_out_peers = C.cast(peers, C.POINTER(C.c_void_p)), 9
    assert L.sfgs_rasterize_forward(C.byref(a)) == -2
    # fused activations
    assert L.sfgs_activations_forward(0, None, None, None, None, None, None, None, None) == 0
    assert L.sfgs_activations_forward(4, None, None, None, None, None, None, None, None) == -2
    assert L.sfgs_activations_backward(-1, None, None, None, None, None, None, None, None, None, None, None) == -2
    assert L.sfgs_activations_backward(4, None, None, None, None, None, None, None, None, None, None, None) == -2


def test_activation_wrapper_rejects_cpu_tensors():
    import torch
    from sfgs.activations import fused_activations
    with pytest.raises(ValueError, match="CUDA float32"):
        fused_activations(torch.zeros(4, 1), torch.zeros(4, 3), torch.zeros(4, 4), torch.zeros(4, 1, dtype=torch.float64))


def test_python_wrapper_validation():
    import torch
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    z = torch.zeros(4, 4)
    rs = GaussianRasterizationSettings(16, 16, 1.0, 1.0, 0.1, torch.zeros(1), torch.zeros(3), 1.0, z, z, 3,
                                       torch.zeros(3), False, False)
    assert rs._fields == ("image_height", "image_width", "tanfovx", "tanfovy", "kernel_size", "subpixel_offset", "bg",
                          "scale_modifier", "viewmatrix", "projmatrix", "sh_degree", "campos", "prefiltered", "debug")
    r = GaussianRasterizer(rs)
    m = torch.zeros(5, 3)
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(m, m, torch.zeros(5, 1), scales=m, rotations=torch.zeros(5, 4))
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(m, m, torch.zeros(5, 1), shs=torch.zeros(5, 16, 3), colors_precomp=m, scales=m, rotations=torch.zeros(5, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(m, m, torch.zeros(5, 1), shs=torch.zeros(5, 16, 3))
    with pytest.raises(ValueError):
        r(m, m, torch.zeros(5, 1), shs=torch.zeros(5, 16, 3), cov3Ds_precomp=torch.zeros(5, 6))
    from sfgs import rasterizer
    with pytest.raises(RuntimeError, match="num_points, 3"):
        rasterizer.rasterize_gaussians(torch.zeros(3), torch.zeros(5, 2), m, m, m, m, 1.0, m, m, m, 0, z, z, 1.0, 1.0,
                                       0.1, 16, 16, m, 3, torch.zeros(3), False, False)


def test_sibling_packages_import():
    import fused_ssim
    import simple_knn._C as knn
    assert callable(fused_ssim.fused_ssim) and callable(knn.distCUDA2)
