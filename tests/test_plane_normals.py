"""Plane normals: sfgs_rasterize_forward_plane_normals / sfgs_rasterize_backward_plane_normals and the Python surface on
top of them (rasterize_gaussians(ray_depth=True, plane_normals=True), diff_gauss.GaussianRasterizer(settings,
ray_depth=True, plane_normals=True), sfgs.ortho.OrthoRasterizer(settings, ray_depth=True, plane_normals=True)).

Record i's normal is that of its ray-depth plane, n = sigma u / |u| with u = w3 - g_x T0 - g_y T1 (g the ray-depth slope,
T0, T1 the rows of T = J W, w3 the view's depth row), flipped toward the camera.  The oracles: a float64 evaluation of u
from the GPU's cov3D, the float64 walk of tests/test_ray_depth.py for the normal map, tests/plane_normal_chain_f64.py
for the per-Gaussian stage, central differences, the shortest-axis normal of flat splats at kernel_size 0, and scenes
of known geometry."""
import ctypes as C
import json
import math
import os
import subprocess
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if _p not in sys.path:     # the child process of the rejection test starts bare
        sys.path.insert(0, _p)

import helpers as Hh  # noqa: E402
from helpers import bits, release_cached_frames  # noqa: F401,E402

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4
EPS32 = 2.0 ** -24


# ----------------------------------------------------------------------------- rejections (no device)
def _rejections():
    """{case: [code, message]} of both entries for every rejected case; run in a child with no visible device."""
    from sfgs import native as N
    L = N.lib()
    buf = (C.c_double * 4096)()
    ptr = C.addressof(buf)
    peer_tab = (C.c_void_p * 2)(ptr, ptr)
    peers = C.cast(peer_tab, C.POINTER(C.c_void_p))
    alloc = N.ALLOC_FN(lambda _u, _n: None)

    def fwd_args(**kw):
        a = N.ForwardArgs()
        a.geom_alloc = a.binning_alloc = a.image_alloc = alloc
        a.P, a.D, a.M, a.width, a.height = 8, 3, 16, 32, 32
        for f in ("background", "means3D", "shs", "opacities", "scales", "rotations", "viewmatrix", "projmatrix",
                  "cam_pos", "out_color", "out_depth", "out_norm", "out_alpha", "radii"):
            setattr(a, f, ptr)
        a.tan_fovx = a.tan_fovy = 0.5
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    def bwd_args(**kw):
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
        for k, v in kw.items():
            setattr(b, k, v)
        return b

    def fwd(a, q=0.5, dq=None, pos=None, off=None, ortho=0):
        return L.sfgs_rasterize_forward_plane_normals(None if a is None else C.byref(a), off, ortho, q, dq, pos)

    def bwd(b, pos=None, g=None, ncam=0, cam=ptr, det=0, off=None, ortho=0):
        return L.sfgs_rasterize_backward_plane_normals(None if b is None else C.byref(b), off, ortho, det, pos, g, cam,
                                                       ncam)

    cases = {
        "fwd null args": lambda: fwd(None),
        "fwd quantile null pos": lambda: fwd(fwd_args(), dq=ptr),
        "fwd quantile q=0": lambda: fwd(fwd_args(), q=0.0, dq=ptr, pos=ptr),
        "fwd quantile q=nan": lambda: fwd(fwd_args(), q=float("nan"), dq=ptr, pos=ptr),
        "fwd quantile bad q before ED": lambda: fwd(fwd_args(ED=2), q=1.0, dq=ptr, pos=ptr),
        "fwd ED=2": lambda: fwd(fwd_args(ED=2, extra_attrs=ptr, out_extra=ptr)),
        "fwd ED=2 quantile": lambda: fwd(fwd_args(ED=2, extra_attrs=ptr, out_extra=ptr), dq=ptr, pos=ptr),
        "fwd band": lambda: fwd(fwd_args(tile_row_begin=0, tile_row_end=1)),
        "fwd out_peers": lambda: fwd(fwd_args(out_peers=peers, n_out_peers=2)),
        "fwd out_peers before norm3D_precomp": lambda: fwd(fwd_args(out_peers=peers, n_out_peers=2,
                                                                    norm3D_precomp=ptr)),
        "fwd norm3D_precomp": lambda: fwd(fwd_args(norm3D_precomp=ptr)),
        "fwd norm3D_precomp ortho": lambda: fwd(fwd_args(norm3D_precomp=ptr, tan_fovx=-1.0), ortho=1),
        "fwd ED with offsets": lambda: fwd(fwd_args(ED=2), off=ptr),
        "fwd ortho bad extent": lambda: fwd(fwd_args(tan_fovx=-1.0), ortho=1),
        "fwd bad sizes": lambda: fwd(fwd_args(width=0)),
        "fwd null output": lambda: fwd(fwd_args(out_depth=None)),
        "fwd misaligned rotations": lambda: fwd(fwd_args(rotations=ptr + 4)),
        "bwd null args": lambda: bwd(None),
        "bwd pos without cotangent": lambda: bwd(bwd_args(), pos=ptr),
        "bwd cotangent without pos": lambda: bwd(bwd_args(), g=ptr),
        **{f"bwd ncam={n}": (lambda n=n: bwd(bwd_args(), ncam=n)) for n in (-1, 1, 36, 38)},
        "bwd ncam before ED": lambda: bwd(bwd_args(ED=2), ncam=36),
        "bwd ED=2": lambda: bwd(bwd_args(ED=2, extra_attrs=ptr, dL_dextra=ptr, dL_dpix_extra=ptr)),
        "bwd band": lambda: bwd(bwd_args(tile_row_begin=0, tile_row_end=1)),
        "bwd acc_peers": lambda: bwd(bwd_args(acc_peers=peers, n_peers=1, peer_slice=8, phase=1, acc=ptr)),
        "bwd phase 2": lambda: bwd(bwd_args(phase=2, acc=ptr, gauss_begin=0, gauss_end=8)),
        "bwd ncam=35 phase 1": lambda: bwd(bwd_args(phase=1, acc=ptr), ncam=35),
        "bwd ncam=37 ortho": lambda: bwd(bwd_args(), ncam=37, ortho=1),
        "bwd ncam=37 ortho before norm3D_precomp": lambda: bwd(bwd_args(norm3D_precomp=ptr), ncam=37, ortho=1),
        "bwd norm3D_precomp": lambda: bwd(bwd_args(norm3D_precomp=ptr)),
        "bwd norm3D_precomp ortho phase 1": lambda: bwd(bwd_args(norm3D_precomp=ptr, phase=1, acc=ptr), ortho=1),
        "bwd ortho phase 1": lambda: bwd(bwd_args(phase=1, acc=ptr), ortho=1),
        "bwd ncam=35 null dL_dcamera": lambda: bwd(bwd_args(), ncam=35, cam=None),
        "bwd ncam=37 null scratch": lambda: bwd(bwd_args(scratch_alloc=N.ALLOC_FN()), ncam=37),
        "bwd det null radii": lambda: bwd(bwd_args(radii=None), det=1),
        "bwd bad sizes": lambda: bwd(bwd_args(height=-1)),
        "bwd null pixel gradient": lambda: bwd(bwd_args(dL_dpix=None)),
    }
    return {name: [call(), N.last_error()] for name, call in cases.items()}


_FWD, _BWD = "forward_plane_normals", "backward_plane_normals"
_BAD_Q = "the quantile must be finite with 0 < q < 1"
_NULL_IN = "null depth_q_pos or dL_dpix_depth_q"
_NORM = "norm3D_precomp is not supported with plane normals"
EXPECTED = {
    "fwd null args": (SFGS_E_BADARG, _FWD, "null args"),
    "fwd quantile null pos": (SFGS_E_BADARG, _FWD, "null out_depth_q_pos"),
    "fwd quantile q=0": (SFGS_E_BADARG, _FWD, _BAD_Q),
    "fwd quantile q=nan": (SFGS_E_BADARG, _FWD, _BAD_Q),
    "fwd quantile bad q before ED": (SFGS_E_BADARG, _FWD, _BAD_Q),
    "fwd ED=2": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with plane normals"),
    "fwd ED=2 quantile": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with plane normals"),
    "fwd band": (SFGS_E_UNSUPPORTED, _FWD, "tile-row bands are not supported with plane normals"),
    "fwd out_peers": (SFGS_E_UNSUPPORTED, _FWD, "out_peers are not supported with plane normals"),
    "fwd out_peers before norm3D_precomp": (SFGS_E_UNSUPPORTED, _FWD, "out_peers are not supported with plane normals"),
    "fwd norm3D_precomp": (SFGS_E_UNSUPPORTED, _FWD, _NORM),
    "fwd norm3D_precomp ortho": (SFGS_E_UNSUPPORTED, _FWD, _NORM),
    "fwd ED with offsets": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with plane normals"),
    "fwd ortho bad extent": (SFGS_E_BADARG, _FWD, "the half-extents tan_fovx, tan_fovy must be finite and > 0"),
    "fwd bad sizes": (SFGS_E_BADARG, _FWD, "bad sizes"),
    "fwd null output": (SFGS_E_BADARG, _FWD, "null output"),
    "fwd misaligned rotations": (SFGS_E_BADARG, _FWD, "rotations must be 16-byte aligned"),
    "bwd null args": (SFGS_E_BADARG, _BWD, "null args"),
    "bwd pos without cotangent": (SFGS_E_BADARG, _BWD, _NULL_IN),
    "bwd cotangent without pos": (SFGS_E_BADARG, _BWD, _NULL_IN),
    **{f"bwd ncam={n}": (SFGS_E_BADARG, _BWD, "ncam must be 0, 35 or 37") for n in (-1, 1, 36, 38)},
    "bwd ncam before ED": (SFGS_E_BADARG, _BWD, "ncam must be 0, 35 or 37"),
    "bwd ED=2": (SFGS_E_UNSUPPORTED, _BWD, "extra_attrs are not supported with plane normals"),
    "bwd band": (SFGS_E_UNSUPPORTED, _BWD, "tile-row bands are not supported with plane normals"),
    "bwd acc_peers": (SFGS_E_UNSUPPORTED, _BWD, "acc_peers are not supported with plane normals"),
    "bwd phase 2": (SFGS_E_UNSUPPORTED, _BWD, "phase 2 is not supported with plane normals"),
    "bwd ncam=35 phase 1": (SFGS_E_UNSUPPORTED, _BWD,
                            "camera gradients are formed by the one-call backward (phase 0) only"),
    "bwd ncam=37 ortho": (SFGS_E_UNSUPPORTED, _BWD, "the orthographic camera has no camera gradients"),
    "bwd ncam=37 ortho before norm3D_precomp": (SFGS_E_UNSUPPORTED, _BWD,
                                                "the orthographic camera has no camera gradients"),
    "bwd norm3D_precomp": (SFGS_E_UNSUPPORTED, _BWD, _NORM),
    "bwd norm3D_precomp ortho phase 1": (SFGS_E_UNSUPPORTED, _BWD, _NORM),
    "bwd ortho phase 1": (SFGS_E_UNSUPPORTED, _BWD,
                          "phases 1 and 2 (the two-phase backward) are not supported with an orthographic camera"),
    "bwd ncam=35 null dL_dcamera": (SFGS_E_BADARG, _BWD, "null dL_dcamera"),
    "bwd ncam=37 null scratch": (SFGS_E_BADARG, _BWD, "null scratch allocator"),
    "bwd det null radii": (SFGS_E_BADARG, _BWD, "radii missing"),
    "bwd bad sizes": (SFGS_E_BADARG, _BWD, "bad sizes"),
    "bwd null pixel gradient": (SFGS_E_BADARG, _BWD, "null pixel gradient"),
}


def test_entry_rejections_before_any_cuda_work():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert set(got) == set(EXPECTED)
    for name, (code, entry, what) in EXPECTED.items():
        assert got[name] == [code, f"{entry}: {what}"], (name, got[name])


def test_python_layer_rejects_before_native_calls(monkeypatch):
    from sfgs import native as N
    from sfgs import rasterizer as R

    def no_lib():
        raise AssertionError("native library called")
    monkeypatch.setattr(N, "lib", no_lib)
    m = torch.zeros((4, 3))
    e = torch.empty(0)
    nrm = torch.zeros((4, 3))

    def fwd(rd=True, **kw):
        return R.rasterize_gaussians(e, m, e, e, e, e, 1.0, e, kw.pop("nrm", e), e, kw.pop("F", 0), e, e, 1.0, 1.0,
                                     0.1, 8, 8, e, 0, e, False, False, ray_depth=rd, plane_normals=True, **kw)
    with pytest.raises(N.SfgsError, match="plane normals .* need ray_depth=True"):
        fwd(rd=False)
    for kw, what in ((dict(depth_distortion=True), "depth_distortion"), (dict(graph=True), "graph"),
                     (dict(tile_rows=(0, 1)), "tile_rows"), (dict(out_peers=[0]), "out_peers"),
                     (dict(F=2), "extra_attrs"), (dict(nrm=nrm), "norm3Ds_precomp")):
        with pytest.raises(N.SfgsError, match=f"plane_normals=True.*{what}.*not supported with plane normals"):
            fwd(**kw)
    g = torch.zeros((3, 8, 8))

    def bwd(rd=True, **kw):
        return R.rasterize_gaussians_backward(
            e, m, e, e, e, e, kw.pop("ex", e), 1.0, e, kw.pop("nrm", e), e, e, 1.0, 1.0, 0.1, g, g[:1], g, g[:1], e, e,
            0, e, e, 0, e, e, e, False, ray_depth=rd, plane_normals=True, **kw)
    with pytest.raises(N.SfgsError, match="plane normals .* need ray_depth=True"):
        bwd(rd=False)
    for kw, what in ((dict(distortion_state=torch.zeros((2, 8, 8)), dL_dout_distortion=g[:1]), "distortion_state"),
                     (dict(graph=True), "graph"), (dict(tile_rows=(0, 1)), "tile_rows"),
                     (dict(acc_peers=[0], phase=1), "acc_peers"), (dict(ex=torch.zeros((4, 2))), "extra_attrs"),
                     (dict(nrm=nrm), "norm3Ds_precomp")):
        with pytest.raises(N.SfgsError, match=f"plane_normals=True.*{what}.*not supported with plane normals"):
            bwd(**kw)
    # ray depth's own messages are unchanged without the option
    with pytest.raises(N.SfgsError, match="graph not supported with ray depth"):
        R.rasterize_gaussians(e, m, e, e, e, e, 1.0, e, e, e, 0, e, e, 1.0, 1.0, 0.1, 8, 8, e, 0, e, False, False,
                              graph=True, ray_depth=True)


def test_modules_reject_before_native_calls(monkeypatch):
    """diff_gauss and OrthoRasterizer raise on plane normals without ray depth and with the distortion, and diff_gauss
    raises under stream capture (naming plane normals) before any capture-time work."""
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from sfgs import native as N
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer

    def no_lib():
        raise AssertionError("native library called")
    monkeypatch.setattr(N, "lib", no_lib)
    m = torch.zeros((4, 3))
    kw = dict(shs=torch.zeros((4, 16, 3)), scales=torch.ones((4, 3)), rotations=torch.zeros((4, 4)))
    rs = GaussianRasterizationSettings(8, 8, 1.0, 1.0, 0.1, None, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3,
                                       torch.zeros(3), False, False)
    ors = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3, False,
                                     False)
    for mod in (lambda **k: GaussianRasterizer(rs, **k), lambda **k: OrthoRasterizer(ors, **k)):
        with pytest.raises(N.SfgsError, match="need ray_depth=True"):
            mod(plane_normals=True)(m, m, torch.ones((4, 1)), **kw)
        with pytest.raises(N.SfgsError, match="depth_distortion together with plane_normals"):
            mod(depth_distortion=True, ray_depth=True, plane_normals=True)(m, m, torch.ones((4, 1)), **kw)
        # norm3Ds_precomp reaches the rasterizer's check (which names plane normals) before any native call
        with pytest.raises(N.SfgsError, match="norm3Ds_precomp not supported with plane normals"):
            mod(ray_depth=True, plane_normals=True)(m, m, torch.ones((4, 1)), **kw, norm3Ds_precomp=torch.zeros((4, 3)))

    def no_capacity(*a, **k):
        raise AssertionError("capture-time work before the plane normals' check")
    monkeypatch.setattr(diff_gauss._graphs, "resolve_capacity", no_capacity)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    mc = types.SimpleNamespace(is_cuda=True)
    with pytest.raises(N.SfgsError, match="plane normals cannot be captured"):
        diff_gauss._RasterizeGaussians.forward(types.SimpleNamespace(), mc, m, m, m, m, m, m, m, m, torch.empty(0),
                                               rs, False, None, None, None, None, None, None, False, None, False, True,
                                               True)


def test_modules_keep_the_option():
    import diff_gauss
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer
    rs = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, False, False)
    r = OrthoRasterizer(rs, ray_depth=True, plane_normals=True)
    assert r.plane_normals and r.to("cpu") is r
    g = diff_gauss.GaussianRasterizer(None, ray_depth=True, plane_normals=True)
    assert g.plane_normals and not diff_gauss.GaussianRasterizer(None).plane_normals


# ----------------------------------------------------------------------------- the entry each combination reaches
def _recording(monkeypatch):
    import test_ray_depth as RD
    from sfgs import native as N
    rec = RD._Recorder()
    monkeypatch.setattr(N, "lib", lambda: rec)
    RD._cuda_free_ptr(monkeypatch)
    return rec


@pytest.mark.parametrize("ortho", [False, True])
@pytest.mark.parametrize("offsets", [False, True])
@pytest.mark.parametrize("quantile", [None, 0.5])
def test_forward_entry_and_arguments(monkeypatch, ortho, offsets, quantile):
    from sfgs import rasterizer as R
    rec = _recording(monkeypatch)
    H, W, P = 8, 8, 4
    m = torch.zeros((P, 3))
    e = torch.empty(0)
    off = torch.zeros((H, W, 2)) if offsets else None
    calls = []
    for pn in (False, True):
        out = R.rasterize_gaussians(torch.zeros(3), m, e, torch.ones(P, 1), torch.ones(P, 3), torch.ones(P, 4), 1.0,
                                    e, e, e, 0, torch.eye(4), torch.eye(4), 1.0, 1.0, 0.1, H, W,
                                    torch.zeros(P, 16, 3), 3, torch.zeros(3), False, False, subpixel_offset=off,
                                    ortho=ortho, depth_quantile=quantile, ray_depth=True, plane_normals=pn)
        calls.append(out)
    assert [c[0] for c in rec.calls] == ["sfgs_rasterize_forward_ray_depth", "sfgs_rasterize_forward_plane_normals"]
    (_, a0), (_, a1) = rec.calls
    out = calls[1]
    assert a1[0] == (off.data_ptr() if offsets else None) and a1[1] == int(ortho)
    assert len(out) == len(calls[0])
    if quantile is None:
        assert a1[2] == 0.0 and a1[3] is None and a1[4] is None and len(out) == 10
    else:
        assert a1[2] == 0.5 and a1[3] == out[10].data_ptr() and a1[4] == out[11].data_ptr()
        assert tuple(out[10].shape) == (1, H, W) and out[11].dtype == torch.int32
    assert a0[:2] == a1[:2] and a0[2] == a1[2]


@pytest.mark.parametrize("ortho,ncam", [(False, 0), (False, 35), (False, 37), (True, 0)])
@pytest.mark.parametrize("offsets", [False, True])
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("quantile", [False, True])
def test_backward_entry_and_arguments(monkeypatch, ortho, ncam, offsets, det, quantile):
    from sfgs import rasterizer as R
    rec = _recording(monkeypatch)
    H, W, P = 8, 8, 4
    m = torch.zeros((P, 3))
    e = torch.empty(0)
    g = torch.zeros((3, H, W))
    off = torch.zeros((H, W, 2)) if offsets else None
    qkw = dict(depth_q_pos=torch.zeros((H, W), dtype=torch.int32), dL_dout_depth_q=torch.zeros((1, H, W))) \
        if quantile else {}
    monkeypatch.setattr(R, "_check_pixel_inputs", lambda *a: None)
    with Hh.deterministic(det):
        out = R.rasterize_gaussians_backward(
            torch.zeros(3), m, torch.ones(P, dtype=torch.int32), e, torch.ones(P, 3), torch.ones(P, 4), e, 1.0, e, e,
            torch.eye(4), torch.eye(4), 1.0, 1.0, 0.1, g, g[:1], g, g[:1], e, torch.zeros(P, 16, 3), 3, torch.zeros(3),
            torch.zeros(8, dtype=torch.uint8), 5, torch.zeros(8, dtype=torch.uint8), torch.zeros(8, dtype=torch.uint8),
            g[:1], False, subpixel_offset=off, ortho=ortho, camera_grad=ncam > 0, intrinsics_grad=ncam == 37,
            ray_depth=True, plane_normals=True, **qkw)
    assert len(rec.calls) == 1
    entry, args = rec.calls[0]
    assert entry == "sfgs_rasterize_backward_plane_normals"
    assert args[0] == (off.data_ptr() if offsets else None) and args[1] == int(ortho) and args[2] == int(det)
    if quantile:
        assert args[3] == qkw["depth_q_pos"].data_ptr() and args[4] == qkw["dL_dout_depth_q"].data_ptr()
    else:
        assert args[3] is None and args[4] is None
    assert args[6] == ncam and (args[5] is None) == (ncam == 0)
    assert len(out) == 10 + (3 if ncam else 0) + (2 if ncam == 37 else 0)


# ----------------------------------------------------------------------------- the restatement on CPU
def _case(seed, P=6, ortho=False):
    import test_ray_depth as RD
    torch.manual_seed(seed)
    W, H, tanx, tany = 96, 64, 0.6, 0.4
    view, proj = RD._pinhole(W, H, tanx, tany)
    if ortho:
        from sfgs.ortho import projection_matrix
        tanx, tany = 3.0, 2.0
        proj = view @ projection_matrix(tanx, tany, 0.01, 100.0).double()
    f = lambda *s: torch.randn(*s, dtype=torch.float64)  # noqa: E731
    m, sc, q = f(P, 3) * 0.5, f(P, 3).abs() * 0.2 + 0.05, f(P, 4)
    return W, H, tanx, tany, view, proj, m, sc, q, f


@pytest.mark.parametrize("ortho,focal,colors", [(False, False, False), (False, True, False), (True, False, False),
                                                (False, True, True)])
def test_chain_without_plane_normals_is_ray_depth_chain(ortho, focal, colors):
    """plane_normal_chain_f64.chain without the keyword returns ray_depth_chain_f64.chain's results bit for bit (every
    key, with and without ray depth)."""
    import plane_normal_chain_f64 as PC
    import ray_depth_chain_f64 as RC
    W, H, tx, ty, view, proj, m, sc, q, f = _case(5, ortho=ortho)
    P = m.shape[0]
    acc = f(P, 16)
    vis = torch.tensor([True, True, False, True, True, True])
    clamped = torch.rand(P, 3) < 0.3
    shs = None if colors else f(P, 16, 3) * 0.3
    for rd in (False, True):
        kw = dict(scales=sc, rotations=q, norm_rec=f(P, 3), ortho=ortho, focal=focal, ray_depth=rd)
        args = (acc, vis, m, torch.rand(P, dtype=torch.float64), clamped, shs, 3, view.float(), proj.float(),
                torch.tensor([0.1, -0.2, -6.0]), W, H, tx, ty, 0.1)
        a, b = RC.chain(*args, **kw), PC.chain(*args, **kw)
        assert set(a) == set(b)
        for k in a:
            if isinstance(a[k], torch.Tensor):
                assert torch.equal(a[k], b[k]), k
            elif isinstance(a[k], tuple):
                assert all(torch.equal(x, y) for x, y in zip(a[k], b[k])), k
            else:
                assert a[k] == b[k], k


def plane_normal_f64(m, sc, q, view, W, H, tanx, tany, ks, campos=None, ortho=False):
    """Independent float64 forward of the plane normal n [n,3] of Gaussians (m, sc, q) under a row-vector view."""
    import chain_f64 as CH
    t = m @ view[:3, :3] + view[3, :3]
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    n_ = m.shape[0]
    J = torch.zeros((n_, 2, 3), dtype=torch.float64)
    if ortho:
        J[:, 0, 0], J[:, 1, 1] = fx, fy
    else:
        limx, limy = 1.3 * tanx, 1.3 * tany
        z = t[:, 2]
        tx = torch.clamp(t[:, 0] / z, -limx, limx) * z
        ty = torch.clamp(t[:, 1] / z, -limy, limy) * z
        J[:, 0, 0], J[:, 0, 2] = fx / z, -fx * tx / (z * z)
        J[:, 1, 1], J[:, 1, 2] = fy / z, -fy * ty / (z * z)
    T = J @ view[:3, :3].T
    Sig = CH.sym6_to_mat(CH.cov3d(sc, CH.quat_to_rot(q)))
    cov2 = T @ Sig @ T.transpose(1, 2) + ks * torch.eye(2, dtype=torch.float64)
    w3 = view[:3, 2]
    s = torch.einsum("i,gij,gkj->gk", w3, Sig, T)
    g = torch.linalg.solve(cov2, s.unsqueeze(-1)).squeeze(-1)
    u = w3 - (g.unsqueeze(-1) * T).sum(1)
    d = w3.expand_as(u) if ortho else m - campos
    sgn = torch.where((d * u).sum(1) > 0, -1.0, 1.0).to(u.dtype)
    return sgn[:, None] * u / u.norm(dim=1, keepdim=True)


@pytest.mark.parametrize("ortho", [False, True])
def test_chain_plane_normals_matches_central_differences(ortho):
    """plane_normal_chain_f64.chain(ray_depth=True, plane_normals=True)'s means3D / scales / rotations gradients, and
    for the pinhole camera its viewmatrix and tan_fovx / tan_fovy gradients (exact=True), are those of sum c . n with
    n evaluated independently (plane_normal_f64); every acc word but the normal's 4-6 is 0."""
    import plane_normal_chain_f64 as PC
    W, H, tanx, tany, view, proj, m, sc, q, f = _case(3, P=5, ortho=ortho)
    P = m.shape[0]
    acc = torch.zeros((P, 16), dtype=torch.float64)
    acc[:, 4:7] = f(P, 3)
    vis = torch.ones(P, dtype=torch.bool)
    campos = torch.tensor([0.0, 0.0, -6.0], dtype=torch.float64)
    ks = float(torch.tensor(0.1, dtype=torch.float32))
    vw = view.float().double()
    n0 = plane_normal_f64(m, sc, q, vw, W, H, tanx, tany, ks, campos, ortho)
    r = PC.chain(acc, vis, m, torch.ones(P), torch.zeros(P, 3, dtype=torch.bool), None, 0, view.float(), proj.float(),
                 campos.float(), W, H, tanx, tany, 0.1, scales=sc, rotations=q, norm_rec=n0, ortho=ortho,
                 focal=not ortho, exact=True, ray_depth=True, plane_normals=True)
    assert torch.allclose(r["plane_normal"], n0, atol=1e-12)
    assert int((r["norm3D"] != 0).sum()) == 0

    def L(m_=m, sc_=sc, q_=q, vw_=vw, tx_=tanx, ty_=tany):
        return float((acc[:, 4:7] * plane_normal_f64(m_, sc_, q_, vw_, W, H, tx_, ty_, ks, campos, ortho)).sum())

    h = 1e-6
    checks = [("means3D", "m_", m), ("scales", "sc_", sc), ("rot", "q_", q)]
    if not ortho:
        checks.append(("view", "vw_", vw))
    for name, arg, v in checks:
        fd = torch.zeros_like(v)
        for i in range(v.numel()):
            if name == "view" and (i % 4 == 3):
                continue                  # the 4th column of the row-vector view is not read
            e = torch.zeros(v.numel(), dtype=v.dtype)
            e[i] = h
            e = e.view_as(v)
            fd.view(-1)[i] = (L(**{arg: v + e}) - L(**{arg: v - e})) / (2 * h)
        gv = r[name].reshape(fd.shape)
        assert torch.allclose(gv, fd, rtol=1e-5, atol=1e-6 * float(fd.abs().max())), (name, (gv - fd).abs().max())
    if not ortho:
        for name, arg, v in (("tanx", "tx_", tanx), ("tany", "ty_", tany)):
            fd = (L(**{arg: v + h}) - L(**{arg: v - h})) / (2 * h)
            assert abs(float(r[name]) - fd) <= 1e-5 * max(abs(fd), 1e-3), (name, float(r[name]), fd)


def test_zero_dilation_flat_surfel_identity():
    """kernel_size = 0 and a flat splat (scale_z = 0): the plane normal is the splat's shortest-axis normal up to sign,
    in float64 over 2000 random cameras and surfels."""
    import chain_f64 as CH
    g = torch.Generator().manual_seed(17)
    worst = 0.0
    for _ in range(20):
        n_ = 100
        # a random rotation of the pinhole view of RD._pinhole, and surfels in front of it
        Q = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))[0]
        view = torch.eye(4, dtype=torch.float64)
        view[:3, :3] = Q
        cam_c = torch.randn(3, generator=g, dtype=torch.float64) * 2
        view[3, :3] = -cam_c @ Q
        tanx, tany = 0.3 + 0.5 * float(torch.rand(1, generator=g)), 0.3 + 0.4 * float(torch.rand(1, generator=g))
        dirs = torch.stack([(torch.rand(n_, generator=g, dtype=torch.float64) - 0.5) * 2 * tanx,
                            (torch.rand(n_, generator=g, dtype=torch.float64) - 0.5) * 2 * tany,
                            torch.ones(n_, dtype=torch.float64)], 1)
        z = 2 + 20 * torch.rand(n_, 1, generator=g, dtype=torch.float64)
        m = (dirs * z) @ Q.T + cam_c
        sc = torch.rand(n_, 3, generator=g, dtype=torch.float64) * 0.5 + 0.05
        sc[:, 2] = 0.0
        q = torch.randn(n_, 4, generator=g, dtype=torch.float64)
        q = q / q.norm(dim=1, keepdim=True)          # a rotation: Sigma's null space is R's third column
        n = plane_normal_f64(m, sc, q, view, 640, 480, tanx, tany, 0.0, cam_c)
        axis = CH.quat_to_rot(q)[:, :, 2]
        axis = axis / axis.norm(dim=1, keepdim=True)
        worst = max(worst, float((1 - (n * axis).sum(1).abs()).max()))
    print(f"\n[plane normals kernel_size=0] worst 1 - |cos| {worst:.2e} over 2000 flat surfels")
    assert worst <= 1e-12


# ----------------------------------------------------------------------------- GPU helpers
def _run(d, cam, D, bg, plane=True, ks=0.1, **kw):
    from sfgs import rasterizer as R
    e = torch.empty(0, device=d["means3D"].device)
    out = R.rasterize_gaussians(bg, d["means3D"], kw.pop("colors", e), d["opacities"], d["scales"], d["rotations"],
                                1.0, e, e, e, 0, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, ks,
                                cam.height, cam.width, d["shs"] if "shs" in d else e, D, d["campos"], False, False,
                                ray_depth=True, plane_normals=plane, **kw)
    return dict(zip(Hh.FWD_KEYS, out[:10])), out[10:]


def _headline_form(dev, form):
    import test_ray_depth as RD
    cam, D, d, bg = RD._headline(dev)
    cam, d, kw = RD._form(form, cam, d, dev)
    return cam, D, d, bg, kw


# ----------------------------------------------------------------------------- GPU: no interference
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pinhole", "jitter", "ortho"])
def test_no_interference_forward(cuda_device, form):
    """Colour, alpha, depth, depth_q and its positions, n_contrib, radii, binning and record words 0-10 and 14-15 are
    bit-identical to the ray_depth=True call; words 11-13 (the normal) differ."""
    dev = cuda_device
    cam, D, d, bg, kw = _headline_form(dev, form)
    a, sa = _run(d, cam, D, bg, plane=False, depth_quantile=0.5, **kw)
    b, sb = _run(d, cam, D, bg, depth_quantile=0.5, **kw)
    for k in ("color", "depth", "alpha", "radii"):
        assert torch.equal(bits(a[k]), bits(b[k])), k
    assert torch.equal(bits(sa[0]), bits(sb[0])) and torch.equal(sa[1], sb[1])
    assert a["num_rendered"] == b["num_rendered"] > 0
    P = d["means3D"].shape[0]
    Ia, Ib = Hh.our_internals(a, P, cam.height, cam.width), Hh.our_internals(b, P, cam.height, cam.width)
    for k in ("n_contrib", "point_list", "ranges", "keys"):
        assert torch.equal(Ia[k], Ib[k]), k
    vis = a["radii"] > 0
    assert torch.equal(bits(Ia["rec"][vis, :11]), bits(Ib["rec"][vis, :11]))
    assert torch.equal(bits(Ia["rec"][vis, 14:16]), bits(Ib["rec"][vis, 14:16]))
    assert not torch.equal(Ia["rec"][vis, 11:14], Ib["rec"][vis, 11:14])
    nn = Ib["rec"][vis, 11:14].double().norm(dim=1)
    assert float((nn - 1).abs().max()) <= 1e-6 and not torch.equal(a["norm"], b["norm"])


@pytest.mark.gpu
@pytest.mark.parametrize("form,ncam", [("pinhole", 0), ("pinhole", 35), ("pinhole", 37), ("jitter", 37),
                                       ("ortho", 0)])
def test_no_interference_deterministic_backward(cuda_device, form, ncam):
    """With a zero normal cotangent the ten deterministic gradients and the camera / focal terms of the plane-normal
    backward (on its forward's buffers) equal those of the ray-depth backward (on the ray-depth forward's).  Tensors
    that are not equal as values are named: the PLANE instantiation of the per-Gaussian adjoint adds terms (zero here)
    to the conic, dL/dT and dL/dw3 sums, and the compiler contracts the products around them into FMAs differently.
    Each such tensor is held to the float32 rounding scale of that gradient on this frame: the worst difference
    between float32 and float64 evaluations of tests/ray_depth_chain_f64.py (the camera terms: 4 eps of the sum of
    their terms' magnitudes, as in tests/test_ray_depth.py)."""
    import ray_depth_chain_f64 as RC
    dev = cuda_device
    cam, D, d, bg, kw = _headline_form(dev, form)
    fa, _ = _run(d, cam, D, bg, plane=False, **kw)
    fb, _ = _run(d, cam, D, bg, **kw)
    g = torch.Generator(device=dev).manual_seed(1)
    H, W = cam.height, cam.width
    cot = (torch.randn((3, H, W), generator=g, device=dev), torch.randn((1, H, W), generator=g, device=dev),
           torch.zeros((3, H, W), device=dev), torch.randn((1, H, W), generator=g, device=dev))
    off = kw.get("subpixel_offset")
    kw.update(camera_grad=ncam > 0, intrinsics_grad=ncam == 37)
    a = Hh.run_ours_backward(d, cam, D, bg, fa, cot, det=True, ray_depth=True, **kw)
    b = Hh.run_ours_backward(d, cam, D, bg, fb, cot, det=True, ray_depth=True, plane_normals=True, **kw)
    assert set(a) == set(b)
    differ = [k for k in a if not torch.equal(a[k], b[k])]
    cam_keys = ("view", "proj", "campos", "tanx", "tany")
    report = []
    if differ:
        ri = Hh.restatement_inputs(fa, d, cam, D, bg, cot, off=off)
        # the blend adjoint's sums (phase 1, which the orthographic entries do not offer; the blend adjoint does not
        # read the camera)
        ri["acc"] = Hh.run_ours_backward(d, cam, D, bg, fa, cot, det=True, phase=1, subpixel_offset=off,
                                         ray_depth=True)
        ri.update(cov3D=None, scales=d["scales"], rotations=d["rotations"])
        focal = form != "ortho"
        r64 = RC.chain(**ri, ortho=form == "ortho", focal=focal, dtype=torch.float64, ray_depth=True)
        r32 = RC.chain(**ri, ortho=form == "ortho", focal=focal, dtype=torch.float32, ray_depth=True)
        for k in differ:
            diff = float((a[k].double() - b[k].double()).abs().max())
            if k in cam_keys:
                flat = lambda r: torch.cat([r[j].reshape(-1) for j in cam_keys if j in r]).double()  # noqa: E731
                ratio = float(((flat(a) - flat(b)).abs()
                               / (4 * EPS32 * r64["abs"][:flat(a).numel()].double() + 1e-30)).max())
            else:
                lim = float((r32[k].double() - r64[k].double()).abs().max()) + 1e-30
                ratio = diff / lim
            report.append((k, diff, ratio, int((a[k] != b[k]).sum())))
    print(f"\n[plane normals no interference {form} ncam={ncam}] tensors not equal: "
          + (", ".join(f"{k} (max |diff| {dd:.2e}, {n} elements, {r:.3f} of its bound)" for k, dd, r, n in report)
             or "none"))
    assert all(r <= 1.0 for _, _, r, _ in report), report


# ----------------------------------------------------------------------------- GPU: normal words and map
def _normal_bound(d, I, idx, cam, ortho):
    """float64 plane normals of records idx from the GPU's cov3D, and the per-record bound of the GPU's words: g's
    bound of tests/test_ray_depth.py (64 eps |C| (|w3| |Sigma| |T|)) moves u by |dg| |T|, and n by twice that over |u|,
    plus 16 eps for the normalisation."""
    import test_ray_depth as RD
    Sig, T, w3 = RD._sigma_and_view(d, I, idx, cam, ortho=ortho)
    Cm = I["rec"][idx][:, [2, 3, 3, 4]].double().reshape(-1, 2, 2)
    s = torch.einsum("i,gij,gkj->gk", w3, Sig, T)
    g = (Cm @ s.unsqueeze(-1)).squeeze(-1)
    u = w3 - (g.unsqueeze(-1) * T).sum(1)
    m = d["means3D"][idx].double()
    dv = w3.expand_as(u) if ortho else m - d["campos"].double()
    side = (dv * u).sum(1)
    n = torch.where(side > 0, -1.0, 1.0).to(u.dtype)[:, None] * u / u.norm(dim=1, keepdim=True)
    s_mag = torch.einsum("i,gij,gkj->gk", w3.abs(), Sig.abs(), T.abs())
    glim = 64 * EPS32 * (Cm.abs() @ s_mag.unsqueeze(-1)).squeeze(-1)
    lim = 2 * (glim * T.norm(dim=2)).sum(1) / u.norm(dim=1) + 16 * EPS32
    # a footprint seen edge-on may take either sign within rounding
    sure = side.abs() > 4 * lim * dv.norm(dim=1) * u.norm(dim=1)
    return n, lim, sure


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pinhole", "jitter", "ortho"])
def test_normal_words_and_map(cuda_device, form):
    """The normal words of every visible record against the float64 plane normal (from the GPU's cov3D and conic),
    within _normal_bound; and the normal map on 96 random tiles against the float64 sum of w n over the forward's
    applied set: |err| <= (8 n + 16) eps sum |w n| per pixel and channel."""
    import test_ray_depth as RD
    dev = cuda_device
    cam, D, d, bg, kw = _headline_form(dev, form)
    off = kw.get("subpixel_offset")
    W, H = cam.width, cam.height
    f, _ = _run(d, cam, D, bg, **kw)
    P = d["means3D"].shape[0]
    I = Hh.our_internals(f, P, H, W)
    vis = torch.nonzero(f["radii"] > 0).flatten()
    n64, lim, sure = _normal_bound(d, I, vis, cam, form == "ortho")
    gpu = I["rec"][vis, 11:14].double()
    ratio_n = float((((gpu - n64).abs().max(1).values / lim)[sure]).max())
    rec = I["rec"].double()
    tiles = torch.randperm(I["ranges"].shape[0], generator=torch.Generator().manual_seed(7))[:96].tolist()
    worst, npix = 0.0, 0
    for tile in tiles:
        pid, px, py = RD._tile_pixels(tile, W, H, dev, off)
        M, near, r0, r1, _ = RD._applied(I, tile, pid, px, py)
        if r1 == r0:
            continue
        pl = I["point_list"][r0:r1].long()
        w, *_ = RD._composite(rec, pl, M, px, py, torch.float64)
        ref = w @ rec[pl][:, 11:14]
        n = M.sum(1).double()
        lim_m = (8 * n + 16)[:, None] * EPS32 * (w @ rec[pl][:, 11:14].abs()) + 1e-30
        got = f["norm"].reshape(3, -1)[:, pid].T.double()
        ok = ~near
        if ok.any():
            worst = max(worst, float(((got - ref).abs() / lim_m)[ok].max()))
        npix += int(ok.sum())
    print(f"\n[plane normals {form}] normal words worst err / bound {ratio_n:.3f} over {int(sure.sum())} of "
          f"{vis.numel()} records; normal map worst err / bound {worst:.3f} over {npix} pixels")
    assert int(sure.sum()) >= 0.99 * vis.numel()
    assert ratio_n <= 1.0 and worst <= 1.0


@pytest.mark.gpu
def test_zero_dilation_flat_surfels(cuda_device):
    """kernel_size = 0 and flat splats (scale_z = 0): the plane-normal words equal the shortest-axis words of the
    ray_depth=True call up to the float32 bound of _normal_bound plus 8 eps for the shortest-axis words, over
    well-conditioned footprints (smaller 2D eigenvalue >= 1 px^2, condition number <= 100)."""
    import test_ray_depth as RD
    dev = cuda_device
    scene, cam, d = RD._small_case(dev, seed=9, P=4000)
    d = dict(d, scales=d["scales"].clone(), rotations=torch.nn.functional.normalize(d["rotations"], dim=1))
    d["scales"][:, 2] = 0.0
    bg = torch.zeros(3, device=dev)
    a, _ = _run(d, cam, scene.sh_degree, bg, plane=False, ks=0.0)
    b, _ = _run(d, cam, scene.sh_degree, bg, ks=0.0)
    P = d["means3D"].shape[0]
    Ia, Ib = Hh.our_internals(a, P, cam.height, cam.width), Hh.our_internals(b, P, cam.height, cam.width)
    vis = torch.nonzero(b["radii"] > 0).flatten()
    Cm = Ib["rec"][vis][:, [2, 3, 3, 4]].double().reshape(-1, 2, 2)
    ev = torch.linalg.eigvalsh(torch.linalg.inv(Cm))
    good = (ev[:, 0] >= 1.0) & (ev[:, 1] <= 100 * ev[:, 0])
    _, lim, sure = _normal_bound(d, Ib, vis, cam, False)
    good &= sure
    na, nb = Ia["rec"][vis, 11:14].double(), Ib["rec"][vis, 11:14].double()
    err = (na - nb).abs().max(1).values / (lim + 8 * EPS32)
    print(f"\n[plane normals kernel_size=0 flat] {int(good.sum())} of {vis.numel()} well-conditioned records; worst "
          f"err / bound {float(err[good].max()):.3f}; median |n_plane - n_axis| {float((na - nb).abs()[good].median()):.2e}")
    assert int(good.sum()) >= 100
    assert float(err[good].max()) <= 1.0


# ----------------------------------------------------------------------------- GPU: gradients against the restatement
def _chain_case(dev):
    def make():
        import plane_normal_chain_f64 as PC
        import test_ray_depth as RD
        from sfgs import synthetic as S
        cam, D, d, _ = RD._headline(dev)
        bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
        f, side = _run(d, cam, D, bg, depth_quantile=0.5)
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=6)]
        cq = torch.randn((1, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(8), device=dev)
        bkw = dict(depth_q_pos=side[1], dL_dout_depth_q=cq, ray_depth=True, plane_normals=True)
        a = Hh.restatement_inputs(f, d, cam, D, bg, cot)
        a["acc"] = Hh.run_ours_backward(d, cam, D, bg, f, cot, det=True, phase=1, **bkw)
        a.update(cov3D=None, scales=d["scales"], rotations=d["rotations"])
        r64 = PC.chain(**a, focal=True, dtype=torch.float64, ray_depth=True, plane_normals=True)
        r32 = PC.chain(**a, focal=True, dtype=torch.float32, ray_depth=True, plane_normals=True)
        return cam, D, d, bg, f, cot, bkw, r64, r32
    return Hh.cached("chain", "jax004-plane-normals", make)


@pytest.mark.gpu
@pytest.mark.parametrize("ncam", [0, 35, 37])
def test_gradients_against_restatement(cuda_device, ncam):
    """The ten gradients and the camera / focal terms of the deterministic backward with every cotangent plus depth_q's,
    against plane_normal_chain_f64.chain(ray_depth=True, plane_normals=True) on the same sums, with ray depth's bar:
    four times the float32 restatement's error (+1e-6 of the largest value) for the gradients, twice it (or 1e-6 of the
    terms' magnitude) for the camera terms.  dL_dnorm3D is 0."""
    import test_ray_depth as RD
    cam, D, d, bg, f, cot, bkw, r64, r32 = _chain_case(cuda_device)
    g = Hh.run_ours_backward(d, cam, D, bg, f, cot, det=True, camera_grad=ncam > 0, intrinsics_grad=ncam == 37, **bkw)
    assert int((g["norm3D"] != 0).sum()) == 0
    worst = {}
    for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rot"):
        ref, ref32 = r64[k].double(), r32[k].double()
        ours = g[k].detach().double().reshape(ref.shape)
        lim = 4.0 * float((ref32 - ref).abs().max()) + 1e-6 * float(ref.abs().max())
        worst[k] = float((ours - ref).abs().max()) / lim
    print(f"\n[plane normals chain ncam={ncam}] worst err / bound per gradient: "
          + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), (ncam, worst)
    if ncam:
        gpu = torch.cat([g["view"].reshape(16), g["proj"].reshape(16), g["campos"].reshape(3)]
                        + ([g["tanx"].reshape(1), g["tany"].reshape(1)] if ncam == 37 else [])).double()
        f64, f32 = RD._camera_flat(r64, ncam), RD._camera_flat(r32, ncam)
        tol = torch.maximum(2.0 * (f32 - f64).abs(), 1e-6 * r64["abs"][:ncam].double())
        err = (gpu - f64).abs()
        print(f"[plane normals chain ncam={ncam}] camera max err / tol {float((err / tol.clamp_min(1e-300)).max()):.3f}")
        assert (err <= tol).all(), (ncam, err, tol)


# ----------------------------------------------------------------------------- GPU: finite differences
@pytest.mark.gpu
def test_finite_differences(cuda_device):
    """d/d means3D, scales, rotations and tan_fovx of sum c . normal_map (the blended, un-normalised normals) on a small
    scene against central differences, over the pixels whose applied set is the same at -eps, 0 and +eps."""
    import test_ray_depth as RD
    dev = cuda_device
    scene, cam, d = RD._small_case(dev, seed=6)
    bg = torch.zeros(3, device=dev)
    W, H, D = cam.width, cam.height, scene.sh_degree
    P = d["means3D"].shape[0]
    tag = torch.rand(P, generator=torch.Generator(device=dev).manual_seed(1), device=dev, dtype=torch.float64)

    def fwd(m, s, q, tanx=cam.tanfovx):
        c = types.SimpleNamespace(width=W, height=H, tanfovx=tanx, tanfovy=cam.tanfovy)
        return _run(dict(d, means3D=m, scales=s, rotations=q), c, D, bg)[0]

    def applied_sets(out):
        I = Hh.our_internals(out, P, H, W)
        h = torch.zeros(H * W, dtype=torch.float64, device=dev)
        for tile in range(I["ranges"].shape[0]):
            pid, px, py = RD._tile_pixels(tile, W, H, dev)
            M, near, r0, r1, _ = RD._applied(I, tile, pid, px, py)
            if r1 > r0:
                h[pid] = (M.double() * tag[I["point_list"][r0:r1].long()][None, :]).sum(1)
                h[pid[near]] = -1.0
        return h
    f0 = fwd(d["means3D"], d["scales"], d["rotations"])
    set0 = applied_sets(f0)
    c = torch.randn((3, H, W), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    z = torch.zeros_like
    cot = (z(f0["color"]), z(f0["depth"]), c, z(f0["alpha"]))
    bkw = dict(ray_depth=True, plane_normals=True)
    g_all = Hh.run_ours_backward(d, cam, D, bg, f0, cot, det=True, **bkw)
    picks = torch.argsort(g_all["rot"].abs().sum(1), descending=True)[:5].tolist()
    worst = 0.0

    def check(outs, grad_of, what):
        stable = set0 >= 0
        for out in outs:
            stable &= applied_sets(out) == set0
        cm = c * stable.reshape(1, H, W)
        fdv = float(((outs[0]["norm"].double() - outs[1]["norm"].double()) * cm).sum()) / (2 * eps)
        g = Hh.run_ours_backward(d, cam, D, bg, f0, (cot[0], cot[1], cm, cot[3]), det=True, **bkw, **grad_of[1])
        an = float(grad_of[0](g))
        err = abs(an - fdv) / max(abs(fdv), abs(an), 1e-3)
        assert err <= 3e-2, (what, an, fdv)
        return err
    for i in picks:
        for what, k, eps in ([("means3D", k, 1e-3) for k in range(3)] + [("scales", k, 1e-4) for k in range(3)]
                             + [("rot", k, 1e-3) for k in range(4)]):
            outs = []
            for s in (1.0, -1.0):
                v = {"means3D": d["means3D"].clone(), "scales": d["scales"].clone(), "rot": d["rotations"].clone()}
                v[what][i, k] += s * eps
                outs.append(fwd(v["means3D"], v["scales"], v["rot"]))
            worst = max(worst, check(outs, (lambda g, what=what, i=i, k=k: g[what][i, k], {}), (what, i, k)))
    eps = 1e-4
    outs = [fwd(d["means3D"], d["scales"], d["rotations"], cam.tanfovx + s * eps) for s in (1.0, -1.0)]
    worst = max(worst, check(outs, (lambda g: g["tanx"], dict(camera_grad=True, intrinsics_grad=True)), "tanx"))
    print(f"\n[plane normals FD] {len(picks)} Gaussians x (3 means + 3 scales + 4 rotations) and tan_fovx: worst "
          f"relative error {worst:.2e}")


# ----------------------------------------------------------------------------- GPU: geometry
def _roof_views(dev, theta, ext):
    """A nadir orthographic camera over the roof and an oblique pinhole one looking at it from the down-slope side."""
    from sfgs import synthetic as S
    from sfgs.ortho import nadir_camera
    ocam = nadir_camera(-ext, ext, -ext, ext, 0.1, 30.0)
    pcam = S.orbit_camera(elevation_deg=55.0, radius=20.0, fov_deg=40.0, width=320, height=240)
    return ocam, pcam


def _render(means, scales, rots, opac, cam, ortho, dev, plane=True, ks=0.1):
    """(depth, normal map (un-normalised), alpha) of the roof, with the OrthoRasterizer / GaussianRasterizer module."""
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer
    colors = torch.zeros((means.shape[0], 3), device=dev)
    if ortho:
        rs = OrthoRasterizationSettings(cam.image_height, cam.image_width, cam.half_width, cam.half_height, ks,
                                        torch.zeros(3, device=dev), 1.0, cam.viewmatrix.to(dev), cam.projmatrix.to(dev),
                                        0, False, False)
        rast = OrthoRasterizer(rs, ray_depth=True, plane_normals=plane)
    else:
        t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
        rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, ks, None,
                                           torch.zeros(3, device=dev), 1.0, t(cam.viewmatrix), t(cam.projmatrix), 0,
                                           t(cam.campos), False, False)
        rast = GaussianRasterizer(rs, ray_depth=True, plane_normals=plane)
    out = rast(means, torch.zeros_like(means), opac, colors_precomp=colors, scales=scales, rotations=rots)
    return out[1][0], out[2], out[3][0]


def _world_points(depth, alpha, cam, ortho):
    """World points [H,W,3] of the alpha-normalised ray-depth map: unprojected through the camera."""
    dep = depth.double() / alpha.double().clamp_min(1e-12)
    if ortho:
        V = cam.viewmatrix.double().to(depth.device)
        H, W = dep.shape
        ndc_x = (2 * torch.arange(W, dtype=torch.float64, device=depth.device) + 1) / W - 1
        ndc_y = (2 * torch.arange(H, dtype=torch.float64, device=depth.device) + 1) / H - 1
        Y, X = torch.meshgrid(ndc_y * cam.half_height, ndc_x * cam.half_width, indexing="ij")
        tv = torch.stack([X, Y, dep], -1)
    else:
        V = torch.from_numpy(cam.viewmatrix).double().to(depth.device)
        H, W = dep.shape
        ndc_x = (2 * torch.arange(W, dtype=torch.float64, device=depth.device) + 1) / W - 1
        ndc_y = (2 * torch.arange(H, dtype=torch.float64, device=depth.device) + 1) / H - 1
        Y, X = torch.meshgrid(ndc_y * cam.tanfovy, ndc_x * cam.tanfovx, indexing="ij")
        tv = torch.stack([X * dep, Y * dep, dep], -1)
    # t = m V[:3,:3] + V[3,:3]  ->  m = (t - V[3,:3]) V[:3,:3]^-1
    return (tv - V[3, :3]) @ torch.linalg.inv(V[:3, :3])


def _fd_normals(Xw, toward):
    """Unit normals [H-2,W-2,3] of the point map from central differences, flipped to face `toward` (a direction the
    camera looks from, [3] or [H-2,W-2,3])."""
    dx = Xw[1:-1, 2:] - Xw[1:-1, :-2]
    dy = Xw[2:, 1:-1] - Xw[:-2, 1:-1]
    n = torch.linalg.cross(dx, dy)
    n = n / n.norm(dim=-1, keepdim=True).clamp_min(1e-30)
    return torch.where(((n * toward).sum(-1, keepdim=True) < 0), -n, n)


@pytest.mark.gpu
@pytest.mark.parametrize("ortho", [True, False])
def test_sloped_roof(cuda_device, ortho):
    """A roof of thin flat surfels at 30 degrees, seen by a nadir orthographic camera and by an oblique pinhole one.
    In the interior (alpha > 0.99, 3 m from the edges):
      - the normalised plane-normal map is the analytic roof normal (facing the camera) within 1 degree;
      - the finite-difference normal of the rendered (alpha-normalised) ray-depth map agrees with the plane-normal map
        within 3 degrees on average and 10 at worst (the RaDe-GS relation: the map is the normal of the depth rendered);
    the dilation's tilt (kernel_size 0.1) and the blend of neighbouring splats bound the differences."""
    import test_ray_depth as RD
    dev = cuda_device
    theta, sp, ext = math.radians(30.0), 0.5, 12.0
    means, scales, rots, opac = RD._sloped_roof(dev, theta, sp, ext)
    ocam, pcam = _roof_views(dev, theta, ext)
    cam = ocam if ortho else pcam
    depth, nmap, alpha = _render(means, scales, rots, opac, cam, ortho, dev)
    truth = torch.tensor([-math.sin(theta), 0.0, math.cos(theta)], dtype=torch.float64, device=dev)
    if ortho:
        look = cam.viewmatrix.double().to(dev)[:3, 2]
        toward = -look
    else:
        toward = torch.from_numpy(pcam.campos).double().to(dev)
    Xw = _world_points(depth, alpha, cam, ortho)
    if not ortho:
        toward = toward - Xw[1:-1, 1:-1]
        truth_s = torch.where((toward * truth).sum(-1, keepdim=True) < 0, -truth, truth)
    else:
        truth_s = (truth if float(truth @ toward) > 0 else -truth).expand(Xw.shape[0] - 2, Xw.shape[1] - 2, 3)
    n = nmap.permute(1, 2, 0).double()
    n = n / n.norm(dim=-1, keepdim=True).clamp_min(1e-30)
    n = n[1:-1, 1:-1]
    inner = (alpha[1:-1, 1:-1] > 0.99) & (Xw[1:-1, 1:-1, 0].abs() < ext - 3) & (Xw[1:-1, 1:-1, 1].abs() < ext - 3)
    for a_ in (alpha[:-2, 1:-1], alpha[2:, 1:-1], alpha[1:-1, :-2], alpha[1:-1, 2:]):
        inner &= a_ > 0.99
    ang = lambda a, b: torch.rad2deg(torch.arccos((a * b).sum(-1).clamp(-1, 1)))  # noqa: E731
    e_truth = ang(n, truth_s)[inner]
    e_fd = ang(n, _fd_normals(Xw, toward))[inner]
    _, n_ax, _ = _render(means, scales, rots, opac, cam, ortho, dev, plane=False)
    print(f"\n[plane normals roof {'ortho' if ortho else 'pinhole'}] {int(inner.sum())} pixels; plane map vs roof: "
          f"worst {float(e_truth.max()):.3f} deg (mean {float(e_truth.mean()):.3f}); plane map vs depth FD normal: "
          f"worst {float(e_fd.max()):.3f} deg (mean {float(e_fd.mean()):.3f})")
    assert int(inner.sum()) > 1000
    assert float(e_truth.max()) <= 1.0
    assert float(e_fd.mean()) <= 3.0 and float(e_fd.max()) <= 10.0
    assert bool(torch.isfinite(n_ax).all())


@pytest.mark.gpu
def test_rotation_fit_to_roof_normal(cuda_device):
    """Surfels of the 30-degree roof with rotations perturbed by about 20 degrees, under a nadir orthographic camera:
    200 Adam steps on the rotations alone, on the mean over covered pixels of alpha (1 - N . n_roof) with N the
    normalised plane-normal map, bring the mean angle between the map and the roof normal below 1 degree."""
    import test_ray_depth as RD
    dev = cuda_device
    theta, sp, ext = math.radians(30.0), 0.5, 8.0
    means, scales, rots_true, opac = RD._sloped_roof(dev, theta, sp, ext)
    ocam, _ = _roof_views(dev, theta, ext)
    g = torch.Generator(device=dev).manual_seed(2)
    q = (rots_true + 0.18 * torch.randn(rots_true.shape, generator=g, device=dev)).clone().requires_grad_(True)
    truth = torch.tensor([-math.sin(theta), 0.0, math.cos(theta)], device=dev)
    look = ocam.viewmatrix.to(dev)[:3, 2]
    truth = truth if float(truth @ -look) > 0 else -truth

    def angle_and_loss():
        _, nmap, alpha = _render(means, scales, q, opac, ocam, True, dev)
        N = torch.nn.functional.normalize(nmap, dim=0)
        inner = (alpha > 0.99).detach()
        cosv = (N * truth[:, None, None]).sum(0)
        loss = (alpha * (1 - cosv))[inner].mean()
        ang = torch.rad2deg(torch.arccos(cosv.detach().clamp(-1, 1)))[inner].mean()
        return float(ang), loss
    opt = torch.optim.Adam([q], lr=0.01)
    first, _ = angle_and_loss()
    for _ in range(200):
        opt.zero_grad()
        _, loss = angle_and_loss()
        loss.backward()
        assert bool(torch.isfinite(q.grad).all())
        opt.step()
    last, _ = angle_and_loss()
    print(f"\n[plane normals rotation fit] mean angle to the roof normal {first:.3f} -> {last:.3f} deg after 200 Adam "
          "steps on rotations")
    assert first > 5.0 and last <= 1.0


# ----------------------------------------------------------------------------- GPU: composition
@pytest.mark.gpu
def test_diff_gauss_composition(cuda_device, monkeypatch):
    """diff_gauss with offsets, the deterministic mode and camera / focal gradients: six outputs (seven with the
    quantile), every one but the normal bit-identical to the ray_depth=True call; two deterministic runs bit-identical;
    a normal-only loss reaches positions, scales, rotations, opacities, the view and tan_fovx, and not the SH
    coefficients."""
    import diff_gauss
    import test_ray_depth as RD
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam, d = RD._small_case(dev, seed=11)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, seed=4)
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", True)

    def run(pn, view_grad=False, tan_grad=False, det=False, only=False, q=None):
        leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
        view = d["viewmatrix"].clone().requires_grad_(view_grad)
        tanx = torch.tensor(cam.tanfovx, requires_grad=True) if tan_grad else cam.tanfovx
        rs = GaussianRasterizationSettings(cam.height, cam.width, tanx, cam.tanfovy, 0.1, off,
                                           torch.zeros(3, device=dev), 1.0, view, d["projmatrix"], scene.sh_degree,
                                           d["campos"], False, False)
        means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
        out = GaussianRasterizer(rs, depth_quantile=q, ray_depth=True, plane_normals=pn)(
            leaves["means3D"], means2D, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
            rotations=leaves["rotations"])
        loss = (out[2] * out[3]).sum() if only else (out[0].sum() + 0.01 * out[1].sum() + out[2].sum()
                                                     + (out[6].mean() if q else 0.0))
        with Hh.deterministic(det):
            loss.backward()
        grads = [leaves[k].grad for k in leaves] + ([view.grad] if view_grad else []) + ([tanx.grad] if tan_grad
                                                                                          else [])
        return out, grads

    o0, _ = run(False)
    for kw in (dict(), dict(view_grad=True), dict(view_grad=True, tan_grad=True), dict(q=0.5)):
        o1, g1 = run(True, det=True, **kw)
        assert len(o1) == (7 if kw.get("q") else 6)
        for i in (0, 1, 3, 4, 5):
            assert torch.equal(bits(o0[i]), bits(o1[i])), i
        assert not torch.equal(o0[2], o1[2])
        _, g2 = run(True, det=True, **kw)
        for a, b in zip(g1, g2):
            assert a is not None and torch.equal(bits(a), bits(b)) and bool(torch.isfinite(a).all())
    _, g = run(True, view_grad=True, tan_grad=True, det=True, only=True)
    for k in (0, 1, 2, 3, 5, 6):
        assert float(g[k].abs().sum()) > 0, k
    assert int((g[4] != 0).sum()) == 0
    # the plane normal's gradient is not the shortest-axis normal's (which reaches scales through alpha only)
    _, g0 = run(False, det=True, only=True)
    assert not torch.equal(g0[0], g[0]) and not torch.equal(g0[1], g[1])
    # the default (atomic) backward agrees with the deterministic one
    _, gd = run(True, only=True)
    for a, b in zip(g[:4], gd[:4]):
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-12


@pytest.mark.gpu
def test_ortho_rasterizer_composition(cuda_device):
    """OrthoRasterizer with offsets and the deterministic mode: every output but the normal bit-identical to the
    ray_depth=True call, and two deterministic backward runs bit-identical."""
    import test_ray_depth as RD
    from sfgs.ortho import nadir_camera, OrthoRasterizationSettings, OrthoRasterizer
    dev = cuda_device
    theta, sp, ext = math.radians(25.0), 0.5, 8.0
    means, scales, rots, opac = RD._sloped_roof(dev, theta, sp, ext)
    cam = nadir_camera(-ext, ext, -ext, ext, 0.1, 20.0)
    off = Hh.uniform_offsets(cam.image_height, cam.image_width, dev, seed=8)

    def run(pn):
        rs = OrthoRasterizationSettings(cam.image_height, cam.image_width, cam.half_width, cam.half_height, 0.1,
                                        torch.zeros(3, device=dev), 1.0, cam.viewmatrix.to(dev),
                                        cam.projmatrix.to(dev), 0, False, False, subpixel_offset=off)
        leaves = [t.clone().requires_grad_(True) for t in (means, scales, rots)]
        colors = torch.rand((means.shape[0], 3), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
        out = OrthoRasterizer(rs, ray_depth=True, plane_normals=pn)(
            leaves[0], torch.zeros_like(means), opac, colors_precomp=colors, scales=leaves[1], rotations=leaves[2])
        with Hh.deterministic(True):
            (out[0].sum() + 0.1 * out[1].sum() + out[2].sum()).backward()
        return out, [t.grad for t in leaves]
    o0, _ = run(False)
    o1, g1 = run(True)
    _, g2 = run(True)
    for i in (0, 1, 3, 4):
        assert torch.equal(bits(o0[i]), bits(o1[i])), i
    assert not torch.equal(o0[2], o1[2])
    for a, b in zip(g1, g2):
        assert torch.equal(bits(a), bits(b)) and float(a.abs().sum()) > 0


if __name__ == "__main__":
    print(json.dumps(_rejections()))
