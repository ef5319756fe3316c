"""Ray depth: sfgs_rasterize_forward_ray_depth / sfgs_rasterize_backward_ray_depth and the Python surface on top of them
(rasterize_gaussians(ray_depth=True), diff_gauss.GaussianRasterizer(settings, ray_depth=True),
sfgs.ortho.OrthoRasterizer(settings, ray_depth=True), render_height_map(ray_depth=True)).

A record contributes its depth where the pixel's ray meets it, d(p) = z + g . (p - mu), with the slope g = C s (C the
record's conic, s = (w3^T Sigma T0^T, w3^T Sigma T1^T)).  The oracles: a float64 walk of the GPU's lists and records
for the value, a float64 autograd restatement of the compositing for the blend adjoint's sums, tests/ray_depth_chain_f64.py
(ray_depth=True) for the per-Gaussian stage, finite differences, and scenes of known geometry."""
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
        return L.sfgs_rasterize_forward_ray_depth(None if a is None else C.byref(a), off, ortho, q, dq, pos)

    def bwd(b, pos=None, g=None, ncam=0, cam=ptr, det=0, off=None, ortho=0):
        return L.sfgs_rasterize_backward_ray_depth(None if b is None else C.byref(b), off, ortho, det, pos, g, cam,
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
        "bwd ortho phase 1": lambda: bwd(bwd_args(phase=1, acc=ptr), ortho=1),
        "bwd ncam=35 null dL_dcamera": lambda: bwd(bwd_args(), ncam=35, cam=None),
        "bwd ncam=37 null scratch": lambda: bwd(bwd_args(scratch_alloc=N.ALLOC_FN()), ncam=37),
        "bwd det null radii": lambda: bwd(bwd_args(radii=None), det=1),
        "bwd bad sizes": lambda: bwd(bwd_args(height=-1)),
        "bwd null pixel gradient": lambda: bwd(bwd_args(dL_dpix=None)),
    }
    return {name: [call(), N.last_error()] for name, call in cases.items()}


_FWD, _BWD = "forward_ray_depth", "backward_ray_depth"
_BAD_Q = "the quantile must be finite with 0 < q < 1"
_NULL_IN = "null depth_q_pos or dL_dpix_depth_q"
EXPECTED = {
    "fwd null args": (SFGS_E_BADARG, _FWD, "null args"),
    "fwd quantile null pos": (SFGS_E_BADARG, _FWD, "null out_depth_q_pos"),
    "fwd quantile q=0": (SFGS_E_BADARG, _FWD, _BAD_Q),
    "fwd quantile q=nan": (SFGS_E_BADARG, _FWD, _BAD_Q),
    "fwd quantile bad q before ED": (SFGS_E_BADARG, _FWD, _BAD_Q),
    "fwd ED=2": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with ray depth"),
    "fwd ED=2 quantile": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with ray depth"),
    "fwd band": (SFGS_E_UNSUPPORTED, _FWD, "tile-row bands are not supported with ray depth"),
    "fwd out_peers": (SFGS_E_UNSUPPORTED, _FWD, "out_peers are not supported with ray depth"),
    "fwd ED with offsets": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with ray depth"),
    "fwd ortho bad extent": (SFGS_E_BADARG, _FWD, "the half-extents tan_fovx, tan_fovy must be finite and > 0"),
    "fwd bad sizes": (SFGS_E_BADARG, _FWD, "bad sizes"),
    "fwd null output": (SFGS_E_BADARG, _FWD, "null output"),
    "fwd misaligned rotations": (SFGS_E_BADARG, _FWD, "rotations must be 16-byte aligned"),
    "bwd null args": (SFGS_E_BADARG, _BWD, "null args"),
    "bwd pos without cotangent": (SFGS_E_BADARG, _BWD, _NULL_IN),
    "bwd cotangent without pos": (SFGS_E_BADARG, _BWD, _NULL_IN),
    **{f"bwd ncam={n}": (SFGS_E_BADARG, _BWD, "ncam must be 0, 35 or 37") for n in (-1, 1, 36, 38)},
    "bwd ncam before ED": (SFGS_E_BADARG, _BWD, "ncam must be 0, 35 or 37"),
    "bwd ED=2": (SFGS_E_UNSUPPORTED, _BWD, "extra_attrs are not supported with ray depth"),
    "bwd band": (SFGS_E_UNSUPPORTED, _BWD, "tile-row bands are not supported with ray depth"),
    "bwd acc_peers": (SFGS_E_UNSUPPORTED, _BWD, "acc_peers are not supported with ray depth"),
    "bwd phase 2": (SFGS_E_UNSUPPORTED, _BWD, "phase 2 is not supported with ray depth"),
    "bwd ncam=35 phase 1": (SFGS_E_UNSUPPORTED, _BWD,
                            "camera gradients are formed by the one-call backward (phase 0) only"),
    "bwd ncam=37 ortho": (SFGS_E_UNSUPPORTED, _BWD, "the orthographic camera has no camera gradients"),
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
    fwd = lambda **kw: R.rasterize_gaussians(e, m, e, e, e, e, 1.0, e, e, e, kw.pop("F", 0), e, e, 1.0, 1.0, 0.1,  # noqa
                                             8, 8, e, 0, e, False, False, ray_depth=True, **kw)
    for kw, what in ((dict(depth_distortion=True), "depth_distortion"), (dict(graph=True), "graph"),
                     (dict(tile_rows=(0, 1)), "tile_rows"), (dict(out_peers=[0]), "out_peers"),
                     (dict(F=2), "extra_attrs")):
        with pytest.raises(N.SfgsError, match=f"{what}.*not supported with ray depth"):
            fwd(**kw)
    g = torch.zeros((3, 8, 8))
    bwd = lambda **kw: R.rasterize_gaussians_backward(  # noqa: E731
        e, m, e, e, e, e, kw.pop("ex", e), 1.0, e, e, e, e, 1.0, 1.0, 0.1, g, g[:1], g, g[:1], e, e, 0, e, e, 0, e, e,
        e, False, ray_depth=True, **kw)
    for kw, what in ((dict(distortion_state=torch.zeros((2, 8, 8)), dL_dout_distortion=g[:1]), "distortion_state"),
                     (dict(graph=True), "graph"), (dict(tile_rows=(0, 1)), "tile_rows"),
                     (dict(acc_peers=[0], phase=1), "acc_peers"), (dict(ex=torch.zeros((4, 2))), "extra_attrs")):
        with pytest.raises(N.SfgsError, match=f"{what}.*not supported with ray depth"):
            bwd(**kw)
    # the quantile's tensors are checked before their pointers are handed over
    with pytest.raises(ValueError, match="come together"):
        bwd(depth_q_pos=torch.zeros((8, 8), dtype=torch.int32))
    with pytest.raises(ValueError, match="dL_dout_depth_q"):
        bwd(depth_q_pos=torch.zeros((8, 8), dtype=torch.int32), dL_dout_depth_q=g[:1].double())


def test_modules_reject_before_native_calls(monkeypatch):
    """diff_gauss and OrthoRasterizer raise on the distortion together with ray depth, and diff_gauss raises under
    stream capture before any capture-time work (the capacity is not resolved)."""
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
    with pytest.raises(N.SfgsError, match="depth_distortion together with ray_depth"):
        GaussianRasterizer(rs, depth_distortion=True, ray_depth=True)(m, m, torch.ones((4, 1)), **kw)
    ors = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3, False,
                                     False)
    with pytest.raises(N.SfgsError, match="depth_distortion together with ray_depth"):
        OrthoRasterizer(ors, depth_distortion=True, ray_depth=True)(m, m, torch.ones((4, 1)), **kw)

    def no_capacity(*a, **k):
        raise AssertionError("capture-time work before ray depth's check")
    monkeypatch.setattr(diff_gauss._graphs, "resolve_capacity", no_capacity)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    mc = types.SimpleNamespace(is_cuda=True)
    with pytest.raises(N.SfgsError, match="ray depth cannot be captured"):
        diff_gauss._RasterizeGaussians.forward(types.SimpleNamespace(), mc, m, m, m, m, m, m, m, m, torch.empty(0),
                                               rs, False, None, None, None, None, None, None, False, None, False, True)


def test_ortho_rasterizer_is_an_ordinary_module():
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer
    rs = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, False, False)

    class Holder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.r = OrthoRasterizer(rs, ray_depth=True)
            self.w = torch.nn.Parameter(torch.zeros(2))

    for m in (OrthoRasterizer(rs, ray_depth=True), Holder()):
        assert m.to("cpu") is m and m.float() is m and m.cpu() is m and m.double() is m
    assert Holder().double().w.dtype == torch.float64


# ----------------------------------------------------------------------------- the entry each combination reaches
class _Recorder:
    """A stand-in for libsfgs.so: records (entry, arguments after the struct) and returns 1 (one instance)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("sfgs_rasterize_"):
            raise AttributeError(name)

        def call(_args, *rest):
            self.calls.append((name, rest))
            return 1
        return call


def _cuda_free_ptr(monkeypatch):
    """_ptr without a device: the tensors' own addresses (nothing is dereferenced by the recorder)."""
    from sfgs import rasterizer as R

    def ptr(t, keep):
        if t is None or t.numel() == 0:
            return None
        keep.append(t)
        return t.data_ptr()
    monkeypatch.setattr(R, "_ptr", ptr)
    monkeypatch.setattr(R, "check_subpixel_offset", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: __import__("contextlib").nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))


@pytest.mark.parametrize("ortho", [False, True])
@pytest.mark.parametrize("offsets", [False, True])
@pytest.mark.parametrize("quantile", [None, 0.5])
def test_forward_entry_and_arguments(monkeypatch, ortho, offsets, quantile):
    from sfgs import native as N
    from sfgs import rasterizer as R
    rec = _Recorder()
    monkeypatch.setattr(N, "lib", lambda: rec)
    _cuda_free_ptr(monkeypatch)
    H, W, P = 8, 8, 4
    m = torch.zeros((P, 3))
    e = torch.empty(0)
    off = torch.zeros((H, W, 2)) if offsets else None
    out = R.rasterize_gaussians(torch.zeros(3), m, e, torch.ones(P, 1), torch.ones(P, 3), torch.ones(P, 4), 1.0, e, e,
                                e, 0, torch.eye(4), torch.eye(4), 1.0, 1.0, 0.1, H, W, torch.zeros(P, 16, 3), 3,
                                torch.zeros(3), False, False, subpixel_offset=off, ortho=ortho,
                                depth_quantile=quantile, ray_depth=True)
    assert len(rec.calls) == 1
    entry, args = rec.calls[0]
    assert entry == "sfgs_rasterize_forward_ray_depth"
    assert args[0] == (off.data_ptr() if offsets else None) and args[1] == int(ortho)
    if quantile is None:
        assert args[2] == 0.0 and args[3] is None and args[4] is None and len(out) == 10
    else:
        assert args[2] == 0.5 and args[3] == out[10].data_ptr() and args[4] == out[11].data_ptr()
        assert tuple(out[10].shape) == (1, H, W) and out[11].dtype == torch.int32


@pytest.mark.parametrize("ortho,ncam", [(False, 0), (False, 35), (False, 37), (True, 0)])
@pytest.mark.parametrize("offsets", [False, True])
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("quantile", [False, True])
def test_backward_entry_and_arguments(monkeypatch, ortho, ncam, offsets, det, quantile):
    from sfgs import native as N
    from sfgs import rasterizer as R
    rec = _Recorder()
    monkeypatch.setattr(N, "lib", lambda: rec)
    _cuda_free_ptr(monkeypatch)
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
            ray_depth=True, **qkw)
    assert len(rec.calls) == 1
    entry, args = rec.calls[0]
    assert entry == "sfgs_rasterize_backward_ray_depth"
    assert args[0] == (off.data_ptr() if offsets else None) and args[1] == int(ortho) and args[2] == int(det)
    if quantile:
        assert args[3] == qkw["depth_q_pos"].data_ptr() and args[4] == qkw["dL_dout_depth_q"].data_ptr()
    else:
        assert args[3] is None and args[4] is None
    assert args[6] == ncam and (args[5] is None) == (ncam == 0)
    assert len(out) == 10 + (3 if ncam else 0) + (2 if ncam == 37 else 0)


# ----------------------------------------------------------------------------- the restatement on CPU
def _pinhole(W, H, tanx, tany, z0=6.0):
    """A pinhole camera at (0, 0, -z0) looking along +z, as row-vector viewmatrix / projmatrix (the library's
    convention: t = [m, 1] view, hom = [m, 1] proj, ndc = hom.xy / hom.w)."""
    view = torch.eye(4, dtype=torch.float64)
    view[3, 2] = z0
    O = torch.zeros((4, 4), dtype=torch.float64)
    O[0, 0], O[1, 1], O[2, 2], O[2, 3], O[3, 2] = 1.0 / tanx, 1.0 / tany, 1.0, 1.0, -0.01
    return view, view @ O


def _slope_and_projection(m, sc, q, view, proj, W, H, tanx, tany, ks):
    """Independent float64 forward of the quantities the ray-depth chain pairs with acc: ndc, t_z and g = C s."""
    import chain_f64 as CH
    t = m @ view[:3, :3] + view[3, :3]
    hom = m @ proj[:3, :] + proj[3, :]
    ndc = hom[:, :2] / (hom[:, 3:4] + 1e-7)
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    limx, limy = 1.3 * tanx, 1.3 * tany
    tx = (t[:, 0] / t[:, 2]).clamp(-limx, limx) * t[:, 2]
    ty = (t[:, 1] / t[:, 2]).clamp(-limy, limy) * t[:, 2]
    z = t[:, 2]
    J = torch.zeros((m.shape[0], 2, 3), dtype=torch.float64)
    J[:, 0, 0], J[:, 0, 2] = fx / z, -fx * tx / (z * z)
    J[:, 1, 1], J[:, 1, 2] = fy / z, -fy * ty / (z * z)
    T = J @ view[:3, :3].T.expand(m.shape[0], 3, 3)
    Sig = CH.sym6_to_mat(CH.cov3d(sc, CH.quat_to_rot(q)))
    cov2 = T @ Sig @ T.transpose(1, 2) + ks * torch.eye(2, dtype=torch.float64)
    w3 = view[:3, 2]
    s = torch.einsum("i,gij,gkj->gk", w3, Sig, T)
    g = torch.linalg.solve(cov2, s.unsqueeze(-1)).squeeze(-1)
    return ndc, z, g


@pytest.mark.parametrize("ortho,focal,colors", [(False, False, False), (False, True, False), (True, False, False),
                                                (False, True, True)])
def test_chain_without_ray_depth_is_chain_f64(ortho, focal, colors):
    """ray_depth_chain_f64.chain without the keyword returns chain_f64.chain's results bit for bit (every key), so the
    ray-depth restatement differs from the shared one by its ray-depth terms only."""
    import chain_f64 as CH
    import ray_depth_chain_f64 as RC
    torch.manual_seed(5)
    P, W, H, ks = 6, 96, 64, 0.1
    view, proj = _pinhole(W, H, 0.6, 0.4)
    tx, ty = (3.0, 2.0) if ortho else (0.6, 0.4)
    if ortho:
        from sfgs.ortho import projection_matrix
        proj = view @ projection_matrix(tx, ty, 0.01, 100.0).double()
    f = lambda *s: torch.randn(*s, dtype=torch.float64)  # noqa: E731
    m, sc, q = f(P, 3) * 0.5, f(P, 3).abs() * 0.2 + 0.05, f(P, 4)
    acc = f(P, 16)
    vis = torch.tensor([True, True, False, True, True, True])
    clamped = torch.rand(P, 3) < 0.3
    shs = None if colors else f(P, 16, 3) * 0.3
    kw = dict(scales=sc, rotations=q, norm_rec=f(P, 3), ortho=ortho, focal=focal)
    args = (acc, vis, m, torch.rand(P, dtype=torch.float64), clamped, shs, 3, view.float(), proj.float(),
            torch.tensor([0.1, -0.2, -6.0]), W, H, tx, ty, ks)
    a, b = CH.chain(*args, **kw), RC.chain(*args, **kw)
    assert set(a) == set(b)
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
        elif isinstance(a[k], tuple):
            assert all(torch.equal(x, y) for x, y in zip(a[k], b[k])), k
        else:
            assert a[k] == b[k], k


def test_chain_ray_depth_matches_central_differences():
    """ray_depth_chain_f64.chain(ray_depth=True)'s means3D / scales / rotations gradients are those of
        sum A3 t_z + A7 ndc_x + A8 ndc_y + A14 g_x + A15 g_y - A3 (g0_x ndc_x W/2 + g0_y ndc_y H/2)
    (g0: g at the evaluation point; the last term is the depth's moving centre), evaluated independently with the
    exact conic inverse; the colour, normal, conic and opacity words are 0, so no kernel-local derivative but the
    conic inverse's (whose 1e-7 guard is far below the tolerance here) enters."""
    import chain_f64 as CH
    import ray_depth_chain_f64 as RC
    torch.manual_seed(3)
    P, W, H, tanx, tany, ks = 5, 96, 64, 0.6, 0.4, 0.1
    view, proj = _pinhole(W, H, tanx, tany)
    f = lambda *s: torch.randn(*s, dtype=torch.float64)  # noqa: E731
    m = f(P, 3) * 0.5
    sc, q = f(P, 3).abs() * 0.2 + 0.05, f(P, 4)
    acc = f(P, 16)
    acc[:, 0:3] = 0.0
    acc[:, 4:7] = 0.0
    acc[:, 9:14] = 0.0
    vis = torch.ones(P, dtype=torch.bool)
    clamped = torch.zeros(P, 3, dtype=torch.bool)
    r = RC.chain(acc, vis, m, torch.ones(P), clamped, None, 0, view.float(), proj.float(), torch.zeros(3), W, H,
                 tanx, tany, ks, scales=sc, rotations=q, norm_rec=torch.zeros(P, 3), ray_depth=True)
    r0 = CH.chain(acc, vis, m, torch.ones(P), clamped, None, 0, view.float(), proj.float(), torch.zeros(3), W, H,
                  tanx, tany, ks, scales=sc, rotations=q, norm_rec=torch.zeros(P, 3))
    assert not torch.equal(r["scales"], r0["scales"])
    vw, pj = view.float().double(), proj.float().double()
    _, _, g0 = _slope_and_projection(m, sc, q, vw, pj, W, H, tanx, tany, float(torch.tensor(ks, dtype=torch.float32)))

    def L(m_, sc_, q_):
        ndc, z, g = _slope_and_projection(m_, sc_, q_, vw, pj, W, H, tanx, tany,
                                          float(torch.tensor(ks, dtype=torch.float32)))
        return float((acc[:, 3] * z + acc[:, 7] * ndc[:, 0] + acc[:, 8] * ndc[:, 1] + acc[:, 14] * g[:, 0]
                      + acc[:, 15] * g[:, 1] - acc[:, 3] * (g0[:, 0] * ndc[:, 0] * 0.5 * W
                                                            + g0[:, 1] * ndc[:, 1] * 0.5 * H)).sum())

    h = 1e-6
    for name, idx in (("means3D", 0), ("scales", 1), ("rot", 2)):
        args = [m, sc, q]
        v = args[idx]
        fd = torch.zeros_like(v)
        for i in range(v.numel()):
            e = torch.zeros(v.numel(), dtype=v.dtype)
            e[i] = h
            e = e.view_as(v)
            up, dn = list(args), list(args)
            up[idx], dn[idx] = v + e, v - e
            fd.view(-1)[i] = (L(*up) - L(*dn)) / (2 * h)
        gv = r[name]
        assert torch.allclose(gv, fd, rtol=1e-5, atol=1e-6 * float(fd.abs().max())), (name, (gv - fd).abs().max())


# ----------------------------------------------------------------------------- GPU helpers
def _headline(dev):
    _, cam, D, d, _ = Hh.frame("jax004", dev)
    return cam, D, d, torch.tensor([0.0, 0.0, 0.0], device=dev)


def _ortho_headline(cam, d):
    from sfgs.ortho import projection_matrix
    oc = types.SimpleNamespace(width=cam.width, height=cam.height, tanfovx=60.0, tanfovy=60.0 * 1080 / 1920)
    proj = d["viewmatrix"].cpu().double() @ projection_matrix(oc.tanfovx, oc.tanfovy, 0.01, 1e4).double()
    return oc, dict(d, projmatrix=proj.float().to(d["means3D"].device))


def _form(form, cam, d, dev):
    kw = {}
    if form == "jitter":
        kw["subpixel_offset"] = Hh.uniform_offsets(cam.height, cam.width, dev, seed=3)
    if form == "ortho":
        cam, d = _ortho_headline(cam, d)
        kw["ortho"] = True
    return cam, d, kw


def _small_case(dev, seed=5, P=3000):
    from sfgs import synthetic as S
    scene = S.blob_scene(P, seed=seed)
    cam = S.simple_camera(160, 120)
    return scene, cam, Hh.to_torch(scene, cam, dev)


def _tile_pixels(tile, W, H, dev, off=None):
    tiles_x = (W + 15) // 16
    ty, tx = divmod(int(tile), tiles_x)
    yy, xx = torch.meshgrid(torch.arange(16, device=dev) + 16 * ty, torch.arange(16, device=dev) + 16 * tx,
                            indexing="ij")
    inside = (xx < W) & (yy < H)
    xx, yy = xx[inside], yy[inside]
    px, py = xx.double(), yy.double()
    if off is not None:       # the kernels' float32 sample position
        px, py = (xx.float() + off[yy, xx, 0]).double(), (yy.float() + off[yy, xx, 1]).double()
    return yy * W + xx, px, py


def _applied(I, tile, pid, px, py):
    """The forward's applied set [pixels, records] (float32 skip tests, cut at n_contrib) and the pixels with a record
    within rounding of a skip threshold."""
    r0, r1 = (int(v) for v in I["ranges"][tile])
    g = I["rec"][I["point_list"][r0:r1].long()]
    dx, dy = g[None, :, 0] - px.float()[:, None], g[None, :, 1] - py.float()[:, None]
    power = -0.5 * (g[None, :, 2] * dx * dx + g[None, :, 4] * dy * dy) - g[None, :, 3] * dx * dy
    araw = g[None, :, 5] * torch.exp(power)
    ok = ~(power > 0) & ~(torch.clamp(araw, max=0.99) < 1.0 / 255.0)
    pos = torch.arange(1, r1 - r0 + 1, device=g.device)
    within = pos[None, :] <= I["n_contrib"][pid].long()[:, None]
    near = ((araw * 255.0 - 1.0).abs() < 1e-5) | (power.abs() < 1e-6)
    return ok & within, (near & within).any(1), r0, r1, power


def _composite(rec, pl, M, px, py, dtype):
    g = rec[pl]
    dx, dy = g[None, :, 0] - px.to(dtype)[:, None], g[None, :, 1] - py.to(dtype)[:, None]
    power = -0.5 * (g[None, :, 2] * dx * dx + g[None, :, 4] * dy * dy) - g[None, :, 3] * dx * dy
    G = torch.exp(power)
    araw = g[None, :, 5] * G
    alpha = araw - (araw - 0.99).clamp(min=0).detach()
    am = torch.where(M, alpha, torch.zeros_like(alpha))
    T_after = torch.cumprod(1 - am, 1)
    T_before = torch.cat([torch.ones_like(T_after[:, :1]), T_after[:, :-1]], 1)
    return am * T_before, T_after[:, -1], g, dx, dy, G, araw


def _run(d, cam, D, bg, ray_depth=True, **kw):
    from sfgs import rasterizer as R
    e = torch.empty(0, device=d["means3D"].device)
    out = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cam.height,
                                cam.width, d["shs"], D, d["campos"], False, False, ray_depth=ray_depth, **kw)
    return dict(zip(Hh.FWD_KEYS, out[:10])), out[10:]


# ----------------------------------------------------------------------------- GPU: no interference
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pinhole", "jitter", "ortho"])
def test_no_interference_forward(cuda_device, form):
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    cam, d, kw = _form(form, cam, d, dev)
    a, _ = _run(d, cam, D, bg, ray_depth=False, **kw)
    b, _ = _run(d, cam, D, bg, **kw)
    for k in ("color", "norm", "alpha", "radii"):
        assert torch.equal(bits(a[k]), bits(b[k])), k
    assert a["num_rendered"] == b["num_rendered"] > 0
    P = d["means3D"].shape[0]
    Ia, Ib = Hh.our_internals(a, P, cam.height, cam.width), Hh.our_internals(b, P, cam.height, cam.width)
    for k in ("n_contrib", "point_list", "ranges", "keys"):
        assert torch.equal(Ia[k], Ib[k]), k
    vis = a["radii"] > 0
    assert torch.equal(bits(Ia["rec"][vis, :14]), bits(Ib["rec"][vis, :14]))
    assert int((Ia["rec"][vis, 14:16] != 0).sum()) == 0 and int((Ib["rec"][vis, 14:16] != 0).sum()) > 0
    assert not torch.equal(a["depth"], b["depth"]) and bool(torch.isfinite(b["depth"]).all())


@pytest.mark.gpu
@pytest.mark.parametrize("form,ncam", [("pinhole", 0), ("pinhole", 35), ("pinhole", 37), ("jitter", 37),
                                       ("ortho", 0)])
def test_no_interference_deterministic_backward(cuda_device, form, ncam):
    """With a zero depth cotangent the ten deterministic gradients of the ray-depth backward (on the ray-depth forward's
    buffers) are those of the default backward (on the default forward's).  The camera and focal terms are summed from
    products the RAYD instantiation of the per-Gaussian adjoint contracts into FMAs differently, so they are held to
    4 eps of the sum of their terms' magnitudes instead of bit equality."""
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    cam, d, kw = _form(form, cam, d, dev)
    fa, _ = _run(d, cam, D, bg, ray_depth=False, **kw)
    fb, _ = _run(d, cam, D, bg, **kw)
    g = torch.Generator(device=dev).manual_seed(1)
    H, W = cam.height, cam.width
    cot = (torch.randn((3, H, W), generator=g, device=dev), torch.zeros((1, H, W), device=dev),
           torch.randn((3, H, W), generator=g, device=dev), torch.randn((1, H, W), generator=g, device=dev))
    kw.update(camera_grad=ncam > 0, intrinsics_grad=ncam == 37)
    a = Hh.run_ours_backward(d, cam, D, bg, fa, cot, det=True, **kw)
    b = Hh.run_ours_backward(d, cam, D, bg, fb, cot, det=True, ray_depth=True, **kw)
    assert set(a) == set(b)
    cam_keys = ("view", "proj", "campos", "tanx", "tany")
    for k in a:      # equal as values: the sign of a zero may differ
        if k not in cam_keys:
            assert torch.equal(a[k], b[k]), k
    if ncam:
        import chain_f64 as CH
        ri = Hh.restatement_inputs(fa, d, cam, D, bg, cot, off=kw.get("subpixel_offset"))
        ri.update(cov3D=None, scales=d["scales"], rotations=d["rotations"])
        mag = CH.chain(**ri, focal=True, dtype=torch.float64)["abs"]
        flat = lambda r: torch.cat([r[k].reshape(-1) for k in cam_keys if k in r]).double()  # noqa: E731
        ratio = float(((flat(a) - flat(b)).abs() / (4 * EPS32 * mag[:flat(a).numel()].double() + 1e-30)).max())
        print(f"\n[ray depth no interference {form} ncam={ncam}] camera terms: worst difference / (4 eps sum |terms|) "
              f"{ratio:.3f}")
        assert ratio <= 1.0


# ----------------------------------------------------------------------------- GPU: forward value
def _sigma_and_view(d, I, idx, cam, ortho=False):
    """float64 Sigma [n,3,3], T [n,2,3] and w3 of records idx from the GPU's cov3D and the view (the kernels' J)."""
    import chain_f64 as CH
    V = d["viewmatrix"].double().reshape(4, 4)
    m = d["means3D"][idx].double()
    t = m @ V[:3, :3] + V[3, :3]
    W_, H_ = cam.width, cam.height
    fx = float(torch.tensor(W_, dtype=torch.float32) / (2 * torch.tensor(cam.tanfovx, dtype=torch.float32)))
    fy = float(torch.tensor(H_, dtype=torch.float32) / (2 * torch.tensor(cam.tanfovy, dtype=torch.float32)))
    n = idx.numel()
    J = torch.zeros((n, 2, 3), dtype=torch.float64, device=m.device)
    if ortho:
        J[:, 0, 0], J[:, 1, 1] = fx, fy
    else:
        limx, limy = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
        z = t[:, 2]
        tx = (t[:, 0] / z).clamp(-limx, limx) * z
        ty = (t[:, 1] / z).clamp(-limy, limy) * z
        J[:, 0, 0], J[:, 0, 2] = fx / z, -fx * tx / (z * z)
        J[:, 1, 1], J[:, 1, 2] = fy / z, -fy * ty / (z * z)
    T = J @ V[:3, :3].T
    Sig = CH.sym6_to_mat(I["cov3D"][idx].double())
    return Sig, T, V[:3, 2]


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pinhole", "jitter", "ortho"])
def test_forward_value(cuda_device, form):
    """On 96 random tiles of the headline frame:
      - the slope words against float64 C s from cov3D and the view, C the record's float conic: |err| <= 64 eps
        |C| (|w3| |Sigma| |T|) (s and g are a few dozen float operations on those products, which cancel in s);
      - out_depth against the float64 sum of w d(p) over the forward's applied set: |err| <= (8 n + 16) eps
        sum |w d| per pixel (n applied records: the walk's T and the sum each lose <= ~2 eps per record);
      - every applied pair within the Cauchy-Schwarz bound |d(p) - z| <= sigma_z sqrt(-2 power) (+ rounding)."""
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    cam, d, kw = _form(form, cam, d, dev)
    off = kw.get("subpixel_offset")
    W, H = cam.width, cam.height
    f, _ = _run(d, cam, D, bg, **kw)
    P = d["means3D"].shape[0]
    I = Hh.our_internals(f, P, H, W)
    vis = torch.nonzero(f["radii"] > 0).flatten()
    Sig, T, w3 = _sigma_and_view(d, I, vis, cam, ortho=form == "ortho")
    s = torch.einsum("i,gij,gkj->gk", w3, Sig, T)
    Cm = I["rec"][vis][:, [2, 3, 3, 4]].double().reshape(-1, 2, 2)
    g64 = (Cm @ s.unsqueeze(-1)).squeeze(-1)
    gpu = I["rec"][vis, 14:16].double()
    # s = w3^T Sigma T^T cancels (the depth row is nearly orthogonal to the pixel rows): its rounding scale is that of
    # the products it sums
    s_mag = torch.einsum("i,gij,gkj->gk", w3.abs(), Sig.abs(), T.abs())
    lim = 64 * EPS32 * (Cm.abs() @ s_mag.unsqueeze(-1)).squeeze(-1) + 1e-30
    ratio_g = float(((gpu - g64).abs() / lim).max())
    sz = torch.sqrt(torch.einsum("i,gij,j->g", w3, Sig, w3))
    sigz = torch.zeros(P, dtype=torch.float64, device=dev)
    sigz[vis] = sz
    rec = I["rec"].double()
    tiles = torch.randperm(I["ranges"].shape[0], generator=torch.Generator().manual_seed(7))[:96].tolist()
    worst_d, worst_b, npix = 0.0, 0.0, 0
    for tile in tiles:
        pid, px, py = _tile_pixels(tile, W, H, dev, off)
        M, near, r0, r1, power = _applied(I, tile, pid, px, py)
        if r1 == r0:
            continue
        pl = I["point_list"][r0:r1].long()
        w, _, g, dx, dy, _, _ = _composite(rec, pl, M, px, py, torch.float64)
        dep = g[None, :, 6] - g[None, :, 14] * dx - g[None, :, 15] * dy
        ref = (w * dep).sum(1)
        n = M.sum(1).double()
        lim = (8 * n + 16) * EPS32 * (w * dep).abs().sum(1) + 1e-30
        ok = ~near
        if ok.any():
            worst_d = max(worst_d, float(((f["depth"].reshape(-1)[pid].double() - ref).abs() / lim)[ok].max()))
        # the bound, for the applied pairs (the float32 power of the kernel)
        b = sigz[pl][None, :] * torch.sqrt((-2.0 * power.double()).clamp_min(0))
        excess = ((dep - g[None, :, 6]).abs() - b) / (1e-5 * g[None, :, 6].abs() + 1e-30)
        worst_b = max(worst_b, float(torch.where(M, excess, torch.full_like(excess, -1e30)).max()))
        npix += int(ok.sum())
    print(f"\n[ray depth forward {form}] slope words worst err / bound {ratio_g:.3f}; out_depth worst err / bound "
          f"{worst_d:.3f} over {npix} pixels; Cauchy-Schwarz excess / 1e-5 depth {worst_b:.3f}")
    assert ratio_g <= 1.0 and worst_d <= 1.0 and worst_b <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pinhole", "jitter"])
def test_quantile_value(cuda_device, form):
    """With the depth quantile: the selection (depth_q_pos) is bit-identical to the call without ray depth, and
    depth_q is the selected record's d(p) evaluated as the kernel evaluates it (float32 FMAs)."""
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    cam, d, kw = _form(form, cam, d, dev)
    W, H = cam.width, cam.height
    fa, (dqa, posa) = _run(d, cam, D, bg, ray_depth=False, depth_quantile=0.5, **kw)
    fb, (dqb, posb) = _run(d, cam, D, bg, depth_quantile=0.5, **kw)
    assert torch.equal(posa, posb) and int((posb > 0).sum()) > 0
    I = Hh.our_internals(fb, d["means3D"].shape[0], H, W)
    ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    px, py = xs.float(), ys.float()
    if "subpixel_offset" in kw:
        px, py = px + kw["subpixel_offset"][..., 0], py + kw["subpixel_offset"][..., 1]
    tiles_x = (W + 15) // 16
    tile = (ys // 16) * tiles_x + xs // 16
    sel = posb > 0
    inst = I["ranges"][tile[sel], 0].long() + posb[sel].long() - 1
    r = I["rec"][I["point_list"][inst].long()]
    # fmaf(-g14, mx - p.x, fmaf(-g15, my - p.y, z)), in float64 with float32 operands: differs from the kernel's
    # fused float32 result by at most one rounding of the result
    dx, dy = (r[:, 0] - px[sel]).double(), (r[:, 1] - py[sel]).double()
    ref = r[:, 6].double() - r[:, 14].double() * dx - r[:, 15].double() * dy
    err = (dqb[0][sel].double() - ref).abs() / (EPS32 * (r[:, 6].double().abs() + (r[:, 14].double() * dx).abs()
                                                          + (r[:, 15].double() * dy).abs()))
    print(f"\n[ray depth quantile {form}] worst err / (eps x magnitude) {float(err.max()):.3f}")
    assert float(err.max()) <= 2.0
    assert int((dqb[0][~sel] != 0).sum()) == 0


# ----------------------------------------------------------------------------- GPU: phase-1 sums
def blend_restatement(I, W, H, bg, cot, dtype, off=None, dq=None):
    """The phase-1 sums [P,16] in `dtype` with autograd over the GPU's lists and records, the depth attribute being
    d(p) = z + g . (p - mu) with mu held (dL/dmu of d is the per-Gaussian stage's); word 14-15: dL/dg.  dq: (depth_q_pos
    [H,W], cotangent [1,H,W]) of a quantile.  Also the sums of |w c (p - mu)| and |w c| (the rounding scales)."""
    dev = I["rec"].device
    rec = I["rec"].to(dtype).detach().clone().requires_grad_(True)
    bgd = bg.to(dtype)
    loss = torch.zeros((), dtype=dtype, device=dev)
    mag = torch.zeros((rec.shape[0], 3), dtype=torch.float64, device=dev)
    nmax = int(I["n_contrib"].max())
    for tile in range(I["ranges"].shape[0]):
        pid, px, py = _tile_pixels(tile, W, H, dev, off)
        M, _, r0, r1, _ = _applied(I, tile, pid, px, py)
        if r1 == r0:
            continue
        pl = I["point_list"][r0:r1].long()
        w, T, g, dx, dy, _, _ = _composite(rec, pl, M, px, py, dtype)
        dep = g[None, :, 6] - g[None, :, 14] * dx.detach() - g[None, :, 15] * dy.detach()
        col = w @ g[:, 8:11] + T[:, None] * bgd[None, :]
        dsum, nor, alp = (w * dep).sum(1), w @ g[:, 11:14], 1 - T
        ct = lambda t: t.reshape(t.shape[0], -1)[:, pid].to(dtype)  # noqa: E731
        c = ct(cot[1])[0]
        loss = loss + (ct(cot[0]).T * col).sum() + (c * dsum).sum() + (ct(cot[2]).T * nor).sum() + \
            (ct(cot[3])[0] * alp).sum()
        with torch.no_grad():
            wc = (w * c[:, None]).double().abs()
            mag[:, 0].index_add_(0, pl, wc.sum(0))
            mag[:, 1].index_add_(0, pl, (wc * dx.double().abs()).sum(0))
            mag[:, 2].index_add_(0, pl, (wc * dy.double().abs()).sum(0))
        if dq is not None:
            pos, cq = dq[0].reshape(-1)[pid].long(), dq[1].reshape(-1)[pid].to(dtype)
            has = pos > 0
            j = pos[has] - 1
            loss = loss + (cq[has] * dep[has, j]).sum()
            with torch.no_grad():
                mag[:, 0].index_add_(0, pl[j], cq[has].double().abs())
                mag[:, 1].index_add_(0, pl[j], (cq[has].abs() * dx[has, j].abs()).double())
                mag[:, 2].index_add_(0, pl[j], (cq[has].abs() * dy[has, j].abs()).double())
    loss.backward()
    gr = rec.grad
    out = torch.zeros((rec.shape[0], 16), dtype=dtype, device=dev)
    out[:, 3], out[:, 14], out[:, 15] = gr[:, 6], gr[:, 14], gr[:, 15]
    return out, mag, nmax


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("quantile", [False, True])
def test_blend_adjoint_sums(cuda_device, det, quantile):
    """Words 3 (sum w c) and 14-15 (sum w c (p - mu)) of the phase-1 sums against the float64 restatement.  Bound per
    word: (2 n_max + 64) eps times the sum of the terms' magnitudes, +1e-7 of the word's largest value: the adjoint
    recovers each T back to front through up to n_max records (<= 2 eps each) and sums <= 32 pixels' terms per block
    in float32 before the blocks' sums are added.  Every other word equals the same backward's without ray depth
    where the depth cotangent is 0.  Pixels with a record at a float32 skip threshold get zero cotangents."""
    dev = cuda_device
    scene, cam, d = _small_case(dev)
    W, H, D = cam.width, cam.height, scene.sh_degree
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    qkw = dict(depth_quantile=0.5) if quantile else {}
    f, side = _run(d, cam, D, bg, **qkw)
    I = Hh.our_internals(f, d["means3D"].shape[0], H, W)
    keep = torch.ones(H * W, device=dev)
    for tile in range(I["ranges"].shape[0]):
        pid, px, py = _tile_pixels(tile, W, H, dev)
        _, near, *_ = _applied(I, tile, pid, px, py)
        keep[pid[near]] = 0
    keep = keep.reshape(1, H, W)
    gen = torch.Generator(device=dev).manual_seed(4)
    cot = tuple(torch.randn(s, generator=gen, device=dev) * keep for s in ((3, H, W), (1, H, W), (3, H, W), (1, H, W)))
    dq = (side[1], torch.randn((1, H, W), generator=gen, device=dev) * keep) if quantile else None
    bkw = dict(depth_q_pos=dq[0], dL_dout_depth_q=dq[1]) if quantile else {}
    acc = lambda: Hh.run_ours_backward(d, cam, D, bg, f, cot, det=det, phase=1, ray_depth=True, **bkw)  # noqa: E731
    a = acc()
    r64, mag, nmax = blend_restatement(I, W, H, bg, cot, torch.float64, dq=dq)
    vis = f["radii"] > 0
    worst = []
    for k, mi in ((3, 0), (14, 1), (15, 2)):
        ref = r64[vis, k]
        lim = (2 * nmax + 64) * EPS32 * mag[vis, mi] + 1e-7 * float(ref.abs().max()) + 1e-30
        worst.append(float(((a[vis, k].double() - ref).abs() / lim).max()))
    # the words ray depth does not touch, against the default backward with the depth cotangent set to 0
    cz = (cot[0], torch.zeros_like(cot[1]), cot[2], cot[3])
    az = Hh.run_ours_backward(d, cam, D, bg, f, cz, det=True, phase=1, ray_depth=True)
    fa, _ = _run(d, cam, D, bg, ray_depth=False)
    a0 = Hh.run_ours_backward(d, cam, D, bg, fa, cz, det=True, phase=1)
    print(f"\n[ray depth blend adjoint det={det} quantile={quantile}] n_max {nmax}; worst err / bound on words 3, 14, "
          f"15: " + ", ".join(f"{v:.3f}" for v in worst))
    assert all(v <= 1.0 for v in worst), worst
    assert torch.equal(az[:, :14], a0[:, :14])
    assert int((a[~vis] != 0).sum()) == 0
    if det:
        assert torch.equal(bits(a), bits(acc()))


# ----------------------------------------------------------------------------- GPU: gradients against the restatement
def _chain_case(dev):
    def make():
        import ray_depth_chain_f64 as RC
        from sfgs import synthetic as S
        cam, D, d, _ = _headline(dev)
        bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
        f, side = _run(d, cam, D, bg, depth_quantile=0.5)
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=6)]
        cq = torch.randn((1, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(8), device=dev)
        bkw = dict(depth_q_pos=side[1], dL_dout_depth_q=cq, ray_depth=True)
        a = Hh.restatement_inputs(f, d, cam, D, bg, cot)
        a["acc"] = Hh.run_ours_backward(d, cam, D, bg, f, cot, det=True, phase=1, **bkw)
        a.update(cov3D=None, scales=d["scales"], rotations=d["rotations"])
        r64 = RC.chain(**a, focal=True, dtype=torch.float64, ray_depth=True)
        r32 = RC.chain(**a, focal=True, dtype=torch.float32, ray_depth=True)
        return cam, D, d, bg, f, cot, bkw, r64, r32
    return Hh.cached("chain", "jax004-ray-depth", make)


def _camera_flat(r, ncam):
    v = [r["view"].reshape(16), r["proj"].reshape(16), r["campos"].reshape(3)]
    if ncam == 37:
        v += [r["tanx"].reshape(1), r["tany"].reshape(1)]
    return torch.cat(v).double()


@pytest.mark.gpu
@pytest.mark.parametrize("ncam", [0, 35, 37])
def test_gradients_against_restatement(cuda_device, ncam):
    """The ten gradients and the camera / focal terms of the deterministic backward with every cotangent plus
    depth_q's, against ray_depth_chain_f64.chain(ray_depth=True) on the same sums, with the bounds of test_depth_quantile.py, except
    that the gradients' bar is four (not two) times the float32 restatement's error: the slope's s = w3^T Sigma T^T
    cancels, and the kernel (from X = T Sigma) and the restatement (an einsum) round its products in different orders,
    so their errors are independent draws of the same size rather than one a small multiple of the other."""
    cam, D, d, bg, f, cot, bkw, r64, r32 = _chain_case(cuda_device)
    g = Hh.run_ours_backward(d, cam, D, bg, f, cot, det=True, camera_grad=ncam > 0, intrinsics_grad=ncam == 37, **bkw)
    worst = {}
    for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot"):
        ref, ref32 = r64[k].double(), r32[k].double()
        ours = g[k].detach().double().reshape(ref.shape)
        lim = 4.0 * float((ref32 - ref).abs().max()) + 1e-6 * float(ref.abs().max())
        worst[k] = float((ours - ref).abs().max()) / lim
    print(f"\n[ray depth chain ncam={ncam}] worst err / bound per gradient: "
          + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), (ncam, worst)
    if ncam:
        gpu = torch.cat([g["view"].reshape(16), g["proj"].reshape(16), g["campos"].reshape(3)]
                        + ([g["tanx"].reshape(1), g["tany"].reshape(1)] if ncam == 37 else [])).double()
        f64, f32 = _camera_flat(r64, ncam), _camera_flat(r32, ncam)
        tol = torch.maximum(2.0 * (f32 - f64).abs(), 1e-6 * r64["abs"][:ncam].double())
        err = (gpu - f64).abs()
        print(f"[ray depth chain ncam={ncam}] camera max err / tol {float((err / tol.clamp_min(1e-300)).max()):.3f}")
        assert (err <= tol).all(), (ncam, err, tol)


# ----------------------------------------------------------------------------- GPU: finite differences
@pytest.mark.gpu
def test_finite_differences(cuda_device):
    """d/d means3D, d/d scales and d/d rotations of sum c out_depth (ray depth) on a small scene against central
    differences, over the pixels whose applied set is the same at -eps, 0 and +eps."""
    from sfgs import rasterizer as R
    dev = cuda_device
    scene, cam, d = _small_case(dev, seed=6)
    bg = torch.zeros(3, device=dev)
    W, H, D = cam.width, cam.height, scene.sh_degree
    e = torch.empty(0, device=dev)

    def fwd(m, s, q):
        return R.rasterize_gaussians(bg, m, e, d["opacities"], s, q, 1.0, e, e, e, 0, d["viewmatrix"],
                                     d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"], D, d["campos"],
                                     False, False, ray_depth=True)
    base = fwd(d["means3D"], d["scales"], d["rotations"])
    f0 = dict(zip(Hh.FWD_KEYS, base[:10]))
    P = d["means3D"].shape[0]
    tag = torch.rand(P, generator=torch.Generator(device=dev).manual_seed(1), device=dev, dtype=torch.float64)

    def applied_sets(out):
        I = Hh.our_internals(dict(zip(Hh.FWD_KEYS, out[:10])), P, H, W)
        h = torch.zeros(H * W, dtype=torch.float64, device=dev)
        for tile in range(I["ranges"].shape[0]):
            pid, px, py = _tile_pixels(tile, W, H, dev)
            M, near, r0, r1, _ = _applied(I, tile, pid, px, py)
            if r1 > r0:
                h[pid] = (M.double() * tag[I["point_list"][r0:r1].long()][None, :]).sum(1)
                h[pid[near]] = -1.0
        return h
    set0 = applied_sets(base)
    c = torch.randn((1, H, W), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    z = torch.zeros_like
    cot = (z(f0["color"]), c, z(f0["norm"]), z(f0["alpha"]))
    g_all = Hh.run_ours_backward(d, cam, D, bg, f0, cot, det=True, ray_depth=True)
    picks = torch.argsort(g_all["rot"].abs().sum(1), descending=True)[:5].tolist()
    worst = 0.0
    for i in picks:
        for what, k, eps in ([("means3D", k, 1e-3) for k in range(3)] + [("scales", k, 1e-4) for k in range(3)]
                             + [("rot", k, 1e-3) for k in range(4)]):
            outs = []
            for s in (1.0, -1.0):
                v = {"means3D": d["means3D"].clone(), "scales": d["scales"].clone(), "rot": d["rotations"].clone()}
                v[what][i, k] += s * eps
                outs.append(fwd(v["means3D"], v["scales"], v["rot"]))
            stable = set0 >= 0
            for out in outs:
                stable &= applied_sets(out) == set0
            cm = c * stable.reshape(1, H, W)
            fdv = float(((outs[0][2].double() - outs[1][2].double()) * cm).sum()) / (2 * eps)
            g = Hh.run_ours_backward(d, cam, D, bg, f0, (cot[0], cm, cot[2], cot[3]), det=True, ray_depth=True)
            an = float(g[what][i, k])
            err = abs(an - fdv) / max(abs(fdv), abs(an), 1e-3)
            worst = max(worst, err)
            assert err <= 3e-2, (what, i, k, an, fdv)
    print(f"\n[ray depth FD] {len(picks)} Gaussians x (3 means + 3 scales + 4 rotations): worst relative error "
          f"{worst:.2e}")


# ----------------------------------------------------------------------------- GPU: geometry
def _sloped_roof(dev, theta, spacing, extent, thick=1e-3):
    """Flat surfels tiling the plane z = x tan(theta) over [-extent, extent]^2, each rotated into the plane."""
    xs = torch.arange(-extent + spacing / 2, extent, spacing)
    X, Y = torch.meshgrid(xs, xs, indexing="ij")
    X, Y = X.flatten(), Y.flatten()
    P = X.numel()
    u = spacing / math.cos(theta)       # along the slope the surfels are spaced by spacing / cos
    means = torch.stack([X, Y, X * math.tan(theta)], 1).to(dev)
    scales = torch.tensor([0.7 * u, 0.7 * spacing, thick]).expand(P, 3).contiguous().to(dev)
    phi = -theta                        # rotation about +y by -theta takes +x to (cos theta, 0, sin theta)
    rots = torch.tensor([math.cos(phi / 2), 0.0, math.sin(phi / 2), 0.0]).expand(P, 4).contiguous().to(dev)
    opac = torch.full((P, 1), 0.99, device=dev)
    return means, scales, rots, opac


@pytest.mark.gpu
@pytest.mark.parametrize("quantile", [None, 0.5])
def test_dsm_of_a_sloped_roof(cuda_device, quantile):
    """A nadir orthographic DSM of a roof of thin surfels at 30 degrees.  The ray-depth map's interior error is within
    the bound from the Mip shrinkage and the thickness: for a surfel of 2D variance Sigma_xx (pixels^2) the kernel's
    slope is (Sigma2D + k I)^-1 s, the plane's s_x / Sigma_xx without thickness; an applied pair lies within
    sqrt(2 ln(255 o) (Sigma_xx + k)) pixels of the centre, so a pair's depth is off the plane by at most |g - g_plane|
    times that, and a pixel's (alpha-normalised or selected) depth, a convex combination, by no more; plus float32
    rounding of depths ~ z_top.  The centre-depth map's error on the same scene exceeds that bound."""
    from sfgs.ortho import nadir_camera, render_height_map
    dev = cuda_device
    theta, sp, ext, ks = math.radians(30.0), 0.5, 12.0, 0.1
    means, scales, rots, opac = _sloped_roof(dev, theta, sp, ext)
    res = 0.1
    cam = nadir_camera(-ext, ext, -ext, ext, res, 30.0)
    # the bound, float64, from one surfel (all are alike)
    import chain_f64 as CH
    Sig = CH.sym6_to_mat(CH.cov3d(scales[:1].double().cpu(), CH.quat_to_rot(rots[:1].double().cpu())))[0]
    V = cam.viewmatrix.double()
    h = cam.image_width / (2 * cam.half_width)
    T = h * V[:3, :2].T                 # J W with the constant J = diag(h, h) (square pixels)
    w3 = V[:3, 2]
    s = T @ Sig @ w3
    S2 = T @ Sig @ T.T
    gk = torch.linalg.solve(S2 + ks * torch.eye(2, dtype=torch.float64), s)
    # depth = z_top - z, z = x tan(theta), pixel x = (x - xmin) h: d depth / d pixel_x = -tan(theta) / h
    g_plane = torch.tensor([-math.tan(theta) / h, 0.0], dtype=torch.float64)
    reach = torch.sqrt(2.0 * math.log(255.0 * 0.99) * (torch.diagonal(S2) + ks))
    bound = float(((gk - g_plane).abs() * reach).sum()) + 64 * EPS32 * 30.0
    colors = torch.zeros((means.shape[0], 3), device=dev)
    kw = dict(colors_precomp=colors, kernel_size=ks, surface_quantile=quantile)
    ray = render_height_map(cam, means, opac, scales, rots, ray_depth=True, **kw)
    ctr = render_height_map(cam, means, opac, scales, rots, **kw)
    xs = cam.xmin + (torch.arange(cam.image_width, device=dev) + 0.5) * res
    ys = cam.ymax - (torch.arange(cam.image_height, device=dev) + 0.5) * res
    Y, X = torch.meshgrid(ys, xs, indexing="ij")
    truth = X * math.tan(theta)
    interior = (X.abs() < ext - 3.0) & (Y.abs() < ext - 3.0)
    e_ray = (ray - truth).abs()[interior]
    e_ctr = (ctr - truth).abs()[interior]
    assert bool(torch.isfinite(e_ray).all()) and bool(torch.isfinite(e_ctr).all())
    print(f"\n[ray depth DSM q={quantile}] bound {bound:.2e}; ray-depth worst {float(e_ray.max()):.2e} (mean "
          f"{float(e_ray.mean()):.2e}); centre-depth worst {float(e_ctr.max()):.2e} (mean {float(e_ctr.mean()):.2e}); "
          f"worst / bound {float(e_ray.max()) / bound:.3f}")
    assert float(e_ray.max()) <= bound
    assert float(e_ctr.max()) > bound


@pytest.mark.gpu
def test_oblique_ground(cuda_device):
    """An oblique pinhole view of a flat ground of surfels: the depth (alpha-normalised) against the analytic
    ray-plane depth, for both modes.  The ray-depth mean error is the smaller one."""
    from sfgs import synthetic as S
    dev = cuda_device
    sp, ext = 0.3, 25.0
    xs = torch.arange(-ext + sp / 2, ext, sp)
    X, Y = torch.meshgrid(xs, xs, indexing="ij")
    P = X.numel()
    means = torch.stack([X.flatten(), Y.flatten(), torch.zeros(P)], 1).to(dev).contiguous()
    scales = torch.tensor([0.7 * sp, 0.7 * sp, 1e-3]).expand(P, 3).contiguous().to(dev)
    rots = torch.tensor([1.0, 0.0, 0.0, 0.0]).expand(P, 4).contiguous().to(dev)
    opac = torch.full((P, 1), 0.99, device=dev)
    cam = S.orbit_camera(elevation_deg=40.0, radius=18.0, fov_deg=50.0, width=320, height=240)
    d = dict(means3D=means, scales=scales, rotations=rots, opacities=opac,
             shs=torch.zeros((P, 1, 3), device=dev), viewmatrix=torch.from_numpy(cam.viewmatrix).to(dev),
             projmatrix=torch.from_numpy(cam.projmatrix).to(dev), campos=torch.from_numpy(cam.campos).to(dev))
    bg = torch.zeros(3, device=dev)
    W, H = cam.width, cam.height
    V = d["viewmatrix"].double().cpu()
    nv = torch.linalg.inv(V[:3, :3])[:, 2]          # the plane z = 0 in view space: (t - b) . nv = 0
    b = V[3, :3]
    ys, xs_ = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    u = (2 * xs_ + 1 - W) / W * cam.tanfovx
    v = (2 * ys + 1 - H) / H * cam.tanfovy
    den = u * nv[0] + v * nv[1] + nv[2]
    truth = (b @ nv) / den
    errs = {}
    for rd in (False, True):
        f, _ = _run(d, cam, 0, bg, ray_depth=rd)
        alpha = f["alpha"][0].double().cpu()
        depth = f["depth"][0].double().cpu() / alpha.clamp_min(1e-12)
        ok = (alpha > 0.99) & (truth > 0) & (truth < 60)
        errs[rd] = (depth - truth).abs()[ok]
    print(f"\n[ray depth oblique ground] mean |depth - ray-plane depth|: centre {float(errs[False].mean()):.3e}, ray "
          f"{float(errs[True].mean()):.3e} over {errs[True].numel()} pixels; worst centre {float(errs[False].max()):.3e}"
          f", ray {float(errs[True].max()):.3e}")
    assert errs[True].numel() > 1000
    assert float(errs[True].mean()) < float(errs[False].mean())


# ----------------------------------------------------------------------------- GPU: composition
@pytest.mark.gpu
def test_diff_gauss_composition(cuda_device, monkeypatch):
    """diff_gauss with offsets, the deterministic mode and camera / focal gradients: six outputs, every one but the
    depth bit-identical to the call without ray depth; two deterministic runs bit-identical; the depth alone reaches
    positions, scales, rotations and the camera."""
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam, d = _small_case(dev, seed=11)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, seed=4)
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", True)

    def run(rd, view_grad=False, tan_grad=False, det=False, only=False, q=None):
        leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
        view = d["viewmatrix"].clone().requires_grad_(view_grad)
        tanx = torch.tensor(cam.tanfovx, requires_grad=True) if tan_grad else cam.tanfovx
        rs = GaussianRasterizationSettings(cam.height, cam.width, tanx, cam.tanfovy, 0.1, off,
                                           torch.zeros(3, device=dev), 1.0, view, d["projmatrix"], scene.sh_degree,
                                           d["campos"], False, False)
        means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
        out = GaussianRasterizer(rs, depth_quantile=q, ray_depth=rd)(
            leaves["means3D"], means2D, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
            rotations=leaves["rotations"])
        loss = out[1].mean() if only else (out[0].sum() + 0.01 * out[1].sum() + (out[6].mean() if q else 0.0))
        with Hh.deterministic(det):
            loss.backward()
        grads = [leaves[k].grad for k in leaves] + ([view.grad] if view_grad else []) + ([tanx.grad] if tan_grad
                                                                                          else [])
        return out, grads

    o0, _ = run(False)
    for kw in (dict(), dict(view_grad=True), dict(view_grad=True, tan_grad=True), dict(q=0.5)):
        o1, g1 = run(True, det=True, **kw)
        assert len(o1) == (7 if kw.get("q") else 6)
        for i in (0, 2, 3, 4, 5):
            assert torch.equal(bits(o0[i]), bits(o1[i])), i
        _, g2 = run(True, det=True, **kw)
        for a, b in zip(g1, g2):
            assert a is not None and torch.equal(bits(a), bits(b)) and bool(torch.isfinite(a).all())
    o, g = run(True, view_grad=True, tan_grad=True, det=True, only=True)
    for k in (0, 1, 2, 3, 5, 6):
        assert float(g[k].abs().sum()) > 0, k
    assert int((g[4] != 0).sum()) == 0
    # the ray depth's gradient with respect to scales and rotations is not the centre depth's (which reaches them
    # through alpha only)
    _, g0 = run(False, det=True, only=True)
    assert not torch.equal(g0[1], g[1]) and not torch.equal(g0[2], g[2])
    # the default (atomic) backward agrees with the deterministic one
    _, gd = run(True, only=True)
    for a, b in zip(g[:4], gd[:4]):
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-12


@pytest.mark.gpu
def test_rotation_fit_to_a_sloped_target(cuda_device):
    """Flat surfels at the right heights but lying level, under a nadir orthographic camera, against the depth of a
    20-degree slope: 60 Adam steps on the rotations alone lower the depth L1, with finite gradients throughout."""
    from sfgs.ortho import nadir_camera, OrthoRasterizationSettings, OrthoRasterizer
    dev = cuda_device
    theta, sp, ext = math.radians(20.0), 0.5, 8.0
    means, scales, rots_true, opac = _sloped_roof(dev, theta, sp, ext)
    cam = nadir_camera(-ext, ext, -ext, ext, 0.1, 20.0)
    rs = OrthoRasterizationSettings(cam.image_height, cam.image_width, cam.half_width, cam.half_height, 0.1,
                                    torch.zeros(3, device=dev), 1.0, cam.viewmatrix.to(dev), cam.projmatrix.to(dev),
                                    0, False, False)
    rast = OrthoRasterizer(rs, ray_depth=True)
    colors = torch.zeros((means.shape[0], 3), device=dev)
    with torch.no_grad():
        out = rast(means, torch.zeros_like(means), opac, colors_precomp=colors, scales=scales, rotations=rots_true)
        target, mask = out[1] / out[3].clamp_min(1e-6), out[3] > 0.9
    q = torch.tensor([1.0, 0.0, 0.0, 0.0], device=dev).expand_as(rots_true).clone().requires_grad_(True)
    opt = torch.optim.Adam([q], lr=0.01)
    first = None
    for _ in range(60):
        opt.zero_grad()
        o = rast(means, torch.zeros_like(means), opac, colors_precomp=colors, scales=scales, rotations=q)
        loss = ((o[1] / o[3].clamp_min(1e-6) - target).abs() * mask).sum() / mask.sum()
        loss.backward()
        assert bool(torch.isfinite(q.grad).all())
        first = float(loss) if first is None else first
        opt.step()
    with torch.no_grad():
        o = rast(means, torch.zeros_like(means), opac, colors_precomp=colors, scales=scales, rotations=q)
        last = float(((o[1] / o[3].clamp_min(1e-6) - target).abs() * mask).sum() / mask.sum())
    print(f"\n[ray depth rotation fit] depth L1 {first:.4e} -> {last:.4e} after 60 Adam steps on rotations")
    assert first > 0 and last <= 0.5 * first


if __name__ == "__main__":
    print(json.dumps(_rejections()))
