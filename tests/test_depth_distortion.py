"""The depth distortion: sfgs_rasterize_forward_distortion / sfgs_rasterize_backward_distortion and the Python surface
on top of them (rasterize_gaussians(depth_distortion=True), diff_gauss.GaussianRasterizer(settings,
depth_distortion=True), sfgs.ortho.OrthoRasterizer(settings, depth_distortion=True)).

The oracle of the value is a float64 walk of each pixel's list with the forward's applied set; the oracle of the blend
adjoint is a float64 autograd restatement of the compositing over the GPU's own lists and records; end to end, the
chain_f64 restatement of the per-Gaussian stage, finite differences and a descent check."""
import ctypes as C
import json
import os
import subprocess
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200")):   # the child process of the rejection test starts bare
    if _p not in sys.path:
        sys.path.insert(0, _p)

import helpers as Hh  # noqa: E402
from helpers import bits, release_cached_frames  # noqa: F401,E402

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4


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

    def fwd(a, r=ptr, s=ptr, off=None, ortho=0):
        return L.sfgs_rasterize_forward_distortion(None if a is None else C.byref(a), off, ortho, r, s)

    def bwd(b, s=ptr, g=ptr, ncam=0, cam=ptr, det=0, off=None, ortho=0):
        return L.sfgs_rasterize_backward_distortion(None if b is None else C.byref(b), off, ortho, det, s, g, cam,
                                                    ncam)

    cases = {
        "fwd null args": lambda: fwd(None),
        "fwd null out_distortion": lambda: fwd(fwd_args(), r=None),
        "fwd null out_distortion_state": lambda: fwd(fwd_args(), s=None),
        "fwd null state before ED": lambda: fwd(fwd_args(ED=2), s=None),
        "fwd ED=2": lambda: fwd(fwd_args(ED=2, extra_attrs=ptr, out_extra=ptr)),
        "fwd band": lambda: fwd(fwd_args(tile_row_begin=0, tile_row_end=1)),
        "fwd out_peers": lambda: fwd(fwd_args(out_peers=peers, n_out_peers=2)),
        "fwd ED with offsets": lambda: fwd(fwd_args(ED=2), off=ptr),
        "fwd ortho bad extent": lambda: fwd(fwd_args(tan_fovx=-1.0), ortho=1),
        "fwd bad sizes": lambda: fwd(fwd_args(width=0)),
        "fwd null output": lambda: fwd(fwd_args(out_depth=None)),
        "fwd misaligned rotations": lambda: fwd(fwd_args(rotations=ptr + 4)),
        "bwd null args": lambda: bwd(None),
        "bwd null distortion_state": lambda: bwd(bwd_args(), s=None),
        "bwd null dL_dpix_distortion": lambda: bwd(bwd_args(), g=None),
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


_FWD, _BWD = "forward_distortion", "backward_distortion"
_NULL_OUT = "null out_distortion or out_distortion_state"
_NULL_IN = "null distortion_state or dL_dpix_distortion"
# case: (code, entry, text of the winning check)
EXPECTED = {
    "fwd null args": (SFGS_E_BADARG, _FWD, "null args"),
    "fwd null out_distortion": (SFGS_E_BADARG, _FWD, _NULL_OUT),
    "fwd null out_distortion_state": (SFGS_E_BADARG, _FWD, _NULL_OUT),
    "fwd null state before ED": (SFGS_E_BADARG, _FWD, _NULL_OUT),
    "fwd ED=2": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with the depth distortion"),
    "fwd band": (SFGS_E_UNSUPPORTED, _FWD, "tile-row bands are not supported with the depth distortion"),
    "fwd out_peers": (SFGS_E_UNSUPPORTED, _FWD, "out_peers are not supported with the depth distortion"),
    "fwd ED with offsets": (SFGS_E_UNSUPPORTED, _FWD, "extra_attrs are not supported with the depth distortion"),
    "fwd ortho bad extent": (SFGS_E_BADARG, _FWD, "the half-extents tan_fovx, tan_fovy must be finite and > 0"),
    "fwd bad sizes": (SFGS_E_BADARG, _FWD, "bad sizes"),
    "fwd null output": (SFGS_E_BADARG, _FWD, "null output"),
    "fwd misaligned rotations": (SFGS_E_BADARG, _FWD, "rotations must be 16-byte aligned"),
    "bwd null args": (SFGS_E_BADARG, _BWD, "null args"),
    "bwd null distortion_state": (SFGS_E_BADARG, _BWD, _NULL_IN),
    "bwd null dL_dpix_distortion": (SFGS_E_BADARG, _BWD, _NULL_IN),
    **{f"bwd ncam={n}": (SFGS_E_BADARG, _BWD, "ncam must be 0, 35 or 37") for n in (-1, 1, 36, 38)},
    "bwd ncam before ED": (SFGS_E_BADARG, _BWD, "ncam must be 0, 35 or 37"),
    "bwd ED=2": (SFGS_E_UNSUPPORTED, _BWD, "extra_attrs are not supported with the depth distortion"),
    "bwd band": (SFGS_E_UNSUPPORTED, _BWD, "tile-row bands are not supported with the depth distortion"),
    "bwd acc_peers": (SFGS_E_UNSUPPORTED, _BWD, "acc_peers are not supported with the depth distortion"),
    "bwd phase 2": (SFGS_E_UNSUPPORTED, _BWD, "phase 2 is not supported with the depth distortion"),
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
                                             8, 8, e, 0, e, False, False, depth_distortion=True, **kw)
    for kw, what in ((dict(depth_quantile=0.5), "depth_quantile"), (dict(graph=True), "graph"),
                     (dict(tile_rows=(0, 1)), "tile_rows"), (dict(out_peers=[0]), "out_peers"),
                     (dict(F=2), "extra_attrs")):
        with pytest.raises(N.SfgsError, match=f"{what}.*not supported with the depth distortion"):
            fwd(**kw)
    g = torch.zeros((3, 8, 8))
    st = torch.zeros((2, 8, 8))
    bwd = lambda **kw: R.rasterize_gaussians_backward(  # noqa: E731
        e, m, e, e, e, e, kw.pop("ex", e), 1.0, e, e, e, e, 1.0, 1.0, 0.1, g, g[:1], g, g[:1], e, e, 0, e, e, 0, e, e,
        e, False, distortion_state=st, dL_dout_distortion=g[:1], **kw)
    for kw, what in ((dict(depth_q_pos=torch.zeros((8, 8), dtype=torch.int32), dL_dout_depth_q=g[:1]),
                      "depth_q_pos"), (dict(graph=True), "graph"), (dict(tile_rows=(0, 1)), "tile_rows"),
                     (dict(acc_peers=[0], phase=1), "acc_peers"), (dict(ex=torch.zeros((4, 2))), "extra_attrs")):
        with pytest.raises(N.SfgsError, match=f"{what}.*not supported with the depth distortion"):
            bwd(**kw)
    # the tensors are checked before their pointers are handed over
    bwd2 = lambda **kw: R.rasterize_gaussians_backward(  # noqa: E731
        e, m, e, e, e, e, e, 1.0, e, e, e, e, 1.0, 1.0, 0.1, g, g[:1], g, g[:1], e, e, 0, e, e, 0, e, e, e, False, **kw)
    for s, c, what in ((st, g[:1].double(), "dL_dout_distortion"), (st, g[:1, :4], "dL_dout_distortion"),
                       (st.int(), g[:1], "distortion_state"), (st[:1], g[:1], "distortion_state")):
        with pytest.raises(ValueError, match=what):
            bwd2(distortion_state=s, dL_dout_distortion=c)
    with pytest.raises(ValueError, match="come together"):
        bwd2(distortion_state=st)


def test_modules_reject_before_native_calls(monkeypatch):
    """diff_gauss and OrthoRasterizer raise on the quantile and the distortion in one call, and diff_gauss raises under
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
    with pytest.raises(N.SfgsError, match="depth_distortion and depth_quantile"):
        GaussianRasterizer(rs, depth_quantile=0.5, depth_distortion=True)(m, m, torch.ones((4, 1)), **kw)
    ors = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3, False,
                                     False)
    with pytest.raises(N.SfgsError, match="depth_distortion and depth_quantile"):
        OrthoRasterizer(ors, depth_quantile=0.5, depth_distortion=True)(m, m, torch.ones((4, 1)), **kw)

    def no_capacity(*a, **k):
        raise AssertionError("capture-time work before the distortion's check")
    monkeypatch.setattr(diff_gauss._graphs, "resolve_capacity", no_capacity)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    mc = types.SimpleNamespace(is_cuda=True)
    with pytest.raises(N.SfgsError, match="depth distortion cannot be captured"):
        diff_gauss._RasterizeGaussians.forward(types.SimpleNamespace(), mc, m, m, m, m, m, m, m, m, torch.empty(0),
                                               rs, False, None, None, None, None, None, None, True)


def test_ortho_rasterizer_rejects_capture_before_native_calls(monkeypatch):
    """OrthoRasterizer runs through diff_gauss's Function: under stream capture it raises before any capture-time
    work (the capacity is not resolved) and before any native call."""
    import diff_gauss
    from sfgs import native as N
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer

    def no_lib():
        raise AssertionError("native library called")

    def no_capacity(*a, **k):
        raise AssertionError("capture-time work before the orthographic camera's check")
    monkeypatch.setattr(N, "lib", no_lib)
    monkeypatch.setattr(diff_gauss._graphs, "resolve_capacity", no_capacity)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    m = torch.zeros((4, 3))
    kw = dict(shs=torch.zeros((4, 16, 3)), scales=torch.ones((4, 3)), rotations=torch.zeros((4, 4)))
    ors = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3, False,
                                     False)
    for opts, what in ((dict(), "the orthographic camera"), (dict(depth_distortion=True), "the depth distortion")):
        with pytest.raises(N.SfgsError, match=f"diff_gauss: {what} cannot be captured in a CUDA graph"):
            OrthoRasterizer(ors, **opts)(m, m, torch.ones((4, 1)), **kw)


def test_ortho_rasterizer_is_an_ordinary_module():
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer
    rs = OrthoRasterizationSettings(8, 8, 1.0, 1.0, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, False, False)

    class Holder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.r = OrthoRasterizer(rs, depth_distortion=True)
            self.w = torch.nn.Parameter(torch.zeros(2))

    for m in (OrthoRasterizer(rs, depth_distortion=True), Holder()):
        assert m.to("cpu") is m and m.float() is m and m.cpu() is m and m.double() is m
    assert Holder().double().w.dtype == torch.float64


# ----------------------------------------------------------------------------- the float64 restatements
def _tile_pixels(tile, W, H, dev, off=None):
    tiles_x = (W + 15) // 16
    ty, tx = divmod(int(tile), tiles_x)
    yy, xx = torch.meshgrid(torch.arange(16, device=dev) + 16 * ty, torch.arange(16, device=dev) + 16 * tx,
                            indexing="ij")
    inside = (xx < W) & (yy < H)
    xx, yy = xx[inside], yy[inside]
    px, py = xx.double(), yy.double()
    if off is not None:
        px, py = px + off[yy, xx, 0].double(), py + off[yy, xx, 1].double()
    return yy * W + xx, px, py


def _applied(I, tile, pid, px, py, clamped=False):
    """The forward's applied set of the tile's pixels [pixels, records]: the skip tests in float32 and the cut at
    n_contrib, and the pixels where a record's float32 skip test is within rounding of its threshold (ambiguous; with
    clamped=True also those that apply a record at the 0.99 alpha clamp, whose gradient the adjoint passes through)."""
    r0, r1 = (int(v) for v in I["ranges"][tile])
    g = I["rec"][I["point_list"][r0:r1].long()]
    dx, dy = g[None, :, 0] - px.float()[:, None], g[None, :, 1] - py.float()[:, None]
    power = -0.5 * (g[None, :, 2] * dx * dx + g[None, :, 4] * dy * dy) - g[None, :, 3] * dx * dy
    araw = g[None, :, 5] * torch.exp(power)
    ok = ~(power > 0) & ~(torch.clamp(araw, max=0.99) < 1.0 / 255.0)
    pos = torch.arange(1, r1 - r0 + 1, device=g.device)
    within = pos[None, :] <= I["n_contrib"][pid].long()[:, None]
    near = ((araw * 255.0 - 1.0).abs() < 1e-5) | (power.abs() < 1e-6) | (clamped & (araw >= 0.99))
    return ok & within, (near & within).any(1), r0, r1


def _composite(rec, pl, M, px, py, dtype):
    """w, T_final, records [P?] of one tile in `dtype`, differentiable w.r.t. rec; the forward's applied set M.  The
    0.99 clamp passes the gradient through, as the kernels' h = G dL/dalpha does."""
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


def _distortion_of(w, m, ref=None):
    """R = A M2 with mu = sum w m / A, M2 = sum w (m - mu)^2 (0 where A = 0), in the dtype of w; with ref [pixels], the
    depths are taken about it first (the float64 walk: a pixel whose records share one depth then gets exactly 0)."""
    A = w.sum(1)
    safe = torch.where(A > 0, A, torch.ones_like(A))
    d = m[None, :] if ref is None else m[None, :] - ref[:, None]
    mu = (w * d).sum(1) / safe
    return A * (w * (d - mu[:, None]) ** 2).sum(1)


def f64_distortion(I, W, H, tiles, off=None):
    """Per pixel of `tiles`: (ids, R64, bound scale A sum w (m - m_first)^2, ambiguous) of a float64 walk with the
    forward's applied set."""
    dev = I["rec"].device
    rec = I["rec"].double()
    ids, Rs, scale, amb = [], [], [], []
    for tile in tiles:
        pid, px, py = _tile_pixels(tile, W, H, dev, off)
        M, near, r0, r1 = _applied(I, tile, pid, px, py)
        if r1 == r0:
            z = torch.zeros_like(px)
            ids.append(pid); Rs.append(z); scale.append(z); amb.append(torch.zeros_like(pid, dtype=torch.bool))
            continue
        w, _, g, *_ = _composite(rec, I["point_list"][r0:r1].long(), M, px, py, torch.float64)
        m = g[:, 6]
        first = torch.where(M.any(1), M.int().argmax(1), torch.zeros_like(pid))
        d = m[None, :] - m[first][:, None]
        ids.append(pid); Rs.append(_distortion_of(w, m, m[first])); amb.append(near)
        scale.append(w.sum(1) * (w * d * d).sum(1))
    return torch.cat(ids), torch.cat(Rs), torch.cat(scale), torch.cat(amb)


def blend_restatement(I, W, H, bg, cot, c, dtype, off=None):
    """The phase-1 sums [P,16] of the blend adjoint restated in `dtype` with autograd over the GPU's lists and
    records, for the cotangents (colour, depth, normal, alpha) and c of the distortion.  Words: 0-2 colour, 3 depth,
    4-6 normal, 7-8 (W/2, H/2) x d/d mean2D, 9 the abs-gradient sum, 10-12 d/d conic (x, y/2, z), 13 d/d opacity."""
    dev = I["rec"].device
    rec = I["rec"].to(dtype).detach().clone().requires_grad_(True)
    bgd = bg.to(dtype)
    loss = torch.zeros((), dtype=dtype, device=dev)
    alphas, keep = [], []
    for tile in range(I["ranges"].shape[0]):
        pid, px, py = _tile_pixels(tile, W, H, dev, off)
        M, _, r0, r1 = _applied(I, tile, pid, px, py)
        if r1 == r0:
            continue
        pl = I["point_list"][r0:r1].long()
        w, T, g, dx, dy, G, araw = _composite(rec, pl, M, px, py, dtype)
        araw.retain_grad()
        col = w @ g[:, 8:11] + T[:, None] * bgd[None, :]
        dep, nor, alp = w @ g[:, 6], w @ g[:, 11:14], 1 - T
        R = _distortion_of(w, g[:, 6])
        ct = lambda t, k: t.reshape(t.shape[0], -1)[:, pid].to(dtype)  # noqa: E731
        loss = loss + (ct(cot[0], 0).T * col).sum() + (ct(cot[1], 0)[0] * dep).sum() + \
            (ct(cot[2], 0).T * nor).sum() + (ct(cot[3], 0)[0] * alp).sum() + (ct(c, 0)[0] * R).sum()
        alphas.append(araw)
        keep.append((pl, g.detach(), dx.detach(), dy.detach(), G.detach()))
    loss.backward()
    gr = rec.grad
    out = torch.zeros((rec.shape[0], 16), dtype=dtype, device=dev)
    out[:, 0:3], out[:, 3], out[:, 4:7] = gr[:, 8:11], gr[:, 6], gr[:, 11:14]
    out[:, 7], out[:, 8] = 0.5 * W * gr[:, 0], 0.5 * H * gr[:, 1]
    out[:, 10], out[:, 11], out[:, 12], out[:, 13] = gr[:, 2], 0.5 * gr[:, 3], gr[:, 4], gr[:, 5]
    for araw, (pl, g, dx, dy, G) in zip(alphas, keep):
        h = G * araw.grad
        u = 0.5 * W * (g[None, :, 2] * dx + g[None, :, 3] * dy)
        v = 0.5 * H * (g[None, :, 3] * dx + g[None, :, 4] * dy)
        out[:, 9].index_add_(0, pl, g[:, 5].abs() * (h.abs() * (u.abs() + v.abs())).sum(0))
    return out


# ----------------------------------------------------------------------------- GPU helpers
def _headline(dev):
    _, cam, D, d, _ = Hh.frame("jax004", dev)
    return cam, D, d, torch.tensor([0.0, 0.0, 0.0], device=dev)


def _ortho_headline(cam, d):
    from sfgs.ortho import projection_matrix
    oc = types.SimpleNamespace(width=cam.width, height=cam.height, tanfovx=60.0, tanfovy=60.0 * 1080 / 1920)
    proj = d["viewmatrix"].cpu().double() @ projection_matrix(oc.tanfovx, oc.tanfovy, 0.01, 1e4).double()
    return oc, dict(d, projmatrix=proj.float().to(d["means3D"].device))


def _run_forward(d, cam, D, bg, **kw):
    """One forward with the distortion: the ten-output dict, distortion and distortion_state."""
    from sfgs import rasterizer as R
    e = torch.empty(0, device=d["means3D"].device)
    out = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cam.height,
                                cam.width, d["shs"], D, d["campos"], False, False, depth_distortion=True, **kw)
    return dict(zip(Hh.FWD_KEYS, out[:10])), out[10], out[11]


def _cot(H, W, dev, seed, others=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda *s: torch.randn(s, generator=g, device=dev)  # noqa: E731
    z = lambda *s: torch.zeros(s, device=dev)  # noqa: E731
    cot = (r(3, H, W), r(1, H, W) * 0.1, r(3, H, W), r(1, H, W)) if others else (z(3, H, W), z(1, H, W),
                                                                               z(3, H, W), z(1, H, W))
    return cot, r(1, H, W)


# ----------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pinhole", "jitter", "ortho"])
def test_no_interference_forward(cuda_device, form):
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    kw = {}
    if form == "jitter":
        kw["subpixel_offset"] = Hh.uniform_offsets(cam.height, cam.width, dev, seed=3)
    if form == "ortho":
        cam, d = _ortho_headline(cam, d)
        kw["ortho"] = True
    a = Hh.run_ours_forward(d, cam, D, bg, **kw)
    b, R, st = _run_forward(d, cam, D, bg, **kw)
    for k in ("color", "depth", "norm", "alpha", "radii"):
        assert torch.equal(bits(a[k]), bits(b[k])), k
    n = a["num_rendered"]
    assert n == b["num_rendered"] and n > 0
    Ia = Hh.our_internals(a, d["means3D"].shape[0], cam.height, cam.width)
    Ib = Hh.our_internals(b, d["means3D"].shape[0], cam.height, cam.width)
    for k in ("n_contrib", "point_list", "ranges"):
        assert torch.equal(Ia[k], Ib[k]), k
    assert bool(torch.isfinite(R).all()) and bool((R >= 0).all()) and float(R.max()) > 0
    assert bool(torch.isfinite(st).all())


@pytest.mark.gpu
@pytest.mark.parametrize("form,ncam", [("pinhole", 0), ("pinhole", 35), ("pinhole", 37), ("jitter", 37),
                                       ("ortho", 0)])
def test_no_interference_deterministic_backward(cuda_device, form, ncam):
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    kw = {}
    if form == "jitter":
        kw["subpixel_offset"] = Hh.uniform_offsets(cam.height, cam.width, dev, seed=3)
    if form == "ortho":
        cam, d = _ortho_headline(cam, d)
        kw["ortho"] = True
    fwd, _, st = _run_forward(d, cam, D, bg, **kw)
    cot, _ = _cot(cam.height, cam.width, dev, seed=1)
    zero = torch.zeros((1, cam.height, cam.width), device=dev)
    kw.update(camera_grad=ncam > 0, intrinsics_grad=ncam == 37)
    a = Hh.run_ours_backward(d, cam, D, bg, fwd, cot, det=True, **kw)
    b = Hh.run_ours_backward(d, cam, D, bg, fwd, cot, det=True, distortion_state=st, dL_dout_distortion=zero, **kw)
    assert set(a) == set(b)
    for k in a:      # equal as values: the sign of a zero may differ
        assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
def test_forward_value(cuda_device):
    dev = cuda_device
    cam, D, d, bg = _headline(dev)
    W, H = cam.width, cam.height
    fwd, R, st = _run_forward(d, cam, D, bg)
    I = Hh.our_internals(fwd, d["means3D"].shape[0], H, W)
    g = torch.Generator().manual_seed(7)
    tiles = torch.randperm(I["ranges"].shape[0], generator=g)[:96].tolist()
    ids, R64, scale, amb = f64_distortion(I, W, H, tiles)
    ours = R.reshape(-1)[ids].double()
    ratio = (ours - R64).abs() / (1e-5 * scale + 1e-30)
    ok = ~amb
    print(f"\n[depth distortion] f64 walk over {ids.numel()} pixels of {len(tiles)} tiles ({int(amb.sum())} with a "
          f"record at a skip threshold): worst |R - R64| / (1e-5 A sum w (m - m_first)^2) {float(ratio[ok].max()):.3e}; "
          f"largest R {float(R64.max()):.3e}")
    assert bool((ratio[ok] <= 1.0).all())
    # the state: mu and M2 = R / A
    A = fwd["alpha"].reshape(-1)[ids].double()
    M2 = st[1].reshape(-1)[ids].double()
    has = ok & (A > 1e-3)
    assert bool(((M2 * A - R64).abs()[has] <= 1e-4 * scale[has] / A[has] + 1e-5 * R64[has] + 1e-30).all())


@pytest.mark.gpu
def test_depth_shift_invariance(cuda_device):
    from sfgs.ortho import nadir_camera, OrthoRasterizationSettings, OrthoRasterizer
    from test_ortho import stepped_surfels
    dev = cuda_device
    means, scales, rots, opac, _, _ = stepped_surfels(dev)
    # semi-transparent floaters above the surface: a real spread of depths along the rays
    g = torch.Generator(device=dev).manual_seed(2)
    F = 4000
    fl = torch.stack([torch.rand(F, generator=g, device=dev) * 56 - 28, torch.rand(F, generator=g, device=dev) * 56 - 28,
                      torch.rand(F, generator=g, device=dev) * 15 + 22], 1)
    means = torch.cat([means, fl])
    scales = torch.cat([scales, torch.full((F, 3), 0.3, device=dev)])
    rots = torch.cat([rots, torch.tensor([1.0, 0, 0, 0], device=dev).expand(F, 4)]).contiguous()
    opac = torch.cat([opac, torch.full((F, 1), 0.3, device=dev)])
    colors = torch.rand((means.shape[0], 3), generator=g, device=dev)
    outs = []
    for z_top in (50.0, 1050.0):
        cam = nadir_camera(-30.0, 30.0, -30.0, 30.0, 60.0 / 256, z_top)
        rs = OrthoRasterizationSettings(cam.image_height, cam.image_width, cam.half_width, cam.half_height, 0.1,
                                        torch.zeros(3, device=dev), 1.0, cam.viewmatrix.to(dev),
                                        cam.projmatrix.to(dev), 0, False, False)
        from sfgs import rasterizer as R
        e = torch.empty(0, device=dev)
        f = R.rasterize_gaussians(rs.bg, means, colors, opac, scales, rots, 1.0, e, e, e, 0, rs.viewmatrix,
                                  rs.projmatrix, cam.half_width, cam.half_height, 0.1, cam.image_height,
                                  cam.image_width, e, 0, torch.zeros(3, device=dev), False, False, ortho=True,
                                  depth_distortion=True)
        o7 = OrthoRasterizer(rs, depth_distortion=True)(means, torch.zeros_like(means), opac, colors_precomp=colors,
                                                        scales=scales, rotations=rots)
        assert torch.equal(bits(o7[6].detach()), bits(f[10]))
        outs.append((cam, dict(zip(Hh.FWD_KEYS, f[:10])), f[10]))
    (cam, a, Ra), (_, b, Rb) = outs
    W, H = cam.image_width, cam.image_height
    assert torch.equal(bits(a["color"]), bits(b["color"])) and torch.equal(bits(a["alpha"]), bits(b["alpha"]))
    P = means.shape[0]
    Ia, Ib = Hh.our_internals(a, P, H, W), Hh.our_internals(b, P, H, W)
    vis = a["radii"] > 0
    assert float((Ib["rec"][vis, 6] - Ia["rec"][vis, 6] - 1000.0).abs().max()) <= 1e-3
    assert float((b["depth"] - a["depth"] - 1000.0 * a["alpha"]).abs().max()) <= 1e-2
    assert float(Ra.max()) > 1.0
    worst = []
    for I, Rv in ((Ia, Ra), (Ib, Rb)):
        ids, R64, scale, amb = f64_distortion(I, W, H, range(I["ranges"].shape[0]))
        ratio = ((Rv.reshape(-1)[ids].double() - R64).abs() / (1e-5 * scale + 1e-30))[~amb]
        worst.append(float(ratio.max()))
    print(f"\n[depth distortion shift] worst |R - R64| / bound at z_top 50 and 1050: {worst[0]:.3e}, {worst[1]:.3e}; "
          f"max |R(1050) - R(50)| / max R {float((Rb - Ra).abs().max() / Ra.max()):.2e}")
    assert max(worst) <= 1.0


def _small_case(dev, seed=5, P=3000):
    from sfgs import synthetic as S
    scene = S.blob_scene(P, seed=seed)
    cam = S.simple_camera(160, 120)
    return scene, cam, Hh.to_torch(scene, cam, dev)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
def test_blend_adjoint_sums(cuda_device, det):
    """Phase-1 sums with every cotangent plus the distortion's against the float64 restatement.  The adjoint recovers T
    back to front, so even on the words the distortion does not touch (colour and normal, 0-2 and 4-6) its worst error
    is a multiple rho of the float32 restatement's (about 60 on this frame).  Bound per word: twice the larger of rho
    times the float32 restatement's worst error and the adjoint's own worst error without the distortion (c = 0), +1e-6
    of the word's largest value: the distortion's terms may be no less accurate than the terms the adjoint already
    forms.  Pixels with a record at a float32 skip threshold get zero cotangents (their applied set is not decidable
    here)."""
    dev = cuda_device
    scene, cam, d = _small_case(dev)
    W, H, D = cam.width, cam.height, scene.sh_degree
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    fwd, _, st = _run_forward(d, cam, D, bg)
    I = Hh.our_internals(fwd, d["means3D"].shape[0], H, W)
    ids, _, _, amb = f64_distortion(I, W, H, range(I["ranges"].shape[0]))
    keep = torch.ones(H * W, device=dev)
    keep[ids[amb]] = 0
    keep = keep.reshape(1, H, W)
    cot, c = _cot(H, W, dev, seed=4)
    cot = tuple(t * keep for t in cot)
    c = c * keep

    def acc(cd):
        return Hh.run_ours_backward(d, cam, D, bg, fwd, cot, det=det, phase=1, distortion_state=st,
                                    dL_dout_distortion=cd)
    a, a0 = acc(c), acc(torch.zeros_like(c))
    r64 = blend_restatement(I, W, H, bg, cot, c, torch.float64)
    r32 = blend_restatement(I, W, H, bg, cot, c, torch.float32).double()
    r64_0 = blend_restatement(I, W, H, bg, cot, torch.zeros_like(c), torch.float64)
    vis = fwd["radii"] > 0
    e32, e0, err, floor, share = [], [], [], [], []
    for k in range(14):
        ref = r64[vis, k]
        e32.append(float((r32[vis, k] - ref).abs().max()) + 1e-30)
        e0.append(float((a0[vis, k].double() - r64_0[vis, k]).abs().max()))
        err.append(float((a[vis, k].double() - ref).abs().max()))
        floor.append(1e-6 * float(ref.abs().max()) + 1e-30)
        share.append(float((ref - r64_0[vis, k]).abs().max() / ref.abs().max().clamp_min(1e-30)))
    rho = max(err[k] / e32[k] for k in (0, 1, 2, 4, 5, 6))
    worst = [err[k] / (2.0 * max(rho * e32[k], e0[k]) + floor[k]) for k in range(14)]
    print(f"\n[depth distortion blend adjoint det={det}] {int(amb.sum())} pixels held out; rho {rho:.1f}; worst err / "
          "bound per word: " + ", ".join(f"{v:.2f}" for v in worst) + "\n  worst err / float32 restatement's: "
          + ", ".join(f"{err[k] / e32[k]:.1f}" for k in range(14)) + "\n  largest distortion term / largest value "
          "per word: " + ", ".join(f"{v:.2f}" for v in share))
    assert all(v <= 1.0 for v in worst), worst
    assert int((a[~vis] != 0).sum()) == 0
    if det:
        assert torch.equal(bits(a), bits(acc(c)))


def _chain_case(dev):
    def make():
        import chain_f64 as CH
        from sfgs import synthetic as S
        cam, D, d, _ = _headline(dev)
        bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
        fwd, _, st = _run_forward(d, cam, D, bg)
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=6)]
        gd = torch.randn((1, cam.height, cam.width), generator=torch.Generator(device=dev).manual_seed(8),
                         device=dev) * 1e-3
        a = Hh.restatement_inputs(fwd, d, cam, D, bg, cot)
        a["acc"] = Hh.run_ours_backward(d, cam, D, bg, fwd, cot, det=True, phase=1, distortion_state=st,
                                        dL_dout_distortion=gd)
        a.update(cov3D=None, scales=d["scales"], rotations=d["rotations"])
        r64 = CH.chain(**a, focal=True, dtype=torch.float64)
        r32 = CH.chain(**a, focal=True, dtype=torch.float32)
        return cam, D, d, bg, fwd, st, cot, gd, r64, r32
    return Hh.cached("chain", "jax004-distortion", make)


def _camera_flat(r, ncam):
    v = [r["view"].reshape(16), r["proj"].reshape(16), r["campos"].reshape(3)]
    if ncam == 37:
        v += [r["tanx"].reshape(1), r["tany"].reshape(1)]
    return torch.cat(v).double()


@pytest.mark.gpu
@pytest.mark.parametrize("ncam", [0, 35, 37])
def test_gradients_against_restatement(cuda_device, ncam):
    """The ten gradients and the camera / focal terms of the deterministic backward with every cotangent plus the
    distortion's, against chain_f64 on the same sums, with the bounds of test_depth_quantile.py."""
    cam, D, d, bg, fwd, st, cot, gd, r64, r32 = _chain_case(cuda_device)
    g = Hh.run_ours_backward(d, cam, D, bg, fwd, cot, det=True, camera_grad=ncam > 0, intrinsics_grad=ncam == 37,
                             distortion_state=st, dL_dout_distortion=gd)
    worst = {}
    for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot"):
        ref, ref32 = r64[k].double(), r32[k].double()
        ours = g[k].detach().double().reshape(ref.shape)
        lim = 2.0 * float((ref32 - ref).abs().max()) + 1e-6 * float(ref.abs().max())
        worst[k] = float((ours - ref).abs().max()) / lim
    print(f"\n[depth distortion chain ncam={ncam}] worst err / bound per gradient: "
          + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), (ncam, worst)
    if ncam:
        gpu = torch.cat([g["view"].reshape(16), g["proj"].reshape(16), g["campos"].reshape(3)]
                        + ([g["tanx"].reshape(1), g["tany"].reshape(1)] if ncam == 37 else [])).double()
        f64, f32 = _camera_flat(r64, ncam), _camera_flat(r32, ncam)
        tol = torch.maximum(2.0 * (f32 - f64).abs(), 1e-6 * r64["abs"][:ncam].double())
        err = (gpu - f64).abs()
        print(f"[depth distortion chain ncam={ncam}] camera max err / tol {float((err / tol.clamp_min(1e-300)).max()):.3f}")
        assert (err <= tol).all(), (ncam, err, tol)


@pytest.mark.gpu
def test_finite_differences(cuda_device):
    """d/d means3D and d/d opacities of sum c R on a small scene against central differences, over the pixels whose
    applied set is the same at -eps, 0 and +eps."""
    from sfgs import rasterizer as R
    dev = cuda_device
    scene, cam, d = _small_case(dev, seed=6)
    bg = torch.zeros(3, device=dev)
    W, H, D = cam.width, cam.height, scene.sh_degree
    e = torch.empty(0, device=dev)

    def fwd(m, o):
        return R.rasterize_gaussians(bg, m, e, o, d["scales"], d["rotations"], 1.0, e, e, e, 0, d["viewmatrix"],
                                     d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"], D, d["campos"],
                                     False, False, depth_distortion=True)
    base = fwd(d["means3D"], d["opacities"])
    f0 = dict(zip(Hh.FWD_KEYS, base[:10]))
    P = d["means3D"].shape[0]
    tag = torch.rand(P, generator=torch.Generator(device=dev).manual_seed(1), device=dev, dtype=torch.float64)

    def applied_sets(out):
        """Per pixel, a float64 sum of random tags over the Gaussians of its applied set (equal sums: equal sets)."""
        I = Hh.our_internals(dict(zip(Hh.FWD_KEYS, out[:10])), P, H, W)
        h = torch.zeros(H * W, dtype=torch.float64, device=dev)
        for tile in range(I["ranges"].shape[0]):
            pid, px, py = _tile_pixels(tile, W, H, dev)
            M, near, r0, r1 = _applied(I, tile, pid, px, py, clamped=True)
            if r1 > r0:
                h[pid] = (M.double() * tag[I["point_list"][r0:r1].long()][None, :]).sum(1)
                h[pid[near]] = -1.0
        return h
    set0 = applied_sets(base)
    c = torch.randn((1, H, W), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    zero = tuple(torch.zeros_like(x) for x in (f0["color"], f0["depth"], f0["norm"], f0["alpha"]))
    g_all = Hh.run_ours_backward(d, cam, D, bg, f0, zero, det=True, distortion_state=base[11], dL_dout_distortion=c)
    picks = torch.argsort(g_all["means3D"].abs().sum(1), descending=True)[:5].tolist()
    worst = 0.0
    for i in picks:
        # opacity: a wider step; a 1e-3 change of R sits near the float32 rounding of R where a faint record lies far
        # in front of the pixel's surface (R is formed about the first applied record's depth)
        for what, k, eps in [("means3D", k, 1e-3) for k in range(3)] + [("opacity", 0, 1e-2)]:
            outs = []
            for s in (1.0, -1.0):
                m, o = d["means3D"].clone(), d["opacities"].clone()
                (m if what == "means3D" else o)[i, k] += s * eps
                outs.append(fwd(m, o))
            stable = set0 >= 0
            for out in outs:
                stable &= applied_sets(out) == set0
            cm = c * stable.reshape(1, H, W)
            fdv = float(((outs[0][10].double() - outs[1][10].double()) * cm).sum()) / (2 * eps)
            g = Hh.run_ours_backward(d, cam, D, bg, f0, zero, det=True, distortion_state=base[11],
                                     dL_dout_distortion=cm)
            an = float(g[what][i, k])
            err = abs(an - fdv) / max(abs(fdv), abs(an), 1e-3)
            worst = max(worst, err)
            assert err <= 3e-2, (what, i, k, an, fdv)
    print(f"\n[depth distortion FD] {len(picks)} Gaussians x (3 means + opacity): worst relative error {worst:.2e}")


@pytest.mark.gpu
def test_diff_gauss_composition(cuda_device, monkeypatch):
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam, d = _small_case(dev, seed=11)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, seed=4)
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", True)

    def run(dist, view_grad=False, tan_grad=False, det=False, only=False):
        leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
        view = d["viewmatrix"].clone().requires_grad_(view_grad)
        tanx = torch.tensor(cam.tanfovx, requires_grad=True) if tan_grad else cam.tanfovx
        rs = GaussianRasterizationSettings(cam.height, cam.width, tanx, cam.tanfovy, 0.1, off,
                                           torch.zeros(3, device=dev), 1.0, view, d["projmatrix"], scene.sh_degree,
                                           d["campos"], False, False)
        means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
        out = GaussianRasterizer(rs, depth_distortion=dist)(leaves["means3D"], means2D, leaves["opacities"],
                                                            shs=leaves["shs"], scales=leaves["scales"],
                                                            rotations=leaves["rotations"])
        loss = out[6].mean() if only else (out[0].sum() + 0.01 * out[1].sum() + (out[6].mean() if dist else 0.0))
        with Hh.deterministic(det):
            loss.backward()
        grads = [leaves[k].grad for k in leaves] + ([view.grad] if view_grad else []) + ([tanx.grad] if tan_grad
                                                                                          else [])
        return out, grads

    o0, _ = run(False)
    assert len(o0) == 6
    for kw in (dict(), dict(view_grad=True), dict(view_grad=True, tan_grad=True)):
        o1, g1 = run(True, det=True, **kw)
        assert len(o1) == 7
        for a, b in zip(o0, o1[:6]):
            assert torch.equal(bits(a), bits(b))
        _, g2 = run(True, det=True, **kw)
        for a, b in zip(g1, g2):
            assert a is not None and torch.equal(bits(a), bits(b)) and bool(torch.isfinite(a).all())
    # the distortion alone reaches positions, opacities, scales and rotations, and the camera; not the colours
    o, g = run(True, view_grad=True, tan_grad=True, det=True, only=True)
    for k in (0, 1, 2, 3, 5, 6):
        assert float(g[k].abs().sum()) > 0, k
    assert int((g[4] != 0).sum()) == 0
    # the default (atomic) backward agrees with the deterministic one
    _, gd = run(True, only=True)
    for a, b in zip(g[:4], gd[:4]):
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-12


@pytest.mark.gpu
def test_descent_removes_floaters(cuda_device):
    """A surface with semi-transparent floaters in front of it: 100 Adam steps on distortion.mean() alone at least
    halve it, with finite gradients throughout."""
    from sfgs.ortho import nadir_camera, OrthoRasterizationSettings, OrthoRasterizer
    from test_ortho import stepped_surfels
    dev = cuda_device
    means, scales, rots, opac, _, _ = stepped_surfels(dev, spacing=0.5, roofs=(), extent=16.0)
    g = torch.Generator(device=dev).manual_seed(9)
    F = 1500
    fl = torch.stack([torch.rand(F, generator=g, device=dev) * 28 - 14, torch.rand(F, generator=g, device=dev) * 28 - 14,
                      torch.rand(F, generator=g, device=dev) * 6 + 2], 1)
    means = torch.cat([means, fl]).contiguous()
    scales = torch.cat([scales, torch.full((F, 3), 0.4, device=dev)]).contiguous()
    rots = torch.cat([rots, torch.tensor([1.0, 0, 0, 0], device=dev).expand(F, 4)]).contiguous()
    logit = torch.logit(torch.cat([opac.clamp(max=0.95), torch.full((F, 1), 0.3, device=dev)])).contiguous()
    cam = nadir_camera(-14.0, 14.0, -14.0, 14.0, 28.0 / 128, 20.0)
    rs = OrthoRasterizationSettings(cam.image_height, cam.image_width, cam.half_width, cam.half_height, 0.1,
                                    torch.zeros(3, device=dev), 1.0, cam.viewmatrix.to(dev), cam.projmatrix.to(dev),
                                    0, False, False)
    rast = OrthoRasterizer(rs, depth_distortion=True)
    colors = torch.full((means.shape[0], 3), 0.5, device=dev)
    m = means.clone().requires_grad_(True)
    lo = logit.clone().requires_grad_(True)
    opt = torch.optim.Adam([m, lo], lr=0.05)
    first = None
    for _ in range(100):
        opt.zero_grad()
        out = rast(m, torch.zeros_like(m), torch.sigmoid(lo), colors_precomp=colors, scales=scales, rotations=rots)
        loss = out[6].mean()
        loss.backward()
        assert bool(torch.isfinite(m.grad).all()) and bool(torch.isfinite(lo.grad).all())
        first = float(loss) if first is None else first
        opt.step()
    with torch.no_grad():
        last = float(rast(m, torch.zeros_like(m), torch.sigmoid(lo), colors_precomp=colors, scales=scales,
                          rotations=rots)[6].mean())
    print(f"\n[depth distortion descent] distortion.mean() {first:.4e} -> {last:.4e} after 100 Adam steps")
    assert first > 0 and last <= 0.5 * first


if __name__ == "__main__":
    print(json.dumps(_rejections()))
