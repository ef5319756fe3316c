"""Orthographic views (sfgs_rasterize_forward_ortho / sfgs_rasterize_backward_ortho, sfgs.ortho).

The reference rasterizer has no orthographic camera; the oracle is tests/ortho_chain_f64.py, a float64 restatement of
the orthographic preprocess blended by the unchanged CPU oracle's blend, and tests/chain_f64.py's per-Gaussian adjoint
(ortho=True).

CPU: the restatement against float64 central differences, projection_matrix, nadir_camera, the C ABI's and the Python
layer's rejections and their order, and the native calls OrthoRasterizer makes.
GPU: the preprocess and the images against the restatement, the pinhole limit, the ten gradients against the
restatement's autograd and an end-to-end finite-difference check, the deterministic backward, offsets, a synthetic DSM
and a height-map fit."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import chain_f64 as CH
import helpers as Hh
import ortho_chain_f64 as OC
from sfgs import synthetic as S

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")


# ----------------------------------------------------------------------------- cameras and scenes
def ortho_view(dist=10.0, elevation=70.0, azimuth=30.0):
    """[4,4] float32 row-vector viewmatrix of a look-at camera at `dist` from the origin (an oblique view)."""
    cam = S.orbit_camera(elevation_deg=elevation, azimuth_deg=azimuth, radius=dist, width=64, height=64)
    return torch.from_numpy(np.ascontiguousarray(cam.viewmatrix))


def ortho_camera(W, H, s_x, s_y, cx=0.0, cy=0.0, **kw):
    from sfgs.ortho import projection_matrix
    view = ortho_view(**kw)
    proj = (view.double() @ projection_matrix(s_x, s_y, 0.01, 100.0, cx, cy).double()).float()
    return view, proj


def scene_tensors(P, seed, D, M, dev, spread=2.0, scale=0.12, colors=False):
    sc = S.blob_scene(P, seed=seed, sh_degree=3, spread=spread, scale=scale)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d = dict(means3D=t(sc.means3D), scales=t(sc.scales), rotations=t(sc.rotations), opacities=t(sc.opacities),
             shs=t(sc.shs[:, :M]).contiguous(), D=D)
    if colors:
        d["colors"] = t(np.random.default_rng(seed).uniform(0, 1, (P, 3)).astype(np.float32))
        d["shs"] = None
    return d


def _frame(d, view, proj, W, H, s_x, s_y):
    """The harness's Gaussians with the matrices, and its camera (the half-extents in place of tan_fov)."""
    dev = d["means3D"].device
    cam = types.SimpleNamespace(width=W, height=H, tanfovx=s_x, tanfovy=s_y)
    return dict(d, viewmatrix=view.to(dev), projmatrix=proj.to(dev), campos=torch.zeros(3, device=dev)), cam


def forward(d, view, proj, W, H, s_x, s_y, bg, ks=0.1, off=None):
    dd, cam = _frame(d, view, proj, W, H, s_x, s_y)
    return Hh.run_ours_forward(dd, cam, d["D"], bg, kernel_size=ks, colors=d.get("colors"), subpixel_offset=off,
                               ortho=True)


def backward(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ks=0.1, off=None, **kw):
    dd, cam = _frame(d, view, proj, W, H, s_x, s_y)
    return Hh.run_ours_backward(dd, cam, d["D"], bg, fwd, cot, kernel_size=ks, colors=d.get("colors"),
                                subpixel_offset=off, **kw)


def restatement(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, off=None):
    """chain_f64.chain(ortho=True) on this frame's phase-1 sums (the blend adjoint reads only the forward's records, so
    the pinhole phase-1 call gives them), with scales and rotations as leaves."""
    dd, cam = _frame(d, view, proj, W, H, s_x, s_y)
    a = Hh.restatement_inputs(fwd, dd, cam, d["D"], bg, cot, d.get("colors"), off, det=None)
    return CH.chain(**dict(a, cov3D=None), scales=d["scales"], rotations=d["rotations"], ortho=True)


def restated(d, view, proj, W, H, s_x, s_y, ks=0.1):
    return OC.preprocess(d["means3D"], d["scales"], d["rotations"], d["opacities"], view, proj, W, H, s_x, s_y, ks,
                         D=d["D"], shs=d.get("shs"), colors=d.get("colors"))


# ----------------------------------------------------------------------------- CPU: the restatement
def test_restatement_matches_central_differences():
    torch.manual_seed(0)
    P, W, H, s_x, s_y = 6, 64, 48, 3.0, 2.5
    view, proj = ortho_camera(W, H, s_x, s_y, cx=0.1, cy=-0.05)
    f = lambda *s: torch.randn(*s, dtype=torch.float64)  # noqa: E731
    x = dict(m=f(P, 3), s=f(P, 3).abs() * 0.2 + 0.05, q=f(P, 4), sh=f(P, 16, 3) * 0.3)
    w = f(P, 9)

    def loss(**kw):
        a = dict(x, **kw)
        return OC.scalar_outputs(a["m"], a["s"], a["q"], None, view, proj, W, H, s_x, s_y, 0.1, 3, a["sh"], w)

    leaves = {k: v.clone().requires_grad_(True) for k, v in x.items()}
    loss(**leaves).backward()
    for k, v in x.items():
        g = leaves[k].grad
        fd = torch.zeros_like(v)
        for i in range(v.numel()):
            e = torch.zeros_like(v).view(-1)
            e[i] = 1e-6
            e = e.view_as(v)
            fd.view(-1)[i] = (loss(**{k: v + e}) - loss(**{k: v - e})) / 2e-6
        assert torch.allclose(g, fd, rtol=1e-6, atol=1e-6 * float(fd.abs().max())), (k, (g - fd).abs().max())


def test_restatement_chain_matches_central_differences():
    """chain's means3D / scales / rotations / sh gradients are those of sum <acc, outputs> (the conic and Mip terms
    switched off, so that no kernel-local derivative enters)."""
    torch.manual_seed(1)
    P, W, H, s_x, s_y = 5, 64, 48, 3.0, 2.5
    view, proj = ortho_camera(W, H, s_x, s_y)
    f = lambda *s: torch.randn(*s, dtype=torch.float64)  # noqa: E731
    m, sc, q, sh = f(P, 3), f(P, 3).abs() * 0.2 + 0.05, f(P, 4), f(P, 16, 3) * 0.3
    acc = f(P, 16)
    acc[:, 10:16] = 0.0
    vis = torch.ones(P, dtype=torch.bool)
    clamped = torch.zeros(P, 3, dtype=torch.bool)
    pre = OC.preprocess(m, sc, q, torch.ones(P, 1), view, proj, W, H, s_x, s_y, 0.1, D=3, shs=sh)
    g = CH.chain(acc, vis, m, torch.ones(P), clamped, sh, 3, view, proj, None, W, H, s_x, s_y, 0.1, scales=sc,
                 rotations=q, norm_rec=pre["norm3D"] + 0 * m, ortho=True)
    d = OC.view_axis(view)

    def L(m_, sh_):
        gg = OC.project(m_, sc, q, view, proj, W, H, s_x, s_y, 0.1)
        rgb = OC.eval_sh(3, sh_, d.expand(P, 3))
        return float((acc[:, 7] * gg["ndc"][:, 0] + acc[:, 8] * gg["ndc"][:, 1] + acc[:, 3] * gg["t"][:, 2]
                      + (acc[:, 0:3] * rgb).sum(1)).sum())

    for name, v, gv in (("means3D", m, g["means3D"]), ("sh", sh, g["sh"])):
        fd = torch.zeros_like(v)
        for i in range(v.numel()):
            e = torch.zeros(v.numel(), dtype=v.dtype)
            e[i] = 1e-6
            e = e.view_as(v)
            fd.view(-1)[i] = (L(m + e, sh) - L(m - e, sh)) / 2e-6 if name == "means3D" else \
                (L(m, sh + e) - L(m, sh - e)) / 2e-6
        assert torch.allclose(gv, fd, rtol=1e-6, atol=1e-7), name


def test_projection_matrix_maps_the_box_to_ndc():
    from sfgs.ortho import projection_matrix
    s_x, s_y, zn, zf = 3.0, 1.5, 0.5, 20.0
    O = projection_matrix(s_x, s_y, zn, zf).double()
    corners = torch.tensor([[sx * s_x, sy * s_y, z, 1.0] for sx in (-1, 1) for sy in (-1, 1) for z in (zn, zf)],
                           dtype=torch.float64)
    p = corners @ O
    assert torch.allclose(p[:, 0].abs(), torch.ones(8, dtype=torch.float64))
    assert torch.allclose(p[:, 1].abs(), torch.ones(8, dtype=torch.float64))
    assert torch.equal(torch.sign(p[:, 0]), torch.sign(corners[:, 0]))
    assert torch.allclose(p[:, 2], torch.where(corners[:, 2] == zn, 0.0, 1.0).double(), atol=1e-6)
    assert torch.allclose(p[:, 3], torch.ones(8, dtype=torch.float64))
    # the principal point: the view axis lands at (cx, cy), the box moves with it
    Oc = projection_matrix(s_x, s_y, zn, zf, cx=0.25, cy=-0.1).double()
    c = torch.tensor([[0.0, 0.0, 3.0, 1.0], [s_x, -s_y, 3.0, 1.0]], dtype=torch.float64) @ Oc
    assert torch.allclose(c[0, :2], torch.tensor([0.25, -0.1], dtype=torch.float64), atol=1e-7)
    assert torch.allclose(c[1, :2], torch.tensor([1.25, -1.1], dtype=torch.float64), atol=1e-6)


def test_nadir_camera_geometry():
    from sfgs.ortho import nadir_camera
    cam = nadir_camera(-10.0, 30.0, 5.0, 25.0, 0.5, 50.0)
    assert (cam.image_width, cam.image_height) == (80, 40)
    assert (cam.half_width, cam.half_height) == (20.0, 10.0)
    V, Pm = cam.viewmatrix.double(), cam.projmatrix.double()
    # the view axis is world -z; t_z = z_top - z
    assert torch.allclose(OC.view_axis(V), torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64))
    rng = np.random.default_rng(0)
    i, j = rng.integers(0, 80, 20), rng.integers(0, 40, 20)
    z = rng.uniform(-5, 40, 20)
    m = torch.tensor(np.stack([-10.0 + (i + 0.5) * 0.5, 25.0 - (j + 0.5) * 0.5, z], 1))
    g = OC.project(m, torch.ones(20, 3, dtype=torch.float64), torch.tensor([[1.0, 0, 0, 0]] * 20, dtype=torch.float64),
                   V, Pm, 80, 40, 20.0, 10.0, 0.0)
    assert torch.allclose(g["pix"], torch.tensor(np.stack([i, j], 1), dtype=torch.float64), atol=1e-4)
    assert torch.allclose(g["t"][:, 2], torch.tensor(50.0 - z), atol=1e-5)
    # north up: +y runs toward row 0, +x toward the last column
    assert torch.allclose(V[:3, :3], torch.tensor([[1.0, 0, 0], [0, -1.0, 0], [0, 0, -1.0]], dtype=torch.float64))


def _fwd_args(P=8, W=32, H=32, s=(2.0, 2.0), band=(0, 0), peers=None, ED=0):
    from sfgs import native as N
    a = N.ForwardArgs()
    a.P, a.width, a.height, a.ED = P, W, H, ED
    a.tan_fovx, a.tan_fovy = s
    a.tile_row_begin, a.tile_row_end = band
    if peers is not None:
        a.out_peers, a.n_out_peers = C.cast(peers, C.POINTER(C.c_void_p)), 2
    return a


def _bwd_args(P=8, W=32, H=32, s=(2.0, 2.0), band=(0, 0), peers=None, phase=0, ED=0):
    from sfgs import native as N
    b = N.BackwardArgs()
    b.P, b.width, b.height, b.ED, b.phase = P, W, H, ED, phase
    b.tan_fovx, b.tan_fovy = s
    b.tile_row_begin, b.tile_row_end = band
    if peers is not None:
        b.acc_peers, b.n_peers, b.peer_slice = C.cast(peers, C.POINTER(C.c_void_p)), 2, 8
    return b


def test_abi_rejects_unsupported_combinations_in_order():
    """Every rejection happens before any CUDA work (no device here), in the documented order: tile-row bands,
    out_peers / acc_peers, phase, then the half-extents, then the pinhole entry's checks."""
    from sfgs import native as N
    L = N.lib()
    dummy = (C.c_float * 64)()
    peers = (C.c_void_p * 2)(C.cast(dummy, C.c_void_p), C.cast(dummy, C.c_void_p))
    off = C.cast(dummy, C.c_void_p)

    def fwd(a, o=None):
        return L.sfgs_rasterize_forward_ortho(C.byref(a) if a is not None else None, o), N.last_error()

    def bwd(b, o=None, det=0):
        return L.sfgs_rasterize_backward_ortho(C.byref(b) if b is not None else None, o, det), N.last_error()

    assert fwd(None) == (SFGS_E_BADARG, "forward_ortho: null args")
    # a band wins over out_peers, which wins over a bad extent, which wins over the pinhole checks (bad sizes)
    rc, msg = fwd(_fwd_args(W=0, s=(0.0, 1.0), band=(0, 2), peers=peers))
    assert rc == SFGS_E_UNSUPPORTED and msg.startswith("forward_ortho: tile-row bands"), msg
    rc, msg = fwd(_fwd_args(W=0, s=(0.0, 1.0), peers=peers))
    assert rc == SFGS_E_UNSUPPORTED and msg.startswith("forward_ortho: out_peers"), msg
    for s in ((0.0, 1.0), (1.0, -2.0), (float("nan"), 1.0), (1.0, float("inf"))):
        rc, msg = fwd(_fwd_args(W=0, s=s))
        assert rc == SFGS_E_BADARG and "half-extents" in msg, (s, msg)
    assert fwd(_fwd_args(W=0)) == (SFGS_E_BADARG, "forward_ortho: bad sizes")
    # the subpixel entry's checks come with offsets
    rc, msg = fwd(_fwd_args(ED=2), off)
    assert rc == SFGS_E_UNSUPPORTED and msg == "forward_ortho: extra_attrs are not supported with subpixel offsets"

    assert bwd(None) == (SFGS_E_BADARG, "backward_ortho: null args")
    rc, msg = bwd(_bwd_args(W=0, s=(0.0, 1.0), band=(0, 2), peers=peers, phase=1))
    assert rc == SFGS_E_UNSUPPORTED and msg.startswith("backward_ortho: phases 1 and 2"), msg
    rc, msg = bwd(_bwd_args(W=0, s=(0.0, 1.0), band=(0, 2), peers=peers))
    assert rc == SFGS_E_UNSUPPORTED and msg.startswith("backward_ortho: acc_peers"), msg
    rc, msg = bwd(_bwd_args(W=0, s=(0.0, 1.0), band=(0, 2)))
    assert rc == SFGS_E_UNSUPPORTED and msg.startswith("backward_ortho: tile-row bands"), msg
    rc, msg = bwd(_bwd_args(W=0, s=(1.0, 0.0)))
    assert rc == SFGS_E_BADARG and "half-extents" in msg, msg
    assert bwd(_bwd_args(W=0)) == (SFGS_E_BADARG, "backward_ortho: bad sizes")
    rc, msg = bwd(_bwd_args(ED=2), off)
    assert rc == SFGS_E_UNSUPPORTED and msg == "backward_ortho: extra_attrs are not supported with subpixel offsets"
    rc, msg = bwd(_bwd_args(ED=2), None, 1)
    assert rc == SFGS_E_UNSUPPORTED and msg == "backward_ortho: extra_attrs have no deterministic implementation"


def test_python_layer_rejects_before_native_calls(monkeypatch):
    from sfgs import native as N
    from sfgs import rasterizer as R

    def no_lib():
        raise AssertionError("a native call was made")
    monkeypatch.setattr(N, "lib", no_lib)
    e, m = torch.empty(0), torch.zeros(4, 3)
    fwd = [e, m, e, m, m, m, 1.0, e, e, e, 0, e, e, 1.0, 1.0, 0.1, 16, 16, e, 0, e, False, False]
    for kw, what in ((dict(graph=True, capacity_hint=10), "graph"), (dict(tile_rows=(0, 1)), "tile_rows"),
                     (dict(out_peers=[0, 0]), "out_peers")):
        with pytest.raises(N.SfgsError, match=what):
            R.rasterize_gaussians(*fwd, ortho=True, **kw)
    bwd = [e, m] + [e] * 27
    for kw, what in ((dict(graph=True), "graph"), (dict(tile_rows=(0, 1)), "tile_rows"),
                     (dict(acc_peers=[0, 0]), "acc_peers"), (dict(phase=2), "phase=2"),
                     (dict(camera_grad=True), "camera_grad"),
                     (dict(camera_grad=True, intrinsics_grad=True), "intrinsics_grad")):
        with pytest.raises(N.SfgsError, match=what):
            R.rasterize_gaussians_backward(*bwd, ortho=True, **kw)


def test_ortho_rasterizer_native_calls(monkeypatch):
    """OrthoRasterizer calls the rasterizer with ortho=True and the fused normalize, passes the half-extents where
    the pinhole path passes tan_fov, and hands the backward the forward's buffers, norm_raw and offsets."""
    from sfgs import ortho as O
    P, H, W = 10, 24, 32
    calls = []

    def fwd(*a, **kw):
        calls.append(("fwd", a[13], a[14], kw))
        return (7, torch.rand(3, H, W), torch.rand(1, H, W), torch.rand(3, H, W), torch.rand(1, H, W),
                torch.ones(P, dtype=torch.int32), torch.empty(0), torch.zeros(8, dtype=torch.uint8),
                torch.zeros(8, dtype=torch.uint8), torch.zeros(8, dtype=torch.uint8), torch.rand(3, H, W))

    def bwd(*a, **kw):
        calls.append(("bwd", a[12], a[13], a[24], kw))
        z = lambda *s: torch.full(s, 0.5)  # noqa: E731
        return (z(P, 3), z(P, 3), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 4, 3), z(P, 3), z(P, 4), torch.empty(0))
    monkeypatch.setattr(O.R, "rasterize_gaussians", fwd)
    monkeypatch.setattr(O.R, "rasterize_gaussians_backward", bwd)
    monkeypatch.setattr(O.R, "check_subpixel_offset", lambda *a: None)
    off = torch.zeros(H, W, 2)
    rs = O.OrthoRasterizationSettings(H, W, 2.5, 1.5, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 1, False,
                                      False, off)
    means = torch.zeros(P, 3, requires_grad=True)
    means2D = torch.zeros(P, 3, requires_grad=True)
    out = O.OrthoRasterizer(rs)(means, means2D, torch.ones(P, 1), shs=torch.zeros(P, 4, 3), scales=torch.ones(P, 3),
                                rotations=torch.ones(P, 4))
    assert len(out) == 6
    (out[0].sum() + out[2].sum()).backward()
    assert [c[0] for c in calls] == ["fwd", "bwd"]
    assert calls[0][1:3] == (2.5, 1.5) and calls[0][3]["ortho"] and calls[0][3]["fuse_normalize"]
    assert calls[0][3]["subpixel_offset"] is off
    assert calls[1][1:4] == (2.5, 1.5, 7)
    kw = calls[1][4]
    assert kw["ortho"] and kw["subpixel_offset"] is off and kw["norm_raw"] is not None
    assert means.grad is not None and means2D.grad is not None
    # camera gradients are not formed: a camera that requires grad raises instead of dropping them
    bad = rs._replace(viewmatrix=torch.eye(4, requires_grad=True))
    with pytest.raises(ValueError, match="camera gradients"):
        O.OrthoRasterizer(bad)(means, means2D, torch.ones(P, 1), shs=torch.zeros(P, 4, 3), scales=torch.ones(P, 3),
                               rotations=torch.ones(P, 4))
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        O.OrthoRasterizer(rs)(means, means2D, torch.ones(P, 1), scales=torch.ones(P, 3), rotations=torch.ones(P, 4))


# ----------------------------------------------------------------------------- GPU
PRE_CASES = [(0, 0, 4), (1, 1, 4), (2, 2, 16), (3, 3, 16), (4, 3, 16), (5, -1, 16)]   # (seed, D, M); D = -1: colours


def _close(a, b, rtol, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    atol = rtol * float(b.abs().max()) if b.numel() else 0.0
    err = (a - b).abs() - rtol * b.abs()
    assert float(err.max()) <= atol, (what, float(err.max()), atol)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PRE_CASES)
def test_preprocess_against_restatement(cuda_device, case):
    seed, D, M = case
    W, H, s_x, s_y = 320, 240, 4.0, 3.0
    view, proj = ortho_camera(W, H, s_x, s_y, cx=0.03, cy=-0.02, azimuth=30.0 + 40 * seed)
    d = scene_tensors(6000, seed, max(D, 0), M, cuda_device, colors=D < 0)
    bg = torch.tensor([0.1, 0.2, 0.3], device=cuda_device)
    fwd = forward(d, view, proj, W, H, s_x, s_y, bg)
    I = Hh.our_internals(fwd, 6000, H, W)
    ref = restated(d, view, proj, W, H, s_x, s_y)
    near = OC.near_integer(ref["lam3"]) & ref["visible"]
    radii, tiles = fwd["radii"].cpu().long(), I["tiles_touched"].cpu().long()
    keep = ~near
    print(f"\n[ortho preprocess] case {case}: {int(ref['visible'].sum())} visible, {int(near.sum())} within 1e-4 of an "
          f"integer radius")
    assert torch.equal(radii[keep], ref["radii"][keep])
    assert torch.equal(tiles[keep], ref["tiles_touched"][keep])
    v = (radii > 0) & ref["visible"]
    assert int(v.sum()) > 500
    _close(I["means2D"].cpu()[v], ref["pix"][v], 1e-5, "centre")
    _close(I["conic_opacity"].cpu()[v, 0:3], ref["conic"][v], 1e-5, "conic")
    _close(I["conic_opacity"].cpu()[v, 3], ref["opacity"][v], 1e-5, "opacity")
    _close(I["depths"].cpu()[v], ref["depth"][v], 1e-5, "depth")
    _close(I["rgb"].cpu()[v], ref["rgb"][v], 1e-5, "colour")
    _close(I["norm3D"].cpu()[v], ref["norm3D"][v], 1e-5, "normal")


def _image_case(dev, seed, off=None, W=96, H=80):
    s_x, s_y = 3.0, 2.5
    view, proj = ortho_camera(W, H, s_x, s_y, cx=0.02, azimuth=20.0 + 50 * seed)
    d = scene_tensors(400, seed, 3, 16, dev, spread=1.5, scale=0.1)
    bg = torch.tensor([0.3, 0.1, 0.2], device=dev)
    return d, view, proj, W, H, s_x, s_y, bg


def _image_close(fwd, ref, what):
    for k in ("color", "alpha", "norm"):
        err = float(np.abs(fwd[k].detach().cpu().numpy() - ref[k]).max())
        assert err <= 1e-5, (what, k, err)
    dmax = max(1.0, float(np.abs(ref["depth"]).max()))
    err = float(np.abs(fwd["depth"].detach().cpu().numpy() - ref["depth"]).max())
    assert err <= 1e-5 * dmax, (what, "depth", err, dmax)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_images_against_restatement(cuda_device, seed):
    d, view, proj, W, H, s_x, s_y, bg = _image_case(cuda_device, seed)
    fwd = forward(d, view, proj, W, H, s_x, s_y, bg)
    ref = OC.render(restated(d, view, proj, W, H, s_x, s_y), W, H, bg.cpu().numpy())
    assert float(fwd["alpha"].max()) > 0.5
    _image_close(fwd, ref, seed)


@pytest.mark.gpu
def test_pinhole_limit(cuda_device):
    """A pinhole camera at distance d on the same axis with tan = s / d converges to the orthographic view."""
    dev = cuda_device
    W = H = 128
    s = 3.0
    D0 = 10.0
    d = scene_tensors(2000, 7, 2, 16, dev, spread=1.0, scale=0.05)
    extent = float(d["means3D"].abs().max())
    view, proj = ortho_camera(W, H, s, s, dist=D0)
    bg = torch.tensor([0.2, 0.2, 0.2], device=dev)
    ortho = forward(d, view, proj, W, H, s, s, bg)
    from sfgs import rasterizer as R
    diffs = []
    for dist in (100.0 * extent, 1000.0 * extent):
        V = view.double().clone()
        V[3, 2] += dist - D0                                 # the camera centre moves back along the view axis
        fov = 2.0 * math.atan(s / dist)
        Pp = torch.from_numpy(S._projection(0.01, 10.0 * dist, fov, fov).T.astype(np.float64))
        full = (V @ Pp).float()
        campos = torch.linalg.inv(V)[3, :3].float()
        e = torch.empty(0, device=dev)
        out = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                    V.float().to(dev), full.to(dev), s / dist, s / dist, 0.1, H, W, d["shs"], d["D"],
                                    campos.to(dev), False, False)
        diffs.append(float((out[1] - ortho["color"]).abs().max()))
    print(f"\n[ortho pinhole limit] max |colour difference| at d = 100, 1000 x extent: {diffs}")
    assert diffs[1] * 5.0 <= diffs[0], diffs


def _grad_check(ours, ref, what):
    for k in GRAD_KEYS:
        if k not in ref:
            continue
        a, b = ours[k].detach().double().cpu().reshape(ref[k].shape), ref[k].double().cpu()
        atol = 1e-4 * float(b.abs().max()) + 1e-7
        err = float(((a - b).abs() - 1e-3 * b.abs()).max())
        assert err <= atol, (what, k, err, atol)


def _gradient_case(dev, seed, colors=False):
    d, view, proj, W, H, s_x, s_y, bg = _image_case(dev, seed)
    if colors:
        d["colors"] = torch.rand(400, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))
        d["shs"] = None
    fwd = forward(d, view, proj, W, H, s_x, s_y, bg)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=seed + 3)]
    ref = restatement(d, view, proj, W, H, s_x, s_y, bg, fwd, cot)
    return d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ref


@pytest.mark.gpu
@pytest.mark.parametrize("seed,colors", [(0, False), (1, False), (2, True)])
def test_gradients_against_restatement(cuda_device, seed, colors):
    d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ref = _gradient_case(cuda_device, seed, colors)
    g = backward(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ortho=True)
    _grad_check(g, ref, (seed, colors))
    assert g["extra"].numel() == 0


@pytest.mark.gpu
def test_end_to_end_finite_differences(cuda_device):
    """OrthoRasterizer's gradients of a weighted image sum against central differences of the GPU forward, for the
    means, scales and opacities of a tiny scene.  The splats are wide and faint: every pixel of the image lies well
    inside every splat's 1/255 contour and tile rectangle, so the rendered images are smooth in the parameters (a pixel
    crossing the 1/255 cut is a jump the analytic gradient does not see, as in the reference)."""
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer
    dev = cuda_device
    W = H = 48
    s = 2.0
    view, proj = ortho_camera(W, H, s, s, dist=6.0)
    rs = OrthoRasterizationSettings(H, W, s, s, 0.1, torch.zeros(3, device=dev), 1.0, view.to(dev), proj.to(dev), 0,
                                    False, False)
    g = torch.Generator().manual_seed(3)
    means = (torch.rand(3, 3, generator=g) - 0.5).to(dev)
    scales = torch.tensor([[2.5, 2.0, 1.5], [2.0, 2.4, 1.8], [2.2, 1.6, 2.6]], device=dev)
    rots = torch.nn.functional.normalize(torch.randn(3, 4, generator=g), dim=1).to(dev)
    opac = torch.tensor([[0.25], [0.3], [0.2]], device=dev)
    colors = torch.rand(3, 3, generator=g).to(dev)
    wc = torch.rand(3, H, W, generator=g).to(dev)
    wd = torch.rand(1, H, W, generator=g).to(dev)

    def loss(m, o, sc):
        out = OrthoRasterizer(rs)(m, torch.zeros_like(m), o, colors_precomp=colors, scales=sc, rotations=rots)
        return (out[0] * wc).double().sum() + (out[1] * wd).double().sum() * 0.1 + out[3].double().sum()

    x0 = dict(m=means, o=opac, sc=scales)
    leaves = {k: v.clone().requires_grad_(True) for k, v in x0.items()}
    with torch.no_grad():
        assert float(OrthoRasterizer(rs)(means, torch.zeros_like(means), opac, colors_precomp=colors, scales=scales,
                                         rotations=rots)[3].min()) > 0.2
    loss(**leaves).backward()
    eps = 1e-2
    for k, x in x0.items():
        fd = torch.zeros_like(x)
        for i in range(x.numel()):
            e = torch.zeros(x.numel(), device=dev)
            e[i] = eps
            e = e.view_as(x)
            with torch.no_grad():
                fd.view(-1)[i] = float((loss(**dict(x0, **{k: x + e})) - loss(**dict(x0, **{k: x - e}))) / (2 * eps))
        gx = leaves[k].grad
        err = float((gx - fd).abs().max())
        assert err <= 0.01 * float(fd.abs().max()) + 1e-3, (k, err, gx, fd)


@pytest.mark.gpu
def test_deterministic_backward(cuda_device):
    d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ref = _gradient_case(cuda_device, 4)
    default = backward(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ortho=True)
    with Hh.deterministic():
        g1 = backward(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ortho=True)
        g2 = backward(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, ortho=True)
    for k in GRAD_KEYS:
        assert torch.equal(g1[k].view(torch.int32), g2[k].view(torch.int32)), k
    _grad_check(default, ref, "default")
    _grad_check(g1, ref, "deterministic")


@pytest.mark.gpu
@pytest.mark.parametrize("ox,oy", [(1, 0), (0, -1), (2, -3)])
def test_integer_offsets_reproduce_shifted_renders(cuda_device, ox, oy):
    dev = cuda_device
    d, view, proj, W, H, s_x, s_y, bg = _image_case(dev, 5)
    off = torch.empty((H, W, 2), device=dev)
    off[..., 0], off[..., 1] = float(ox), float(oy)
    f0 = forward(d, view, proj, W, H, s_x, s_y, bg)
    f1 = forward(d, view, proj, W, H, s_x, s_y, bg, off=off)
    assert torch.equal(f0["radii"], f1["radii"])
    y, x = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    sx, sy = x + ox, y + oy
    ok = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H) & (sx // 16 == x // 16) & (sy // 16 == y // 16)
    src = (sy.clamp(0, H - 1) * W + sx.clamp(0, W - 1))[ok]
    for k in ("color", "depth", "norm", "alpha"):
        a = f1[k].reshape(f1[k].shape[0], -1)[:, ok.flatten()]
        b = f0[k].reshape(f0[k].shape[0], -1)[:, src]
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (k, ox, oy)


@pytest.mark.gpu
def test_fractional_offsets_against_restatement(cuda_device):
    dev = cuda_device
    d, view, proj, W, H, s_x, s_y, bg = _image_case(dev, 6)
    off = (torch.rand((H, W, 2), generator=torch.Generator().manual_seed(6)) - 0.5).to(dev)
    fwd = forward(d, view, proj, W, H, s_x, s_y, bg, off=off)
    ref = OC.render(restated(d, view, proj, W, H, s_x, s_y), W, H, bg.cpu().numpy(), subpixel_offset=off.cpu().numpy())
    _image_close(fwd, ref, "offsets")
    # the backward takes the same offsets: its gradients match the restatement's chain for the offset frame's sums
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=9)]
    ref_g = restatement(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, off)
    _grad_check(backward(d, view, proj, W, H, s_x, s_y, bg, fwd, cot, off=off, ortho=True), ref_g, "offsets")


def stepped_surfels(dev, spacing=0.25, roofs=((-20, -4, -20, 4, 8.0), (6, 22, -12, 12, 20.0)), extent=32.0):
    """Opaque flat surfels tiling a stepped height field over [-extent, extent]^2: ground at z = 0 and box roofs
    (x0, x1, y0, y1, height).  Returns the tensors and a function z(x, y) of the true height."""
    xs = torch.arange(-extent + spacing / 2, extent, spacing)
    X, Y = torch.meshgrid(xs, xs, indexing="ij")
    X, Y = X.flatten(), Y.flatten()

    def height(x, y):
        z = torch.zeros_like(x)
        for x0, x1, y0, y1, h in roofs:
            z = torch.where((x >= x0) & (x < x1) & (y >= y0) & (y < y1), torch.full_like(z, h), z)
        return z
    Z = height(X, Y)
    P = X.numel()
    means = torch.stack([X, Y, Z], 1).to(dev)
    scales = torch.tensor([spacing * 0.7, spacing * 0.7, 1e-3]).expand(P, 3).contiguous().to(dev)
    rots = torch.tensor([1.0, 0.0, 0.0, 0.0]).expand(P, 4).contiguous().to(dev)
    opac = torch.full((P, 1), 0.99, device=dev)
    roof = (Z > 0).to(dev)
    return means, scales, rots, opac, height, roof


def _interior(height, cam, margin=1.0):
    """Pixels whose true height is constant within `margin` world units (away from the roof edges), and that height."""
    r = cam.resolution
    xs = cam.xmin + (torch.arange(cam.image_width) + 0.5) * r
    ys = cam.ymax - (torch.arange(cam.image_height) + 0.5) * r
    Y, X = torch.meshgrid(ys, xs, indexing="ij")
    z = height(X, Y)
    same = torch.ones_like(z, dtype=torch.bool)
    # the corners of the square of half-width `margin` (the boxes are wider than it, so no box corner hides inside)
    for dx, dy in ((margin, margin), (-margin, margin), (margin, -margin), (-margin, -margin)):
        same &= height(X + dx, Y + dy) == z
    return same, z


@pytest.mark.gpu
def test_dsm_of_a_stepped_height_field(cuda_device):
    from sfgs.ortho import nadir_camera, render_height_map
    means, scales, rots, opac, height, _ = stepped_surfels(cuda_device)
    cam = nadir_camera(-30.0, 30.0, -30.0, 30.0, 60.0 / 1024, 50.0)
    assert (cam.image_width, cam.image_height) == (1024, 1024)
    with torch.no_grad():
        dsm = render_height_map(cam, means, opac, scales, rots).cpu()
    inside, z = _interior(height, cam)
    err = (dsm - z)[inside].abs()
    print(f"\n[ortho DSM] 1024^2, {int(inside.sum())} interior pixels: max |height error| {float(err.max()):.2e}, "
          f"mean {float(err.mean()):.2e}")
    assert torch.isfinite(dsm[inside]).all()
    assert float(err.max()) <= 0.05


@pytest.mark.gpu
def test_height_map_fit(cuda_device):
    """Raise the roofs by 3; 200 Adam steps on an L1 against the true height map bring them back."""
    from sfgs.ortho import nadir_camera, render_height_map
    dev = cuda_device
    means, scales, rots, opac, height, roof = stepped_surfels(dev, spacing=0.5)
    cam = nadir_camera(-30.0, 30.0, -30.0, 30.0, 60.0 / 256, 50.0)
    with torch.no_grad():
        target = render_height_map(cam, means, opac, scales, rots)
    z0 = means[:, 2].clone()
    start = means.clone()
    start[roof, 2] += 3.0
    z = start[:, 2].clone().requires_grad_(True)
    opt = torch.optim.Adam([z], lr=0.05)
    xy = means[:, :2]

    def mean_err():
        return float((z.detach() - z0)[roof].abs().mean())
    e0 = mean_err()
    for _ in range(200):
        opt.zero_grad()
        hm = render_height_map(cam, torch.cat([xy, z[:, None]], 1), opac, scales, rots)
        ok = torch.isfinite(hm) & torch.isfinite(target)
        loss = (hm[ok] - target[ok]).abs().mean()
        loss.backward()
        opt.step()
    e1 = mean_err()
    print(f"\n[ortho fit] mean roof height error {e0:.3f} -> {e1:.4f} after 200 Adam steps")
    assert e1 * 10.0 <= e0, (e0, e1)
