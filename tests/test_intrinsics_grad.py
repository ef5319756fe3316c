"""Focal-length gradients (sfgs_rasterize_backward_camera_intrinsics): dL/dtan_fovx and dL/dtan_fovy, after the 35
camera gradients.  The oracle is tests/chain_f64.py, the camera restatement with tan_fov as leaves (focal=True).

CPU: the restatement against the camera restatement (bit for bit) and against finite differences (including clamped
Gaussians), the C ABI's argument checks, and the autograd layer's native calls.
GPU: every other output bit-identical to the camera entry, accuracy against the float64 restatement, reproducibility,
and focal / principal-point refinement end to end through diff_gauss."""
import ctypes as C

import numpy as np
import pytest
import torch

import chain_f64 as CH
import golden_cases as G
import helpers as Hh
from helpers import release_cached_frames  # noqa: F401
from sfgs import synthetic as S

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot", "extra")
CAM_KEYS = ("view", "proj", "campos")


# ----------------------------------------------------------------------------- CPU: the restatement
def _oracle_args(name):
    """The restatement's arguments for a golden case: the CPU oracle's forward and its blend adjoint's sums."""
    from oracle import cpu_oracle as O
    scene, cam, bg, kw = G.build_case(name)
    colors = kw.get("colors")
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, kw["sh_degree"],
                  cam.viewmatrix, cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg,
                  kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"], colors_precomp=colors)
    s = O.blend_backward(o, *kw["cot"])
    acc = CH.acc_from_screen_grads(s["means2D"], s["colors"], s["depths"], s["norm3D"], s["conic"], s["opacity"])
    return dict(acc=acc, radii=o["radii"], means3D=scene.means3D, cov3D=o["cov3D"],
                combined_opacity=o["conic_opacity"][:, 3], clamped=o["clamped"] != 0,
                shs=None if colors is not None else scene.shs, D=kw["sh_degree"], viewmatrix=cam.viewmatrix,
                projmatrix=cam.projmatrix, campos=cam.campos, W=cam.width, H=cam.height, tan_fovx=cam.tanfovx,
                tan_fovy=cam.tanfovy, kernel_size=kw["kernel_size"])


@pytest.mark.parametrize("name", G.CASES)
def test_restatement_extends_the_camera_restatement_bit_for_bit(name):
    a = _oracle_args(name)
    r = CH.chain(**a, focal=True)
    c = CH.chain(**a)
    for k in ("means3D", "view", "proj", "campos"):
        assert torch.equal(r[k], c[k]), (name, k)
    assert torch.equal(r["abs"][:35], c["abs"]), name
    assert r["tanx"] != 0 and r["tany"] != 0, name


def _away_from_kinks(a, scale):
    """tan_fov scale factors near `scale` at which every rasterized Gaussian's |t/t_z| is more than 1e-3 (relative)
    from the clamp bound 1.3 tan_fov."""
    for k in range(200):
        s = scale * (1.0 + 1.7e-3 * k)
        r = CH.chain(**dict(a, tan_fovx=a["tan_fovx"] * s, tan_fovy=a["tan_fovy"] * s), focal=True, exact=True)
        if (torch.cat([r["txtz_lim"], r["tytz_lim"]]) - 1).abs().min() > 1e-3:
            return s, r
    raise AssertionError("no tan_fov scale away from the clamp kinks")


@pytest.mark.parametrize("name", G.CASES)
@pytest.mark.parametrize("scale", [1.0, 0.55])
def test_restatement_matches_finite_differences(name, scale):
    """dL/dtan_fov of the restatement against central differences of the same loss, in float64.  At scale 0.55 the
    field of view is narrowed around the frame's Gaussians, so that many of them lie beyond the clamp bound."""
    a = _oracle_args(name)
    s, r = _away_from_kinks(a, scale)
    tx0, ty0 = a["tan_fovx"] * s, a["tan_fovy"] * s
    clamp_term = []
    if scale < 1.0:
        assert r["n_clamped"] > 0, name
    for key, which in (("tanx", "tan_fovx"), ("tany", "tan_fovy")):
        t0 = tx0 if which == "tan_fovx" else ty0
        h = 1e-6 * t0
        Lg = []
        for sgn in (1.0, -1.0):
            kw = dict(a, tan_fovx=tx0, tan_fovy=ty0)
            kw[which] = t0 + sgn * h
            Lg.append(CH.chain(**kw, focal=True, exact=True, coef=r["coef"])["Lg"])
        fd = float((Lg[0] - Lg[1]).sum()) / (2 * h)
        ad = float(r[key])
        scale_abs = float(r["abs"][35 if key == "tanx" else 36])
        assert abs(fd - ad) <= 1e-6 * scale_abs, (name, scale, key, fd, ad, scale_abs)
        assert abs(fd - ad) <= 1e-5 * abs(ad), (name, scale, key, fd, ad)
        if scale < 1.0:
            # the clamp term matters: without it the gradient misses the finite differences by far more than the
            # tolerance above
            held = CH.chain(**dict(a, tan_fovx=tx0, tan_fovy=ty0), focal=True, exact=True, coef=r["coef"],
                            hold_bound=True)
            clamp_term.append(abs(fd - float(held[key])) / scale_abs)
    if scale < 1.0:
        assert max(clamp_term) > 1e-5, (name, clamp_term)


# ----------------------------------------------------------------------------- CPU: argument checks
def test_abi_rejects_unsupported_combinations_before_cuda_work():
    from sfgs import native as N
    L = N.lib()
    dummy = (C.c_float * 64)()
    ptr = C.cast(dummy, C.c_void_p)
    out = ptr

    def args(**kw):
        b = N.BackwardArgs()
        b.P, b.width, b.height = 8, 32, 32
        b.scratch_alloc = N.ALLOC_FN(lambda _u, _n: None)
        for k, v in kw.items():
            setattr(b, k, v)
        return b
    cases = [
        (args(), None, 0, None, SFGS_E_BADARG, "dL_dcamera"),
        (args(phase=1, acc=ptr), None, 0, out, SFGS_E_UNSUPPORTED, "phase 0"),
        (args(phase=2, acc=ptr, gauss_begin=0, gauss_end=8), None, 0, out, SFGS_E_UNSUPPORTED, "phase 0"),
        (args(ED=2), ptr, 0, out, SFGS_E_UNSUPPORTED, "extra_attrs"),
        (args(ED=2), None, 1, out, SFGS_E_UNSUPPORTED, "extra_attrs"),
        (args(ED=2), ptr, 1, out, SFGS_E_UNSUPPORTED, "extra_attrs"),
    ]
    peers = (C.c_void_p * 1)(ptr)
    pa = args(acc=ptr, n_peers=1, peer_slice=8)
    pa.acc_peers = C.cast(peers, C.POINTER(C.c_void_p))
    cases.append((pa, None, 0, out, SFGS_E_UNSUPPORTED, "acc_peers"))
    nalloc = args()
    nalloc.scratch_alloc = N.ALLOC_FN()
    cases.append((nalloc, None, 0, out, SFGS_E_BADARG, "scratch"))
    for b, off, det, dst, code, what in cases:
        assert L.sfgs_rasterize_backward_camera_intrinsics(C.byref(b), off, det, dst) == code, what
        assert what in N.last_error(), (what, N.last_error())
        if code == SFGS_E_BADARG or what in ("phase 0", "acc_peers"):
            assert "backward_camera_intrinsics" in N.last_error(), N.last_error()
    assert L.sfgs_rasterize_backward_camera_intrinsics(None, None, 0, out) == SFGS_E_BADARG


def test_python_backward_rejects_intrinsics_without_camera_grad():
    from sfgs import rasterizer as R
    e = torch.empty(0)
    with pytest.raises(ValueError, match="camera_grad"):
        R.rasterize_gaussians_backward(*([e] * 29), camera_grad=False, intrinsics_grad=True)


# ----------------------------------------------------------------------------- CPU: the autograd layer's native calls
def _recording_layer(monkeypatch, P, H, W):
    import diff_gauss
    from diff_gauss import _C
    calls = []

    def fwd(*a, fuse_normalize=False, subpixel_offset=None):
        calls.append(("fwd", a[13], a[14]))
        r = (torch.ones(P, dtype=torch.int32),)
        out = (7, torch.rand(3, H, W), torch.rand(1, H, W), torch.rand(3, H, W), torch.rand(1, H, W)) + r + (
            torch.empty(0), torch.zeros(8, dtype=torch.uint8), torch.zeros(8, dtype=torch.uint8),
            torch.zeros(8, dtype=torch.uint8))
        return out + (torch.rand(3, H, W),) if fuse_normalize else out

    def bwd(*a, norm_raw=None, **kw):
        calls.append(("bwd", a[12], a[13], tuple(sorted(kw))))
        z = lambda *s: torch.full(s, 0.5)  # noqa: E731
        out = (z(P, 3), z(P, 3), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 16, 3), z(P, 3), z(P, 4), torch.empty(0))
        if kw.get("camera_grad"):
            out += (z(4, 4), 2 * z(4, 4), 3 * z(3))
        if kw.get("intrinsics_grad"):
            out += (torch.tensor(5.0), torch.tensor(7.0))
        return out
    monkeypatch.setattr(_C, "rasterize_gaussians", fwd)
    monkeypatch.setattr(_C, "rasterize_gaussians_fused", lambda *a, **kw: fwd(*a, fuse_normalize=True, **kw))
    monkeypatch.setattr(_C, "rasterize_gaussians_backward", bwd)
    monkeypatch.setattr(_C, "rasterize_gaussians_backward_fused", bwd)
    return diff_gauss, calls


def _run(diff_gauss, P, H, W, tanx, tany, view_grad=False):
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    view = torch.eye(4).requires_grad_(view_grad)
    rs = GaussianRasterizationSettings(H, W, tanx, tany, 0.1, torch.zeros(1), torch.zeros(3), 1.0, view, torch.eye(4),
                                       3, torch.zeros(3), False, False)
    means = torch.zeros(P, 3, requires_grad=True)
    out = GaussianRasterizer(rs)(means, torch.zeros(P, 3, requires_grad=True), torch.ones(P, 1),
                                 shs=torch.zeros(P, 16, 3), scales=torch.ones(P, 3), rotations=torch.ones(P, 4))
    out[0].sum().backward()
    return view.grad, means.grad


@pytest.mark.parametrize("fuse", [True, False])
def test_autograd_layer_keeps_the_native_calls_without_focal_grad(monkeypatch, fuse):
    """Float tan_fov, and tensors that do not require grad, reach the native layer as before: the same objects, and a
    backward without camera_grad / intrinsics_grad (or with camera_grad only, for a camera that requires grad)."""
    P, H, W = 50, 24, 32
    diff_gauss, calls = _recording_layer(monkeypatch, P, H, W)
    monkeypatch.setattr(diff_gauss, "FUSE_NORMALIZE", fuse)
    tx_t, ty_t = torch.tensor(0.5), torch.tensor(0.4, dtype=torch.float64)
    for tanx, tany in ((0.5, 0.4), (tx_t, ty_t), (tx_t, 0.4)):
        for view_grad in (False, True):
            calls.clear()
            gv, gm = _run(diff_gauss, P, H, W, tanx, tany, view_grad)
            assert [c[0] for c in calls] == ["fwd", "bwd"]
            assert calls[0][1] is tanx and calls[0][2] is tany
            assert calls[1][1] is tanx and calls[1][2] is tany
            assert calls[1][3] == (("camera_grad",) if view_grad else ()), calls[1]
            assert gm is not None and (gv is not None) == view_grad


@pytest.mark.parametrize("fuse", [True, False])
def test_autograd_layer_calls_the_intrinsics_entry_for_focal_leaves(monkeypatch, fuse):
    P, H, W = 50, 24, 32
    diff_gauss, calls = _recording_layer(monkeypatch, P, H, W)
    monkeypatch.setattr(diff_gauss, "FUSE_NORMALIZE", fuse)
    # both leaves, float32 and float64
    tx = torch.tensor(0.5, requires_grad=True)
    ty = torch.tensor(0.4, dtype=torch.float64, requires_grad=True)
    calls.clear()
    gv, gm = _run(diff_gauss, P, H, W, tx, ty)
    bwd = [c for c in calls if c[0] == "bwd"]
    assert len(bwd) == 1 and bwd[0][3] == ("camera_grad", "intrinsics_grad"), bwd
    assert gv is None and gm is not None
    assert tx.grad.shape == () and tx.grad.dtype == torch.float32 and float(tx.grad) == 5.0
    assert ty.grad.shape == () and ty.grad.dtype == torch.float64 and float(ty.grad) == 7.0
    assert tx.grad.device == tx.device and ty.grad.device == ty.device
    # one leaf: a gradient for it alone; the camera gets its gradient from the same call
    ty2 = torch.tensor(0.4, requires_grad=True)
    calls.clear()
    gv, _ = _run(diff_gauss, P, H, W, 0.5, ty2, view_grad=True)
    assert [c[3] for c in calls if c[0] == "bwd"] == [("camera_grad", "intrinsics_grad")]
    assert float(ty2.grad) == 7.0 and torch.equal(gv, torch.full((4, 4), 0.5))
    # the FoV through torch.tan, as a focal refinement writes it
    fov = torch.tensor(0.9, dtype=torch.float64, requires_grad=True)
    _run(diff_gauss, P, H, W, torch.tan(fov * 0.5), torch.tan(fov * 0.4))
    expect = 5.0 * 0.5 / np.cos(0.45) ** 2 + 7.0 * 0.4 / np.cos(0.36) ** 2
    assert abs(float(fov.grad) - expect) <= 1e-12 * expect


# ----------------------------------------------------------------------------- GPU helpers
def _setup(name, dev, jitter, seed=6):
    scene, cam, D, d, colors = Hh.frame(name, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, 23) if jitter else None
    f = Hh.run_ours_forward(d, cam, D, bg, colors=colors, subpixel_offset=off)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=seed)]
    return scene, cam, D, d, colors, bg, off, f, cot


# ----------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["jax004", "orbit", "m4", "precomp"])
def test_other_outputs_and_camera_terms_unchanged(cuda_device, name):
    """The ten gradient tensors and the 35 camera terms of the intrinsics entry are bit-identical to the camera
    entry's, with and without offsets (deterministic calls: the default calls reduce with unordered atomics)."""
    dev = cuda_device
    for jitter in (False, True):
        scene, cam, D, d, colors, bg, off, f, cot = _setup(name, dev, jitter)
        a = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True, camera_grad=True)
        b = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True, camera_grad=True,
                                 intrinsics_grad=True)
        for k in GRAD_KEYS + CAM_KEYS:
            assert a[k].shape == b[k].shape, (name, jitter, k)
            assert torch.equal(Hh.bits(a[k]), Hh.bits(b[k])), (name, jitter, k)
        assert b["tanx"].shape == () and b["tany"].shape == ()
        assert bool(torch.isfinite(b["tanx"])) and bool(torch.isfinite(b["tany"]))
        # the default call forms the same focal terms from the same kernel
        gc = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, camera_grad=True,
                                  intrinsics_grad=True)
        assert bool(torch.isfinite(gc["tanx"])) and bool(torch.isfinite(gc["tany"]))


def _accuracy_case(case, dev):
    """GPU focal gradients of a deterministic call and the restatement (float64 and float32) evaluated on the phase-1
    sums of a deterministic run: the same `acc` bits the call uses."""
    def make():
        name = {"d3": "jax004", "d1": "m4", "precomp": "precomp", "clamp": "clamp"}[case.split("_")[0]]
        scene, cam, D, d, colors, bg, off, f, cot = _setup(name, dev, case.endswith("jitter"))
        g = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True, camera_grad=True,
                                 intrinsics_grad=True)
        a = Hh.restatement_inputs(f, d, cam, D, bg, cot, colors, off)
        r64 = CH.chain(**a, focal=True, dtype=torch.float64)
        r32 = CH.chain(**a, focal=True, dtype=torch.float32)
        return g, r64, r32
    return Hh.cached("case", case, make)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["d3", "d3_jitter", "d1", "d1_jitter", "precomp", "precomp_jitter", "clamp"])
def test_accuracy_against_float64(cuda_device, case):
    """The bound test_camera_grad.py applies to the 35 camera terms: twice the float32 restatement's error, or 1e-6 of
    the sum of the terms' magnitudes."""
    g, r64, r32 = _accuracy_case(case, cuda_device)
    if case == "clamp":
        assert r64["n_clamped"] > 0
    gpu = torch.stack([g["tanx"], g["tany"]]).double()
    f64 = torch.stack([r64["tanx"], r64["tany"]]).double()
    f32 = torch.stack([r32["tanx"], r32["tany"]]).double()
    tol = torch.maximum(2.0 * (f32 - f64).abs(), 1e-6 * r64["abs"][35:37].double())
    err = (gpu - f64).abs()
    print(f"\n[focal {case}] gpu {gpu.tolist()} f64 {f64.tolist()} max err / tol "
          f"{float((err / tol.clamp_min(1e-300)).max()):.3f} clamped {r64['n_clamped']}")
    assert (err <= tol).all(), (case, err, tol)


@pytest.mark.gpu
def test_deterministic_focal_gradients_are_reproducible(cuda_device):
    dev = cuda_device
    for jitter in (False, True):
        scene, cam, D, d, colors, bg, off, f, cot = _setup("jax004", dev, jitter)
        runs = [Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True,
                                     camera_grad=True, intrinsics_grad=True) for _ in range(3)]
        for k in CAM_KEYS + ("tanx", "tany"):
            for r in runs[1:]:
                assert torch.equal(Hh.bits(runs[0][k]), Hh.bits(r[k])), (jitter, k)


def _projection(tanx, tany, cx, cy, W, H, znear=0.01, zfar=100.0):
    """The row-vector projection of getProjectionMatrix(znear, zfar, fovX, fovY, cx, cy) (utils/graphics_utils.py)
    from tensors: P[0,0] = 1 / tanx, P[1,1] = 1 / tany, and the off-centre principal point in P[0,2], P[1,2] (column
    convention); transposed here, as the reference's Camera does."""
    z = torch.zeros((), dtype=tanx.dtype, device=tanx.device)
    one = torch.ones((), dtype=tanx.dtype, device=tanx.device)
    rows = [torch.stack([1 / tanx, z, 2 * cx / W - 1, z]),
            torch.stack([z, 1 / tany, 2 * cy / H - 1, z]),
            torch.stack([z, z, one * zfar / (zfar - znear), one * (-(zfar * znear) / (zfar - znear))]),
            torch.stack([z, z, one, z])]
    return torch.stack(rows).T


@pytest.mark.gpu
def test_focal_and_principal_point_refinement_end_to_end(cuda_device):
    """A synthetic scene rendered with the true intrinsics; the focal perturbed by a few percent and the principal
    point by a few pixels, through torch.tan of FoV leaves and a projection built from tensors.  Adam on the L1 image
    loss must shrink both errors by a clear factor."""
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam = S.blob_scene(6000, seed=21), S.simple_camera(256, 192)
    d = Hh.to_torch(scene, cam, dev)
    W, H = cam.width, cam.height
    view = d["viewmatrix"].reshape(4, 4)
    bg = torch.zeros(3, device=dev)
    f64 = dict(dtype=torch.float64)
    fovx0 = torch.tensor(2 * np.arctan(cam.tanfovx), **f64)
    fovy0 = torch.tensor(2 * np.arctan(cam.tanfovy), **f64)
    c0 = torch.tensor([W / 2, H / 2], **f64)

    def render(fovx, fovy, c):
        tanx, tany = torch.tan(fovx * 0.5), torch.tan(fovy * 0.5)
        proj = _projection(tanx, tany, c[0], c[1], W, H).float().to(dev)
        full = view @ proj
        rs = GaussianRasterizationSettings(H, W, tanx, tany, 0.1, torch.zeros(1, device=dev), bg, 1.0, view, full, 3,
                                           d["campos"], False, False)
        m2d = torch.zeros((scene.P, 3), device=dev, requires_grad=True)
        return GaussianRasterizer(rs)(d["means3D"], m2d, d["opacities"], shs=d["shs"], scales=d["scales"],
                                      rotations=d["rotations"])[0]

    @torch.no_grad()
    def errors(fovx, fovy, c):
        """Focal-length error (px, the norm over x and y) and principal-point error (px)."""
        fx = W / (2 * torch.tan(fovx * 0.5)) - W / (2 * torch.tan(fovx0 * 0.5))
        fy = H / (2 * torch.tan(fovy * 0.5)) - H / (2 * torch.tan(fovy0 * 0.5))
        return float(torch.sqrt(fx ** 2 + fy ** 2)), float((c - c0).norm())

    with torch.no_grad():
        target = render(fovx0, fovy0, c0)
    # focal +4 % in x, -3 % in y; principal point (+3, -2) px
    fovx = (2 * torch.atan(torch.tan(fovx0 * 0.5) / 1.04)).clone().requires_grad_(True)
    fovy = (2 * torch.atan(torch.tan(fovy0 * 0.5) / 0.97)).clone().requires_grad_(True)
    c = (c0 + torch.tensor([3.0, -2.0], **f64)).requires_grad_(True)
    f_start, c_start = errors(fovx, fovy, c)
    opt = torch.optim.Adam([{"params": [fovx, fovy], "lr": 1e-3}, {"params": [c], "lr": 0.1}])
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    for _ in range(300):
        opt.zero_grad()
        (render(fovx, fovy, c) - target).abs().mean().backward()
        assert fovx.grad is not None and torch.isfinite(fovx.grad) and torch.isfinite(c.grad).all()
        opt.step()
        sched.step()
    f_end, c_end = errors(fovx, fovy, c)
    print(f"\n[focal refinement] focal error {f_start:.3f} px -> {f_end:.4f} px ({f_start / max(f_end, 1e-12):.1f}x), "
          f"principal point {c_start:.3f} px -> {c_end:.4f} px ({c_start / max(c_end, 1e-12):.1f}x)")
    assert f_end < 0.1 * f_start, (f_start, f_end)
    assert c_end < 0.1 * c_start, (c_start, c_end)
