"""Camera gradients (sfgs_rasterize_backward_camera): dL/dviewmatrix, dL/dprojmatrix and dL/dcampos, the adjoint of the
chain dL_dmean3D differentiates.  The oracle is tests/chain_f64.py: for given blend-adjoint sums it restates
that chain in torch, and its gradient with respect to means3D must reproduce the library's dL_dmean3D.

CPU: the C ABI's argument checks, the autograd layer's native call sequence (the reference's own render() on a
recording native layer), the restatement against the CPU oracle's dL_dmeans3D, and the translation identity.
GPU: the other outputs bit-identical to the calls without camera gradients, accuracy against the float64 restatement,
the translation identity at 1080p, reproducibility, and pose refinement end to end through diff_gauss."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import chain_f64 as CH
import golden_cases as G
import helpers as Hh
from helpers import release_cached_frames  # noqa: F401
from sfgs import synthetic as S

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")


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
        assert L.sfgs_rasterize_backward_camera(C.byref(b), off, det, dst) == code, what
        assert what in N.last_error(), (what, N.last_error())
    assert L.sfgs_rasterize_backward_camera(None, None, 0, out) == SFGS_E_BADARG


# ----------------------------------------------------------------------------- CPU: the autograd layer's native calls
from test_reference_caller import _camera, _fill, needs_reference, reference_stack  # noqa: E402,F401


def _optimizing_camera(W=80, H=48):
    """Camera(..., optimizing=True) of scene/cameras.py: world_view_transform from R, T leaves through differentiable
    ops, full_proj_transform a bmm of it, camera_center from its inverse."""
    c = _camera(W, H)
    V0 = c.world_view_transform.double().T              # world -> view, column-vector convention
    R = V0[:3, :3].T.clone().requires_grad_(True)       # the reference's R is the transpose of the w2c rotation
    T = V0[:3, 3].clone().requires_grad_(True)
    Rt = torch.cat([torch.cat([R.T, T[:, None]], 1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=torch.float64)], 0)
    wvt = Rt.T.float()
    proj = torch.linalg.solve(c.world_view_transform.double(), c.full_proj_transform.double()).float()
    c.world_view_transform = wvt
    c.full_proj_transform = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0)
    c.camera_center = wvt.inverse()[3, :3]
    return c, R, T


@needs_reference
@pytest.mark.parametrize("mode", ["plain", "camera", "camera_offsets"])
def test_reference_render_calls_the_camera_entry_only_when_the_camera_requires_grad(reference_stack, monkeypatch,
                                                                                      mode):
    import diff_gauss
    from diff_gauss import _C
    render, GaussianModel, rec = reference_stack
    seen = []

    def recording(fn):
        def call(*a, camera_grad=False, subpixel_offset=None, **kw):
            seen.append((camera_grad, subpixel_offset))
            out = fn(*a, **kw)
            if camera_grad:
                g = torch.Generator().manual_seed(2)
                out = out + (torch.rand((4, 4), generator=g), torch.rand((4, 4), generator=g), torch.rand(3, generator=g))
            return out
        return call
    for name in ("rasterize_gaussians_backward", "rasterize_gaussians_backward_fused"):
        monkeypatch.setattr(_C, name, recording(getattr(_C, name)))
    monkeypatch.setattr(_C, "rasterize_gaussians_fused",
                        lambda *a, subpixel_offset=None: _C.rasterize_gaussians(*a, fuse_normalize=True))
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", mode == "camera_offsets")
    pc = GaussianModel(3, False, 4, 32)
    _fill(pc, 200, False)
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
    off = torch.rand((48, 80, 2)) - 0.5
    if mode == "plain":
        cam = _camera()
    else:
        cam, R, T = _optimizing_camera()
    out = render(cam, pc, pipe, torch.zeros(3), kernel_size=0.1, subpixel_offset=off)
    out["render"].mean().backward()
    assert len(rec["fwd"]) == 1 and len(seen) == 1
    if mode == "plain":
        assert seen == [(False, None)]
        return
    assert seen[0][0] is True
    if mode == "camera_offsets":
        assert seen[0][1] is not None and torch.equal(seen[0][1], off)
    else:
        assert seen[0][1] is None
    # the camera gradients reached the pose parameters through the reference's own matrix code
    assert R.grad is not None and T.grad is not None and bool(torch.isfinite(R.grad).all())
    assert pc._xyz.grad is not None


def test_autograd_layer_without_the_reference_tree(monkeypatch):
    """The same through diff_gauss directly: the camera entry only when one of the three camera tensors requires grad,
    and gradients only for those that do, in their dtype."""
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer, _C
    P, H, W = 50, 24, 32
    calls = []

    def fwd(*a, fuse_normalize=False, subpixel_offset=None):
        r = (torch.ones(P, dtype=torch.int32),)
        out = (7, torch.rand(3, H, W), torch.rand(1, H, W), torch.rand(3, H, W), torch.rand(1, H, W)) + r + (
            torch.empty(0), torch.zeros(8, dtype=torch.uint8), torch.zeros(8, dtype=torch.uint8),
            torch.zeros(8, dtype=torch.uint8))
        return out + (torch.rand(3, H, W),) if fuse_normalize else out

    def bwd(*a, norm_raw=None, camera_grad=False, subpixel_offset=None):
        calls.append(camera_grad)
        z = lambda *s: torch.full(s, 0.5)  # noqa: E731
        out = (z(P, 3), z(P, 3), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 16, 3), z(P, 3), z(P, 4), torch.empty(0))
        return out + (z(4, 4), 2 * z(4, 4), 3 * z(3)) if camera_grad else out
    monkeypatch.setattr(_C, "rasterize_gaussians", fwd)
    monkeypatch.setattr(_C, "rasterize_gaussians_fused", lambda *a, **kw: fwd(*a, fuse_normalize=True, **kw))
    monkeypatch.setattr(_C, "rasterize_gaussians_backward", bwd)
    monkeypatch.setattr(_C, "rasterize_gaussians_backward_fused", bwd)

    def run(view_grad, proj_grad, cam_grad):
        view = torch.eye(4).requires_grad_(view_grad)
        proj = torch.eye(4).requires_grad_(proj_grad)
        campos = torch.zeros(3).requires_grad_(cam_grad)
        rs = GaussianRasterizationSettings(H, W, 0.5, 0.5, 0.1, torch.zeros(1), torch.zeros(3), 1.0, view, proj, 3,
                                           campos, False, False)
        means = torch.zeros(P, 3, requires_grad=True)
        out = GaussianRasterizer(rs)(means, torch.zeros(P, 3, requires_grad=True), torch.ones(P, 1),
                                     shs=torch.zeros(P, 16, 3), scales=torch.ones(P, 3), rotations=torch.ones(P, 4))
        out[0].sum().backward()
        return view.grad, proj.grad, campos.grad, means.grad
    for fuse in (True, False):
        monkeypatch.setattr(diff_gauss, "FUSE_NORMALIZE", fuse)
        calls.clear()
        gv, gp, gc, gm = run(False, False, False)
        assert calls == [False] and gv is None and gp is None and gc is None and gm is not None
        calls.clear()
        gv, gp, gc, _ = run(False, True, False)
        assert calls == [True] and gv is None and gc is None and torch.equal(gp, torch.full((4, 4), 1.0))
        gv, gp, gc, _ = run(True, False, True)
        assert gp is None and torch.equal(gv, torch.full((4, 4), 0.5)) and torch.equal(gc, torch.full((3,), 1.5))


# ----------------------------------------------------------------------------- CPU: the restatement and the oracle
def _oracle_case(name):
    from oracle import cpu_oracle as O
    scene, cam, bg, kw = G.build_case(name)
    colors = kw.get("colors")
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, kw["sh_degree"],
                  cam.viewmatrix, cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg,
                  kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"], colors_precomp=colors)
    g = O.backward(o, *kw["cot"])
    s = O.blend_backward(o, *kw["cot"])
    acc = CH.acc_from_screen_grads(s["means2D"], s["colors"], s["depths"], s["norm3D"], s["conic"], s["opacity"])
    r = CH.chain(acc, o["radii"], scene.means3D, o["conic_opacity"][:, 3], o["clamped"] != 0,
                 None if colors is not None else scene.shs, kw["sh_degree"], cam.viewmatrix, cam.projmatrix, cam.campos,
                 cam.width, cam.height, cam.tanfovx, cam.tanfovy, kw["kernel_size"], cov3D=o["cov3D"])
    return scene, cam, g, r


@pytest.mark.parametrize("name", G.CASES)
def test_restatement_reproduces_the_oracle_mean_gradient(name):
    scene, cam, g, r = _oracle_case(name)
    ours, ref = r["means3D"].numpy(), g["means3D"].astype(np.float64)
    err = np.abs(ours - ref).max()
    assert err <= 2e-5 * np.abs(ref).max(), (name, err, np.abs(ref).max())
    if name == "blob_precomp":
        assert torch.equal(r["campos"], torch.zeros(3, dtype=torch.float64))


@pytest.mark.parametrize("name", G.CASES)
def test_translation_identity_of_the_restatement(name):
    scene, cam, g, r = _oracle_case(name)
    res, scale = CH.translation_residual(r, cam.viewmatrix, cam.projmatrix)
    assert (res.abs() <= 1e-12 * scale + 1e-300).all(), (name, res, scale)


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
def test_other_outputs_unchanged(cuda_device, name):
    """Every non-camera output of the camera call is bit-identical to the deterministic calls (with and without
    offsets).  The default and the deterministic backward hand their sums to the same per-Gaussian kernel, so this is
    also the bit-for-bit check for the default calls; those reduce with unordered atomics and do not reproduce
    themselves.  Their camera form is compared within the zero-offset test's bound on the outputs that the near-singular
    conics do not amplify (the means3D / cov3D / scales / rot gradients of two default calls can differ by more than any
    fixed multiple of their spread)."""
    dev = cuda_device
    for jitter in (False, True):
        scene, cam, D, d, colors, bg, off, f, cot = _setup(name, dev, jitter)
        keys = [k for k in GRAD_KEYS if not (colors is not None and k == "sh")]
        a = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True)
        b = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True, camera_grad=True)
        for k in keys:
            assert torch.equal(Hh.bits(a[k]), Hh.bits(b[k])), (name, jitter, "deterministic", k)
        g1, g2 = (Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off) for _ in range(2))
        gc = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, camera_grad=True)
        for k in [k for k in keys if k in ("means2D", "colors", "opacity", "norm3D", "sh")]:
            spread = (g1[k].double() - g2[k].double()).abs().max().item()
            err = (gc[k].double() - g1[k].double()).abs().max().item()
            tol = 1e-4 + 2e-4 * g1[k].abs().max().item() + 2.0 * spread
            assert err <= tol, (name, jitter, k, err, spread, tol)
        assert all(torch.isfinite(gc[k]).all() for k in ("view", "proj", "campos"))


def _accuracy_case(case, dev):
    """GPU camera gradients of a deterministic call and the restatement (float64 and float32) from the phase-1 sums of
    a deterministic run: the same `acc` bits the camera call uses."""
    def make():
        name = {"d3": "jax004", "d1": "m4", "precomp": "precomp"}[case.split("_")[0]]
        scene, cam, D, d, colors, bg, off, f, cot = _setup(name, dev, case.endswith("jitter"))
        g = Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True, camera_grad=True)
        a = Hh.restatement_inputs(f, d, cam, D, bg, cot, colors, off)
        r64 = CH.chain(**a, dtype=torch.float64)
        r32 = CH.chain(**a, dtype=torch.float32)
        return cam, d, g, r64, r32, colors
    return Hh.cached("case", case, make)


def _flat(r):
    return torch.cat([r["view"].reshape(16), r["proj"].reshape(16), r["campos"].reshape(3)]).double()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["d3", "d3_jitter", "d1", "d1_jitter", "precomp", "precomp_jitter"])
def test_accuracy_against_float64(cuda_device, case):
    cam, d, g, r64, r32, colors = _accuracy_case(case, cuda_device)
    gpu, f64, f32 = _flat(g), _flat(r64), _flat(r32)
    tol = torch.maximum(2.0 * (f32 - f64).abs(), 1e-6 * r64["abs"].double())
    err = (gpu - f64).abs()
    print(f"\n[camera {case}] max err / tol {float((err / tol.clamp_min(1e-300)).max()):.3f}")
    assert (err <= tol).all(), (case, torch.nonzero(err > tol).flatten().tolist(), err, tol)
    # entries the forward never reads
    assert torch.equal(g["view"][:, 3], torch.zeros(4, device=g["view"].device))
    assert torch.equal(g["proj"][:, 2], torch.zeros(4, device=g["proj"].device))
    if colors is not None:
        assert torch.equal(g["campos"], torch.zeros(3, device=g["campos"].device))
    # the restatement mirrors the chain: its mean gradient is the library's dL_dmean3D
    ref = r64["means3D"]
    e = (g["means3D"].double() - ref).abs().flatten()
    assert torch.quantile(e[:1 << 24].float(), 0.999).item() <= 1e-5 * ref.abs().max().item(), case


@pytest.mark.gpu
def test_translation_identity_at_1080p(cuda_device):
    cam, d, g, r64, _, _ = _accuracy_case("d3", cuda_device)
    gg = dict(means3D=g["means3D"].double(), view=g["view"].double(), proj=g["proj"].double(),
              campos=g["campos"].double())
    res, _ = CH.translation_residual(gg, d["viewmatrix"].double(), d["projmatrix"].double())
    Vm, Pm = d["viewmatrix"].double().reshape(4, 4), d["projmatrix"].double().reshape(4, 4)
    a = r64["abs"].double()
    scale = (g["means3D"].double().abs().sum(0) + a[32:35] + (Vm[:3].abs() * a[12:16]).sum(1)
             + (Pm[:3].abs() * a[28:32]).sum(1))
    assert (res.abs() <= 1e-5 * scale).all(), (res, scale)


@pytest.mark.gpu
def test_deterministic_camera_gradients_are_reproducible(cuda_device):
    dev = cuda_device
    for jitter in (False, True):
        scene, cam, D, d, colors, bg, off, f, cot = _setup("jax004", dev, jitter)
        runs = [Hh.run_ours_backward(d, cam, D, bg, f, cot, colors=colors, subpixel_offset=off, det=True,
                                     camera_grad=True) for _ in range(3)]
        for k in ("view", "proj", "campos"):
            for r in runs[1:]:
                assert torch.equal(Hh.bits(runs[0][k]), Hh.bits(r[k])), (jitter, k)


def _so3(w):
    """exp of the skew matrix of w (Rodrigues), differentiable at w = 0."""
    th2 = (w * w).sum()
    K = torch.zeros(3, 3, dtype=w.dtype, device=w.device)
    K = K + torch.stack([torch.stack([0 * w[0], -w[2], w[1]]), torch.stack([w[2], 0 * w[0], -w[0]]),
                         torch.stack([-w[1], w[0], 0 * w[0]])])
    th = torch.sqrt(th2 + 1e-30)
    a = torch.where(th2 > 1e-12, torch.sin(th) / th, 1 - th2 / 6)
    b = torch.where(th2 > 1e-12, (1 - torch.cos(th)) / th2, 0.5 - th2 / 24)
    return torch.eye(3, dtype=w.dtype, device=w.device) + a * K + b * (K @ K)


def _pose_camera(R0, T0, proj, w, tau):
    """The matrices of Camera(..., optimizing=True) (scene/cameras.py) for R = R0 exp(w), T = T0 + tau: the row-vector
    world-to-view transform [[R, 0], [T, 1]], its product with the projection and the camera centre from its inverse."""
    R = R0 @ _so3(w)
    T = T0 + tau
    top = torch.cat([R, torch.zeros(3, 1, dtype=R.dtype, device=R.device)], 1)
    bottom = torch.cat([T, torch.ones(1, dtype=R.dtype, device=R.device)])[None]
    wvt = torch.cat([top, bottom], 0).float()
    full = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0)
    return wvt, full, wvt.inverse()[3, :3]


@pytest.mark.gpu
def test_pose_refinement_end_to_end(cuda_device):
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam = S.blob_scene(6000, seed=21), S.simple_camera(256, 192)
    d = Hh.to_torch(scene, cam, dev)
    V0 = d["viewmatrix"].double()
    proj = torch.linalg.solve(V0, d["projmatrix"].double()).float()
    R0, T0 = V0[:3, :3].clone(), V0[3, :3].clone()
    bg = torch.zeros(3, device=dev)
    focal = cam.height / (2 * cam.tanfovy)

    def render(w, tau):
        view, full, campos = _pose_camera(R0, T0, proj, w, tau)
        rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, 0.1,
                                           torch.zeros(1, device=dev), bg, 1.0, view, full, 3, campos, False, False)
        m2d = torch.zeros((scene.P, 3), device=dev, requires_grad=True)
        return GaussianRasterizer(rs)(d["means3D"], m2d, d["opacities"], shs=d["shs"], scales=d["scales"],
                                      rotations=d["rotations"])

    def pixel_error(w, tau):
        """Mean image-plane displacement (px) of the Gaussians' centres between the pose and the true one."""
        with torch.no_grad():
            def px(full):
                h = torch.cat([d["means3D"], torch.ones(scene.P, 1, device=dev)], 1) @ full
                return h[:, :2] / h[:, 3:4]
            _, f1, _ = _pose_camera(R0, T0, proj, w, tau)
            _, f0, _ = _pose_camera(R0, T0, proj, torch.zeros_like(w), torch.zeros_like(tau))
            dx = (px(f1) - px(f0)) * torch.tensor([cam.width / 2, cam.height / 2], device=dev)
            return dx.norm(dim=1).mean().item()

    zero = torch.zeros(3, dtype=torch.float64, device=dev)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            target = render(zero, zero)[0]
        # a small rotation and a translation, scaled so that the start is 2.5 px off
        w0 = torch.tensor([0.004, -0.006, 0.008], dtype=torch.float64, device=dev)
        tau0 = torch.tensor([0.08, -0.06, 0.10], dtype=torch.float64, device=dev)
        s = 2.5 / pixel_error(w0, tau0)
        w, tau = (w0 * s).requires_grad_(True), (tau0 * s).requires_grad_(True)
        start = pixel_error(w, tau)
        assert 2.0 <= start <= 3.0, start
        opt = torch.optim.Adam([{"params": [tau], "lr": 1e-2}, {"params": [w], "lr": 1e-3}])
        sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.95)
        for _ in range(100):
            opt.zero_grad()
            img = render(w, tau)[0]
            ((img - target) ** 2).sum().backward()
            assert w.grad is not None and tau.grad is not None and torch.isfinite(w.grad).all()
            opt.step()
            sched.step()
        end = pixel_error(w, tau)
        print(f"\n[pose refinement] reprojection error {start:.3f} px -> {end:.4f} px (focal {focal:.1f} px)")
        assert end < 0.1 * start, (start, end)
        # detached camera: no gradient, and the default native call
        w2 = w.detach().clone().requires_grad_(True)
        tau2 = tau.detach().clone().requires_grad_(True)
        img = render(w2.detach(), tau2.detach())[0]
        ((img - target) ** 2).sum().backward()
        assert w2.grad is None and tau2.grad is None
    finally:
        torch.use_deterministic_algorithms(prev)
