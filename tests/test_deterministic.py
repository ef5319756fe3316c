"""The deterministic backward (sfgs_rasterize_backward_deterministic, chosen by torch.use_deterministic_algorithms):
argument handling and the row addressing without a GPU; bit-reproducibility, accuracy against the float64
adjudicator, two-phase consistency and a seeded training loop on the GPU."""
import ctypes as C
import types
import warnings

import numpy as np
import pytest
import torch

import helpers as Hh
from golden_cases import build_case
from helpers import deterministic
from sfgs import synthetic as S

SFGS_E_UNSUPPORTED = -4
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot", "extra")


# ----------------------------------------------------------------------------- CPU
def test_unsupported_options_rejected_before_cuda_work():
    from sfgs import native
    L = native.lib()
    b = native.BackwardArgs()
    b.P, b.width, b.height = 8, 32, 32
    dummy = (C.c_float * 64)()
    ptr = C.cast(dummy, C.c_void_p)
    b.geom_buffer = b.binning_buffer = b.image_buffer = ptr
    for f in ("dL_dpix", "dL_dpix_depth", "dL_dpix_norm", "dL_dpix_alpha", "accum_alphas"):
        setattr(b, f, ptr)
    b.phase, b.acc = 1, ptr
    peers = (C.c_void_p * 2)(ptr, ptr)
    b.acc_peers, b.n_peers, b.peer_slice = C.cast(peers, C.POINTER(C.c_void_p)), 2, 4
    assert L.sfgs_rasterize_backward_deterministic(C.byref(b)) == SFGS_E_UNSUPPORTED
    assert "acc_peers" in native.last_error()
    b.acc_peers, b.n_peers, b.peer_slice = None, 0, 0
    b.phase, b.ED = 0, 2
    assert L.sfgs_rasterize_backward_deterministic(C.byref(b)) == SFGS_E_UNSUPPORTED
    assert "extra_attrs" in native.last_error()
    # phase 1 places each partial by the Gaussian's tile rectangle: radii are required
    b.ED, b.phase = 0, 1
    assert L.sfgs_rasterize_backward_deterministic(C.byref(b)) == -2 and "radii" in native.last_error()
    # the default entry point keeps its own answers
    b.phase, b.ED = 0, 2
    b.dL_dpix_extra = b.extra_attrs = b.dL_dextra = None
    assert L.sfgs_rasterize_backward(C.byref(b)) == -2


def _backward_with_extras(P):
    """rasterize_gaussians_backward with extra_attrs on CPU tensors; P == 0 returns before any device work."""
    from sfgs import rasterizer as R
    z = torch.zeros
    img = z(3, 4, 4)
    return R.rasterize_gaussians_backward(z(3), z(P, 3), z(P, dtype=torch.int32), z(0), z(P, 3), z(P, 4), z(5, 2), 1.0,
                                          z(0), z(0), z(4, 4), z(4, 4), 1.0, 1.0, 0.1, img, z(1, 4, 4), img, z(1, 4, 4),
                                          z(2, 4, 4), z(P, 16, 3), 3, z(3), z(1), 0, z(1), z(1), z(1, 4, 4), False)


def test_python_layer_raises_or_warns_for_options_without_deterministic_path():
    with deterministic(True):
        with pytest.raises(RuntimeError, match="does not have a deterministic implementation"):
            _backward_with_extras(0)
    with deterministic(True, warn_only=True):
        with pytest.warns(UserWarning, match="does not have a deterministic implementation"):
            out = _backward_with_extras(0)
        assert out[-1].shape == (0, 2)
    with deterministic(False):
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            _backward_with_extras(0)
    assert not torch.are_deterministic_algorithms_enabled()


def _tile_rect(mx, my, r, gx, gy):
    """tile_rect (sfgs_common.cuh) in float32: (x - r) / 16 truncated toward zero, clamped to [0, grid]."""
    f = np.float32
    c = lambda v, n: int(min(n, max(0, int(v))))  # noqa: E731
    return (c((f(mx) - f(r)) / f(16), gx), c((f(my) - f(r)) / f(16), gy),
            c((f(mx) + f(r) + f(15)) / f(16), gx), c((f(my) + f(r) + f(15)) / f(16), gy))


@pytest.mark.parametrize("seed", range(6))
def test_row_addressing_is_a_bijection_in_emission_order(seed):
    """(g, tile) -> off[g] + rank: the preprocess emits Gaussian g's instances as the kk-th tile of its band-clipped
    rectangle, row-major; the deterministic backward's inverse map puts the instance of (g, tile) at slot off[g] + rank
    with rank recomputed from the rectangle.  Over random rectangles (off the grid, clipped, empty, banded) the slots
    must cover [0, sum tiles_touched) exactly once, and slot off[g] + kk must be the kk-th emitted instance."""
    rng = np.random.default_rng(seed)
    W, H = int(rng.integers(17, 700)), int(rng.integers(17, 500))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    b0 = int(rng.integers(0, gy)) if seed % 2 else 0
    b1 = int(rng.integers(b0, gy + 1)) if seed % 2 else gy
    P = 3000
    mx = rng.uniform(-80, W + 80, P).astype(np.float32)
    my = rng.uniform(-80, H + 80, P).astype(np.float32)
    rad = np.where(rng.uniform(size=P) < 0.05, rng.integers(100, 400, P), rng.integers(0, 40, P))
    rects, tt = [], np.zeros(P, np.int64)
    emitted = []                                   # (g, tile) in the preprocess's order
    for g in range(P):
        x0, y0, x1, y1 = _tile_rect(mx[g], my[g], int(rad[g]), gx, gy)
        y0, y1 = max(y0, b0), min(y1, b1)
        n = (x1 - x0) * (y1 - y0) if y1 > y0 else 0
        rects.append((x0, y0, x1, y1))
        tt[g] = n
        for kk in range(n):
            ty, tx = divmod(kk, x1 - x0)
            emitted.append((g, (y0 + ty) * gx + x0 + tx))
    off = np.concatenate([[0], np.cumsum(tt)[:-1]])
    total = int(tt.sum())
    assert total == len(emitted) and total > 0
    slots = np.full(total, -1, np.int64)
    # the sorted order the inverse map walks: by tile, then any order inside (depth order does not matter here)
    order = sorted(range(total), key=lambda i: (emitted[i][1], rng.integers(1 << 30)))
    for i in order:
        g, tile = emitted[i]
        ty, tx = divmod(tile, gx)
        x0, y0 = rects[g][0], max(_tile_rect(mx[g], my[g], int(rad[g]), gx, gy)[1], b0)
        rank = (ty - y0) * (rects[g][2] - x0) + (tx - x0)
        s = off[g] + rank
        assert 0 <= rank < tt[g] and slots[s] == -1
        slots[s] = i
    assert (slots == np.arange(total)).all()       # a bijection, and slot off[g] + kk is the kk-th emitted instance


# ----------------------------------------------------------------------------- GPU
def _setup(scene, cam, dev, bg=(0.0, 0.0, 0.0), cot_seed=1, **kw):
    d = Hh.to_torch(scene, cam, dev)
    bg_t = torch.tensor(bg, device=dev, dtype=torch.float32)
    sh_degree = kw.pop("sh_degree", scene.sh_degree)
    f = Hh.run_ours_forward(d, cam, sh_degree, bg_t, **kw)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=cot_seed)]
    return d, bg_t, sh_degree, f, cot


def _run_bits(out):
    """The bits of a phase-1 call's sums, or of a backward's gradients, on the host."""
    return [Hh.bits(t).cpu() for t in ([out] if isinstance(out, torch.Tensor) else [out[k] for k in GRAD_KEYS])]


def _assert_three_runs_identical(d, cam, sh_degree, bg, f, cot, **kw):
    runs = [_run_bits(Hh.run_ours_backward(d, cam, sh_degree, bg, f, cot, det=True, **kw)) for _ in range(3)]
    for r in runs[1:]:
        for a, b, k in zip(runs[0], r, GRAD_KEYS):
            assert torch.equal(a, b), f"{k} differs between deterministic runs"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["golden_blob", "banded", "configs1_1M_jax004", "dense_5M_jax004"])
def test_bit_reproducible(cuda_device, case):
    dev = cuda_device
    kw = {}
    if case == "golden_blob":
        scene, cam, bg, kw = build_case("blob_sh3")
        bg = tuple(float(x) for x in bg)
        kw = {k: kw[k] for k in ("kernel_size", "scale_modifier")}
    elif case == "banded":
        scene, cam, bg = S.city_scene(120_000, seed=9, extent=120.0), S.jax004_camera(640, 360), (0.1, 0.0, 0.2)
    else:
        P = 1_000_000 if case.startswith("configs1") else 5_000_000
        scene, cam, bg = S.city_scene(P, seed=0), S.jax004_camera(1920, 1080), (0.0, 0.0, 0.0)
    if case == "banded":
        d = Hh.to_torch(scene, cam, dev)
        bg_t = torch.tensor(bg, device=dev)
        band = (3, 15)
        f = Hh.run_ours_forward(d, cam, 3, bg_t, tile_rows=band)
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=2)]
        _assert_three_runs_identical(d, cam, 3, bg_t, f, cot, tile_rows=band)
        # the band's deterministic gradients match its default ones up to the sums' order
        g_det = Hh.run_ours_backward(d, cam, 3, bg_t, f, cot, tile_rows=band, det=True)
        g_def = Hh.run_ours_backward(d, cam, 3, bg_t, f, cot, tile_rows=band)
        for k in GRAD_KEYS[:-1]:
            assert (g_det[k] - g_def[k]).abs().max().item() <= 1e-5 + 2e-4 * g_def[k].abs().max().item(), k
        return
    d, bg_t, sh_degree, f, cot = _setup(scene, cam, dev, bg=bg, **kw)
    _assert_three_runs_identical(d, cam, sh_degree, bg_t, f, cot, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", list(range(10)))
def test_bit_reproducible_randomised(cuda_device, seed):
    """The generator of the randomised differential configurations (test_gpu_parity)."""
    dev = cuda_device
    rng = np.random.default_rng(1000 + seed)
    P = int(rng.integers(1, 5000))
    W, H = int(rng.integers(17, 400)), int(rng.integers(17, 300))
    deg = int(rng.integers(0, 4))
    scene = S.blob_scene(P, seed=200 + seed, sh_degree=3, spread=float(rng.uniform(0.2, 3.0)),
                         scale=float(rng.uniform(0.01, 0.4)))
    cam = S.simple_camera(W, H, fov_deg=float(rng.uniform(30, 90)), distance=float(rng.uniform(3.0, 10.0)))
    kw = dict(kernel_size=float(rng.choice([0.05, 0.1, 0.3])), scale_modifier=float(rng.uniform(0.5, 2.0)))
    bg = tuple(float(x) for x in rng.uniform(0, 1, 3))
    d, bg_t, _, f, cot = _setup(scene, cam, dev, bg=bg, cot_seed=seed, sh_degree=deg, **kw)
    _assert_three_runs_identical(d, cam, deg, bg_t, f, cot, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["backward_blob", "backward_city", "benched_configs1_1M_jax004"])
def test_accurate_against_float64(cuda_device, tag):
    """One deterministic run passes the default path's float64 gate (ADJ_FACTORS, no outlier budget)."""
    dev = cuda_device
    F = Hh.RefFacts(tag)
    if tag == "backward_blob":
        scene, cam, bg, cs = S.blob_scene(6000, seed=31), S.simple_camera(320, 200), (0.1, 0.2, 0.3), 4
    elif tag == "backward_city":
        scene, cam, bg, cs = S.city_scene(300_000, seed=3), S.jax004_camera(1920, 1080), (0.1, 0.2, 0.3), 4
    else:
        scene, cam, bg, cs = S.city_scene(1_000_000, seed=0), S.jax004_camera(1920, 1080), (0.0, 0.0, 0.0), 1
    d, bg_t, sh, f, cot = _setup(scene, cam, dev, bg=bg, cot_seed=cs)
    P, H, W = scene.P, cam.height, cam.width
    oi = Hh.our_internals(f, P, H, W)
    gb = Hh.run_ours_backward(d, cam, sh, bg_t, f, cot, det=True)
    if F.live:
        from oracle import ref_cuda
        ref = Hh.run_ref_forward(d, cam, sh, bg_t)
        F.adjudicate(d, cam, sh, bg_t, oi, f["alpha"], f["radii"], cot, gb,
                     lambda: (ref_cuda.internals(ref, P, H, W), ref["alpha"], ref["radii"],
                              [Hh.run_ref_backward(d, cam, sh, bg_t, ref, cot) for _ in range(3)]),
                     f"deterministic[{tag}]")
    else:
        F.adjudicate(d, cam, sh, bg_t, oi, f["alpha"], f["radii"], cot, gb, None, f"deterministic[{tag}]")
    inv = f["radii"] == 0
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        assert gb[k][inv].abs().max().item() == 0.0 if inv.any() else True


@pytest.mark.gpu
def test_two_phase_equals_single_call(cuda_device):
    dev = cuda_device
    scene, cam = S.blob_scene(5000, seed=91), S.simple_camera(256, 144)
    d, bg_t, sh, f, cot = _setup(scene, cam, dev, bg=(0.3, 0.2, 0.1), cot_seed=4)
    one = Hh.run_ours_backward(d, cam, sh, bg_t, f, cot, det=True)
    acc = Hh.run_ours_backward(d, cam, sh, bg_t, f, cot, det=True, phase=1)
    assert torch.equal(acc.view(torch.int32),
                       Hh.run_ours_backward(d, cam, sh, bg_t, f, cot, det=True, phase=1).view(torch.int32))
    two = Hh.run_ours_backward(d, cam, sh, bg_t, f, cot, det=True, phase=2, acc=acc, gauss_range=(0, scene.P))
    for k in GRAD_KEYS[:-1]:
        assert torch.equal(one[k].view(torch.int32), two[k].view(torch.int32)), k


@pytest.mark.gpu
def test_default_path_unchanged_and_deterministic_path_used(cuda_device):
    """With torch's flag off the library runs the default kernels (no bwd_order stage); with it on, the ordered ones."""
    from sfgs import native as N
    dev = cuda_device
    scene, cam = S.blob_scene(3000, seed=5), S.simple_camera(160, 96)
    d, bg_t, sh, f, cot = _setup(scene, cam, dev)
    counts = {}
    for on in (False, True):
        N.profile_enable(True)
        try:
            with deterministic(on):
                Hh.run_ours_backward(d, cam, sh, bg_t, f, cot)
            torch.cuda.synchronize(dev)
            counts[on] = {k: v[1] for k, v in N.profile_read().items()}
        finally:
            N.profile_enable(False)
    assert counts[False]["bwd_order"] == 0 and counts[False]["render_bwd"] == 1 and counts[False]["gauss_bwd"] == 1
    assert counts[True]["bwd_order"] == 1 and counts[True]["render_bwd"] == 1 and counts[True]["gauss_bwd"] == 1


def _train(dev, iters=24):
    """A miniature Stage-1 loop: distCUDA2 init, render, L1 + fused SSIM, backward, Adam, densification statistics
    every step and one densify_and_prune (functional form) at the end.  Returns the final parameters."""
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from fused_ssim import fused_ssim
    from simple_knn._C import distCUDA2
    from sfgs import densify as DN
    torch.manual_seed(0)
    target_scene = S.blob_scene(4000, seed=7, spread=1.5, scale=0.12)
    cams = [S.orbit_camera(target=(0, 0, 0), elevation_deg=30.0, azimuth_deg=a, radius=7.0, fov_deg=50.0, width=160,
                           height=128) for a in (0.0, 90.0, 180.0, 270.0)]
    bg = torch.zeros(3, device=dev)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731

    def render(p, cam):
        rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, 0.1, torch.zeros(1, device=dev),
                                           bg, 1.0, t(cam.viewmatrix), t(cam.projmatrix), 3, t(cam.campos), False, False)
        m2d = torch.zeros_like(p["xyz"], requires_grad=True)
        shs = torch.cat([p["f_dc"], p["f_rest"]], 1)
        out = GaussianRasterizer(rs)(p["xyz"], m2d, torch.sigmoid(p["opacity"]), shs=shs, scales=torch.exp(p["scaling"]),
                                     rotations=torch.nn.functional.normalize(p["rotation"]))
        return out[0], out[4], m2d

    with torch.no_grad():
        tp = t(target_scene.shs)
        tparams = dict(xyz=t(target_scene.means3D), f_dc=tp[:, :1].contiguous(), f_rest=tp[:, 1:].contiguous(),
                       opacity=torch.logit(t(target_scene.opacities).clamp(1e-4, 1 - 1e-4)),
                       scaling=torch.log(t(target_scene.scales)), rotation=t(target_scene.rotations))
        targets = [render(tparams, c)[0].clone() for c in cams]
    rng = np.random.default_rng(0)
    xyz = t((target_scene.means3D + rng.normal(0, 0.05, target_scene.means3D.shape)).astype(np.float32))
    P = xyz.shape[0]
    d2 = distCUDA2(xyz).clamp_min(1e-7)
    p = dict(xyz=xyz.clone(), f_dc=torch.zeros((P, 1, 3), device=dev), f_rest=torch.zeros((P, 15, 3), device=dev),
             opacity=torch.full((P, 1), -2.0, device=dev), scaling=torch.log(torch.sqrt(d2))[:, None].repeat(1, 3).contiguous(),
             rotation=t(np.tile(np.array([1, 0, 0, 0], np.float32), (P, 1))))
    for v in p.values():
        v.requires_grad_(True)
    opt = torch.optim.Adam([{"params": [p["xyz"]], "lr": 2e-3}, {"params": [p["scaling"]], "lr": 5e-3},
                            {"params": [p["rotation"]], "lr": 1e-3}, {"params": [p["opacity"]], "lr": 5e-2},
                            {"params": [p["f_dc"], p["f_rest"]], "lr": 2e-2}])
    z = lambda: torch.zeros(P, device=dev)  # noqa: E731
    max_r, acc, acc_abs, acc_abs_max, denom = z(), z(), z(), z(), z()
    for it in range(iters):
        cam, gt = cams[it % 4], targets[it % 4]
        img, radii, m2d = render(p, cam)
        loss = 0.8 * (img - gt).abs().mean() + 0.2 * (1.0 - fused_ssim(img[None], gt[None]))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        vs = types.SimpleNamespace(grad=torch.nn.functional.pad(m2d.grad, (0, 1)).contiguous())
        pc = types.SimpleNamespace(max_radii2D=max_r, xyz_gradient_accum=acc, xyz_gradient_accum_abs=acc_abs,
                                   xyz_gradient_accum_abs_max=acc_abs_max, denom=denom)
        DN.add_densification_stats(pc, vs, radii)
    with torch.no_grad():
        params = {k: v.detach().contiguous() for k, v in p.items()}
        new_p, _, _, totals = DN.densify_tensors(params, None, None, acc, acc_abs, denom, max_grad=2e-4,
                                                 min_opacity=0.005, extent=3.0, max_screen_size=None, percent_dense=0.01)
    return new_p, totals


@pytest.mark.gpu
def test_training_loop_reproducible_end_to_end(cuda_device):
    dev = cuda_device
    with deterministic(True):
        runs = []
        for _ in range(2):
            torch.manual_seed(0)
            runs.append(_train(dev))
    (p0, t0), (p1, t1) = runs
    assert t0 == t1 and t0["new_P"] > 0, (t0, t1)
    for k in p0:
        assert torch.equal(p0[k].view(torch.int32), p1[k].view(torch.int32)), k
