"""GPU parity at the configuration Skyfall-GS trains with (README: `--sh_degree 1 --appearance_enabled
--kernel_size 0.1`).  gaussian_renderer.render() then calls the rasterizer in two ways: with precomputed colours from
the appearance MLP (every training step once an appearance embedding exists, M = 0) and with the stored SH of a
degree-1 model (M = 4).  The SH widths other than 16 take their own paths through the kernels: the preprocess reads
them straight from global memory instead of staging them with cp.async, the per-Gaussian adjoint gathers them in 4- or
16-byte units depending on 3M and writes dL_dsh rows 3M floats wide.

  - randomised configurations at M = 1, 4, 9 and with precomputed colours against the reference CUDA build (indexing,
    colours and clamp flags bit for bit, images within 1e-5, gradients adjudicated in float64);
  - the benched 1M-Gaussian frame at M = 4 and with precomputed colours, default and deterministic backward;
  - dL_dsh beyond the active degree, the SH-degree argument check, the two-phase backward at odd cuts, the autograd
    wrapper with a `colors_precomp` leaf, and the CPU oracle at M = 1, 4, 9 (no reference facts needed).
"""
import numpy as np
import pytest
import torch

import helpers as Hh
from helpers import bits, deterministic
from sfgs import synthetic as S
from test_gpu_parity import check_images, check_indexing, ref_internals

pytestmark = pytest.mark.gpu
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")
ZERO_WHEN_CULLED = ("means2D", "colors", "opacity", "means3D", "sh", "scales", "rot")

SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)


def appearance_colors(shs, means3D, campos, D):
    """`colors_precomp` formed the way the appearance branch of render() forms them, in float32 torch:
    clamp_min(eval_sh(D, sh, normalize(xyz - campos)) + 0.5, 0).  The DC term is first stretched and shifted,
    v -> 1.5 v - 0.3 for v = SH_C0 * dc + 0.5, so that about a fifth of the channels clamp to exactly 0 and some
    exceed 1 (the MLP's output is not confined to [0, 1] either).  shs [P, M, 3] with (D + 1)^2 <= M, D <= 2."""
    assert D <= 2 and (D + 1) ** 2 <= shs.shape[1]
    sh = shs.clone()
    sh[:, 0] = (1.5 * (S.SH_C0 * sh[:, 0] + 0.5) - 0.3 - 0.5) / S.SH_C0
    d = torch.nn.functional.normalize(means3D - campos[None], dim=1)
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    c = S.SH_C0 * sh[:, 0]
    if D > 0:
        c = c - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
    if D > 1:
        xx, yy, zz = x * x, y * y, z * z
        c = (c + SH_C2[0] * x * y * sh[:, 4] + SH_C2[1] * y * z * sh[:, 5] + SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 6]
             + SH_C2[3] * x * z * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
    colors = torch.clamp_min(c + 0.5, 0.0).contiguous()
    zero = float((colors == 0).float().mean())
    assert 0.1 < zero < 0.35 and bool((colors > 1).any()), zero
    return colors


def near_clamp(scene, seed, frac=0.3):
    """Moves the DC term of a fraction of the Gaussians so that SH_C0 * dc + 0.5 lies within 0.1 of the clamp at 0:
    with the view-dependent terms on top, about half of their channels clamp, and dL_dsh of those channels is 0."""
    rng = np.random.default_rng(seed)
    sel = rng.uniform(size=scene.P) < frac
    v = rng.uniform(-0.1, 0.1, size=(int(sel.sum()), 3))
    scene.shs[sel, 0, :] = ((v - 0.5) / S.SH_C0).astype(np.float32)
    return scene


def unpack_clamped(packed):
    return torch.stack([(packed >> k) & 1 for k in range(3)], 1).bool()


def check_colours(F, oi, ri, vis, col):
    """SH mode: colours and clamp flags of the visible Gaussians bit for bit with the reference.  Precomputed mode:
    the blend record carries the input colours unchanged."""
    if col is None:
        F.same("rgb", bits(oi["rgb"][vis]), lambda: bits(ri["rgb"][vis]))
        F.same("clamped", unpack_clamped(oi["clamped"])[vis], lambda: ri["clamped"][vis].bool())
    else:
        assert torch.equal(bits(oi["rgb"][vis]), bits(col[vis]))


def check_clamped_sh_zero(gb, clamped, vis):
    """A clamped channel passes no gradient to any of its SH coefficients."""
    cm = clamped & vis[:, None]
    assert bool(cm.any()), "no clamped channel among the visible Gaussians"
    g = gb["sh"].permute(0, 2, 1)[cm]                 # [n, M] rows of the clamped (Gaussian, channel) pairs
    assert g.abs().max().item() == 0.0


def forward_pair(d, cam, D, bg_t, col, live, **kw):
    ours = Hh.run_ours_forward(d, cam, D, bg_t, colors=col, **kw)
    ref = Hh.run_ref_forward(d, cam, D, bg_t, colors=col, **kw) if live else None
    return ours, ref


# ----------------------------------------------------------------------------- 1. randomised, training widths
# (stored degree m, active degree D, colour mode, kernel_size 0.1): every width and mode, D = m and D < m, the
# README's filter size on half the seeds; everything else is drawn like test_randomised_differential_vs_reference
RANDOMISED = [(1, 1, "sh", True), (1, 0, "sh", False), (2, 2, "sh", True), (2, 1, "sh", False),
              (0, 0, "sh", True), (1, 1, "precomp", False), (2, 2, "precomp", True), (0, 0, "precomp", False)]


@pytest.mark.parametrize("seed", list(range(len(RANDOMISED))))
def test_randomised_training_widths_vs_reference(cuda_device, seed):
    m, D, mode, k01 = RANDOMISED[seed]
    F = Hh.RefFacts(f"trainconf_rand_{seed}")
    dev = cuda_device
    rng = np.random.default_rng(3000 + seed)
    P = int(rng.integers(300, 5000))
    W, H = int(rng.integers(17, 400)), int(rng.integers(17, 300))
    scene = S.blob_scene(P, seed=300 + seed, sh_degree=m, spread=float(rng.uniform(0.2, 3.0)),
                         scale=float(rng.uniform(0.01, 0.4)))
    if mode == "sh":
        near_clamp(scene, seed)
    cam = S.simple_camera(W, H, fov_deg=float(rng.uniform(30, 90)), distance=float(rng.uniform(3.0, 10.0)))
    ks = 0.1 if k01 else float(rng.choice([0.05, 0.3]))
    kw = dict(kernel_size=ks, scale_modifier=float(rng.uniform(0.5, 2.0)))
    bg_t = torch.tensor(rng.uniform(0, 1, 3), device=dev, dtype=torch.float32)
    d = Hh.to_torch(scene, cam, dev)
    col = appearance_colors(d["shs"], d["means3D"], d["campos"], D) if mode == "precomp" else None
    ours, ref = forward_pair(d, cam, D, bg_t, col, F.live, **kw)
    oi, ri = Hh.our_internals(ours, P, H, W), ref_internals(ref, P, H, W)
    check_indexing(F, ours, ref, oi, ri)
    vis = ours["radii"] > 0
    check_colours(F, oi, ri, vis, col)
    check_images(F, ours, ref)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=seed)]
    gbs = [Hh.run_ours_backward(d, cam, D, bg_t, ours, cot, colors=col, **kw) for _ in range(3)]
    if mode == "sh":
        check_clamped_sh_zero(gbs[0], unpack_clamped(oi["clamped"]), vis)
    F.adjudicate(d, cam, D, bg_t, oi, ours["alpha"], ours["radii"], cot, gbs,
                 lambda: (ri, ref["alpha"], ref["radii"],
                          [Hh.run_ref_backward(d, cam, D, bg_t, ref, cot, colors=col, **kw) for _ in range(3)]),
                 f"trainconf_rand[{seed}: M={(m + 1) ** 2} D={D} {mode} k={ks}]", colors=col, **kw)


# ----------------------------------------------------------------------------- 2./3. the benched frame, trained setup
def _headline(dev, mode):
    """bench.py's 1M-Gaussian jax004 frame with a degree-1 model (the geometry is the benched one: the generator draws
    the SH last), kernel 0.1, black background, bench.py's cotangents."""
    scene, cam = S.city_scene(1_000_000, seed=0, sh_degree=1), S.jax004_camera(1920, 1080)
    d = Hh.to_torch(scene, cam, dev)
    bg_t = torch.zeros(3, device=dev)
    col = appearance_colors(d["shs"], d["means3D"], d["campos"], 1) if mode == "precomp" else None
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=1)]
    return scene, cam, d, bg_t, col, cot


@pytest.mark.parametrize("mode", ["m4", "precomp"])
def test_headline_frame_training_config_vs_reference(cuda_device, mode):
    F = Hh.RefFacts(f"trainconf_1M_jax004_{mode}")
    dev = cuda_device
    scene, cam, d, bg_t, col, cot = _headline(dev, mode)
    P, H, W = scene.P, cam.height, cam.width
    ours, ref = forward_pair(d, cam, 1, bg_t, col, F.live)
    oi, ri = Hh.our_internals(ours, P, H, W), ref_internals(ref, P, H, W)
    check_indexing(F, ours, ref, oi, ri)
    vis = ours["radii"] > 0
    check_colours(F, oi, ri, vis, col)
    check_images(F, ours, ref)
    clamped = unpack_clamped(oi["clamped"])
    if F.live:
        oi = None          # the reference's intermediates feed the adjudicator; keep one set resident
    gbs = [Hh.run_ours_backward(d, cam, 1, bg_t, ours, cot, colors=col) for _ in range(3)]
    if col is None:
        check_clamped_sh_zero(gbs[0], clamped, vis)
    F.adjudicate(d, cam, 1, bg_t, oi, ours["alpha"], ours["radii"], cot, gbs,
                 lambda: (ri, ref["alpha"], ref["radii"],
                          [Hh.run_ref_backward(d, cam, 1, bg_t, ref, cot, colors=col) for _ in range(3)]),
                 f"trainconf_1M_jax004[{mode}]", colors=col)
    inv = ~vis
    for k in ZERO_WHEN_CULLED:
        if gbs[0][k].numel():
            assert gbs[0][k][inv].abs().max().item() == 0.0, k       # culled Gaussians get exact zeros


@pytest.mark.parametrize("mode", ["m4", "precomp"])
def test_headline_frame_deterministic_backward(cuda_device, mode):
    """One deterministic run passes the same float64 gate; three runs are byte-identical (M = 4 and M = 0)."""
    F = Hh.RefFacts(f"trainconf_1M_jax004_{mode}")
    F.record = False       # the facts of this frame are recorded by test_headline_frame_training_config_vs_reference
    dev = cuda_device
    scene, cam, d, bg_t, col, cot = _headline(dev, mode)
    P, H, W = scene.P, cam.height, cam.width
    f = Hh.run_ours_forward(d, cam, 1, bg_t, colors=col)
    oi = Hh.our_internals(f, P, H, W)
    with deterministic(True):
        runs = [Hh.run_ours_backward(d, cam, 1, bg_t, f, cot, colors=col) for _ in range(3)]
    for r in runs[1:]:
        for k in GRAD_KEYS:
            assert torch.equal(bits(runs[0][k]), bits(r[k])), f"{k} differs between deterministic runs"
    gb = runs[0]
    if F.live:
        from oracle import ref_cuda
        ref = Hh.run_ref_forward(d, cam, 1, bg_t, colors=col)
        F.adjudicate(d, cam, 1, bg_t, oi, f["alpha"], f["radii"], cot, gb,
                     lambda: (ref_cuda.internals(ref, P, H, W), ref["alpha"], ref["radii"],
                              [Hh.run_ref_backward(d, cam, 1, bg_t, ref, cot, colors=col) for _ in range(3)]),
                     f"deterministic[trainconf_1M_jax004_{mode}]", colors=col)
    else:
        F.adjudicate(d, cam, 1, bg_t, oi, f["alpha"], f["radii"], cot, gb, None,
                     f"deterministic[trainconf_1M_jax004_{mode}]", colors=col)
    inv = f["radii"] == 0
    for k in ZERO_WHEN_CULLED:
        if gb[k].numel():
            assert gb[k][inv].abs().max().item() == 0.0, k


# ----------------------------------------------------------------------------- 4. dL_dsh beyond the active degree
@pytest.mark.parametrize("m,D", [(1, 0), (2, 0), (2, 1)])
def test_dsh_beyond_active_degree_is_zero(cuda_device, m, D):
    """Coefficients k >= (D + 1)^2 do not enter the colour: their gradient is exactly 0 (-0.0 allowed: the kernel
    multiplies dL/dRGB by a zero factor), in the default and the deterministic backward.  The active ones are not."""
    dev = cuda_device
    M, n = (m + 1) ** 2, (D + 1) ** 2
    scene, cam = S.blob_scene(3000, seed=71 + 3 * m + D, sh_degree=m), S.simple_camera(200, 136)
    d = Hh.to_torch(scene, cam, dev)
    bg_t = torch.tensor([0.2, 0.1, 0.3], device=dev)
    f = Hh.run_ours_forward(d, cam, D, bg_t)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=5)]
    gb = Hh.run_ours_backward(d, cam, D, bg_t, f, cot)
    with deterministic(True):
        gd = Hh.run_ours_backward(d, cam, D, bg_t, f, cot)
    for g in (gb["sh"], gd["sh"]):
        assert g.shape == (scene.P, M, 3)
        assert g[:, n:].abs().max().item() == 0.0
        vis = f["radii"] > 0
        assert bool((g[vis, :n] != 0).any(2).all(1).any())


def test_sh_degree_beyond_stored_width_is_rejected(cuda_device):
    """An active degree D whose (D + 1)^2 coefficients the stored width M cannot hold is an argument error (BADARG),
    not a read past the end of each SH row."""
    from sfgs import native as N
    dev = cuda_device
    cam = S.simple_camera(64, 48)
    bg_t = torch.zeros(3, device=dev)
    for m, D in ((0, 1), (1, 2), (2, 3)):
        d = Hh.to_torch(S.blob_scene(100, seed=3, sh_degree=m), cam, dev)
        with pytest.raises(N.SfgsError, match="code -2: forward: SH degree"):
            Hh.run_ours_forward(d, cam, D, bg_t)


# ----------------------------------------------------------------------------- 5. two-phase backward, odd widths
@pytest.mark.parametrize("m", [1, 2])
def test_two_phase_backward_at_odd_sh_widths(cuda_device, m):
    """test_two_phase_backward_equals_single_call at M = 4 and 9, cut at an odd Gaussian index.  At M = 9 the second
    slice's dL_dsh rows (27 floats) then start off a 16-byte boundary, as do the 1-, 3-, 4- and 6-wide arrays: the
    head and tail stores of the epilogue write them.  The per-Gaussian adjoint of each slice is bit-identical to that
    of the whole range fed the same sums."""
    dev = cuda_device
    scene, cam = S.blob_scene(5000, seed=91, sh_degree=m), S.simple_camera(256, 144)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.3, 0.2, 0.1], device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=4)]
    f = Hh.run_ours_forward(d, cam, m, bg)
    one = Hh.run_ours_backward(d, cam, m, bg, f, cot)
    acc = Hh.run_ours_backward(d, cam, m, bg, f, cot, phase=1)
    whole = Hh.run_ours_backward(d, cam, m, bg, f, cot, phase=2, acc=acc.clone(), gauss_range=(0, scene.P))
    for cut in (2173, 97):
        parts = [Hh.run_ours_backward(d, cam, m, bg, f, cot, phase=2, acc=acc[a:b].clone(), gauss_range=(a, b))
                 for a, b in ((0, cut), (cut, scene.P))]
        for k in GRAD_KEYS:
            got = torch.cat([parts[0][k][:cut], parts[1][k][cut:]], 0)
            assert got.shape == one[k].shape, k
            assert torch.equal(bits(got), bits(whole[k])), (cut, k)
            tol = 1e-5 + 2e-4 * one[k].abs().max().item()     # the sums carry the reductions' order noise
            assert (got - one[k]).abs().max().item() <= tol, (cut, k)


# ----------------------------------------------------------------------------- 6. autograd wrapper
@pytest.mark.parametrize("mode", ["precomp", "m4"])
def test_autograd_wrapper_training_config(cuda_device, mode):
    """diff_gauss.GaussianRasterizer called as render() calls it: `colors_precomp` a leaf that requires grad
    (appearance branch), or the stored SH of a degree-1 model; every leaf's gradient equals the native call's."""
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam = S.blob_scene(2000, seed=52, sh_degree=1), S.simple_camera(160, 96)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.2, 0.3, 0.4], device=dev)
    col = appearance_colors(d["shs"], d["means3D"], d["campos"], 1) if mode == "precomp" else None
    names = ["means3D", "opacities", "scales", "rotations"] + (["shs"] if col is None else [])
    leaves = {k: d[k].clone().requires_grad_(True) for k in names}
    if col is not None:
        leaves["colors"] = col.clone().requires_grad_(True)
    m2d = torch.zeros((scene.P, 3), device=dev, requires_grad=True)
    rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, 0.1, torch.zeros(1, device=dev),
                                       bg, 1.0, d["viewmatrix"], d["projmatrix"], 1, d["campos"], False, False)
    color, depth, norm, alpha, radii, _ = GaussianRasterizer(rs)(
        leaves["means3D"], m2d, leaves["opacities"], shs=leaves.get("shs"), colors_precomp=leaves.get("colors"),
        scales=leaves["scales"], rotations=leaves["rotations"])
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=8)]
    (color * cot[0]).sum().add((depth * cot[1]).sum()).add((alpha * cot[3]).sum()).backward()
    f = Hh.run_ours_forward(d, cam, 1, bg, colors=col)
    assert torch.equal(color.detach(), f["color"]) and torch.equal(radii, f["radii"])
    gb = Hh.run_ours_backward(d, cam, 1, bg, f, [cot[0], cot[1], torch.zeros_like(cot[2]), cot[3]], colors=col)
    pairs = [("means3D", "means3D"), ("opacities", "opacity"), ("scales", "scales"), ("rotations", "rot")]
    pairs.append(("shs", "sh") if col is None else ("colors", "colors"))
    for leaf, key in pairs:
        a, b = leaves[leaf].grad, gb[key]
        assert a is not None and a.shape == leaves[leaf].shape, leaf
        assert (a - b).abs().max().item() <= 1e-5 + 1e-5 * b.abs().max().item(), leaf
    if col is None:
        assert leaves["shs"].grad.shape == (scene.P, 4, 3)
    assert m2d.grad.shape == (scene.P, 3)


# ----------------------------------------------------------------------------- 7. CPU oracle at M = 1, 4, 9
@pytest.mark.parametrize("m", [0, 1, 2])
def test_sh_widths_against_cpu_oracle(cuda_device, m):
    """test_against_cpu_oracle's checks and tolerances at M = 1, 4, 9 with D = m: needs neither the reference build
    nor its recorded facts."""
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene, cam = S.blob_scene(2500, seed=41 + m, sh_degree=m), S.simple_camera(190, 150)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    d = Hh.to_torch(scene, cam, dev)
    f = Hh.run_ours_forward(d, cam, m, torch.from_numpy(bg).to(dev))
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, m, cam.viewmatrix,
                  cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg)
    assert np.array_equal(f["radii"].cpu().numpy(), o["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    assert np.array_equal(it["tiles_touched"].cpu().numpy().astype(np.uint32), o["tiles_touched"])
    for k in ("color", "depth", "norm", "alpha"):
        assert np.abs(f[k].cpu().numpy() - o[k]).max() <= 5e-5, k   # glibc expf vs CUDA expf, borderline alpha tests
    cot = S.cotangents(cam.width, cam.height, seed=6)
    gb = Hh.run_ours_backward(d, cam, m, torch.from_numpy(bg).to(dev), f, [torch.from_numpy(c).to(dev) for c in cot])
    og = O.backward(o, *cot)
    assert gb["sh"].shape == og["sh"].shape == (scene.P, (m + 1) ** 2, 3)
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        a, b = gb[k].cpu().numpy().astype(np.float64), og[k].astype(np.float64)
        assert np.abs(a - b).max() <= 1e-4 + 2e-4 * np.abs(b).max(), k
