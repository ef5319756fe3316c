"""GPU parity tests (run with `-m gpu` on an H100): the CUDA path through the C ABI against
  (1) the unmodified reference CUDA rasterizer — bit-exact tile/key indexing, 1e-5 images, gradients adjudicated by a
      float64 evaluation of the reference's algorithm (helpers.adjudicate_gradients: our error against float64 <= 2x
      the reference build's own error + 1e-5, every element, no outlier budget).  Live where the reference build is in
      oracle/_ref; elsewhere against what such a run on an H100 recorded (helpers.RefFacts, tests/golden/reference/),
  (2) the CPU oracle (oracle/sfgs_oracle.c),
  (3) the committed golden fixtures produced by the reference (tests/golden/ref_*.npz),
plus edge cases and size-independent properties at the BASELINE.json full size.
"""
import os

import numpy as np
import pytest
import torch

import helpers as Hh
from golden_cases import CASES, build_case
from sfgs import synthetic as S

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
IMG_ATOL = 1e-5          # north_star: 1e-5 abs on rendered RGB / depth


def ref_available():
    from oracle import ref_cuda
    return ref_cuda.available()


def ref_internals(ref, P, H, W):
    from oracle import ref_cuda
    return ref_cuda.internals(ref, P, H, W) if ref is not None else None


def bits(t):
    return t.contiguous().view(torch.int32) if t.dtype.is_floating_point else t


def run_pair(scene, cam, dev, bg=(0.1, 0.2, 0.3), colors=None, live=True, **kw):
    """This library's forward and, when `live`, the reference build's (else None)."""
    d = Hh.to_torch(scene, cam, dev)
    bg_t = torch.tensor(bg, device=dev, dtype=torch.float32)
    col = None if colors is None else torch.from_numpy(colors).to(dev)
    sh_degree = kw.pop("sh_degree", scene.sh_degree)
    ours = Hh.run_ours_forward(d, cam, sh_degree, bg_t, colors=col, **kw)
    ref = Hh.run_ref_forward(d, cam, sh_degree, bg_t, colors=col, **kw) if live else None
    return d, bg_t, col, ours, ref


def check_indexing(F, ours, ref, oi, ri, full=True):
    """Every indexing quantity bit for bit (radii, num_rendered, ranges, point_list, n_contrib; with `full` also
    tiles_touched, depths / means2D / cov3D / conic and the keys)."""
    assert ours["num_rendered"] == F.value("num_rendered", lambda: int(ref["num_rendered"]))
    F.same("radii", ours["radii"], lambda: ref["radii"])
    F.same("ranges", oi["ranges"], lambda: ri["ranges"])
    F.same("point_list", oi["point_list"], lambda: ri["point_list"])
    F.same("n_contrib", oi["n_contrib"], lambda: ri["n_contrib"])
    if full:
        vis = ours["radii"] > 0
        F.same("tiles_touched", oi["tiles_touched"], lambda: ri["tiles_touched"])
        for k in ("depths", "means2D", "cov3D", "conic_opacity"):
            F.same(k, bits(oi[k][vis]), lambda: bits(ri[k][vis]))
        F.same("keys", Hh.ref_style_keys(oi["ranges"], oi["keys"]), lambda: ri["keys"])


def check_images(F, ours, ref, tag=""):
    for k in ("color", "depth", "norm", "alpha"):
        F.close(k + tag, ours[k], lambda: ref[k], IMG_ATOL)




@pytest.mark.parametrize("case", ["blob", "city", "precomp", "modifier"])
def test_forward_bit_exact_indexing_vs_reference(cuda_device, case):
    F = Hh.RefFacts(f"indexing_{case}")
    dev = cuda_device
    kw, colors = {}, None
    if case == "blob":
        scene, cam = S.blob_scene(6000, seed=21), S.simple_camera(333, 217)
    elif case == "city":
        scene, cam = S.city_scene(200_000, seed=2), S.jax004_camera(1920, 1080)
    elif case == "precomp":
        scene, cam = S.blob_scene(3000, seed=22, sh_degree=0), S.simple_camera(256, 256)
        colors = np.random.default_rng(0).uniform(0, 1, (scene.P, 3)).astype(np.float32)
    else:
        scene, cam = S.blob_scene(3000, seed=23), S.simple_camera(200, 120)
        kw = dict(kernel_size=0.3, scale_modifier=1.7, sh_degree=2)
    d, bg_t, col, ours, ref = run_pair(scene, cam, dev, colors=colors, live=F.live, **kw)
    P, H, W = scene.P, cam.height, cam.width
    oi, ri = Hh.our_internals(ours, P, H, W), ref_internals(ref, P, H, W)
    check_indexing(F, ours, ref, oi, ri)
    vis = ours["radii"] > 0
    if colors is None:
        F.same("rgb", bits(oi["rgb"][vis]), lambda: bits(ri["rgb"][vis]))     # colours, hence clamp flags, bit for bit
    check_images(F, ours, ref)


@pytest.mark.parametrize("case", ["blob", "city"])
def test_backward_vs_reference_adjudicated_by_float64(cuda_device, case):
    F = Hh.RefFacts(f"backward_{case}")
    dev = cuda_device
    if case == "blob":
        scene, cam = S.blob_scene(6000, seed=31), S.simple_camera(320, 200)
    else:
        scene, cam = S.city_scene(300_000, seed=3), S.jax004_camera(1920, 1080)
    d, bg_t, col, ours, ref = run_pair(scene, cam, dev, live=F.live)
    P, H, W = scene.P, cam.height, cam.width
    oi = Hh.our_internals(ours, P, H, W)
    check_indexing(F, ours, ref, oi, ref_internals(ref, P, H, W), full=False)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=4)]
    gb = Hh.run_ours_backward(d, cam, scene.sh_degree, bg_t, ours, cot)
    gbs = [gb] + [Hh.run_ours_backward(d, cam, scene.sh_degree, bg_t, ours, cot) for _ in range(2)]     # this library's reductions are unordered too
    F.adjudicate(d, cam, scene.sh_degree, bg_t, oi, ours["alpha"], ours["radii"], cot, gbs,
                 lambda: (ref_internals(ref, P, H, W), ref["alpha"], ref["radii"],
                          [Hh.run_ref_backward(d, cam, scene.sh_degree, bg_t, ref, cot) for _ in range(3)]),
                 f"backward_vs_reference[{case}]")
    # culled Gaussians get exact zeros
    inv = ours["radii"] == 0
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        assert gb[k][inv].abs().max().item() == 0.0 if inv.any() else True


@pytest.mark.parametrize("seed", list(range(10)))
def test_randomised_differential_vs_reference(cuda_device, seed):
    """Seeded random configurations (image sizes off the tile grid, every SH degree, scale modifiers, filter sizes,
    backgrounds, cluster tightness) against the unmodified reference CUDA rasterizer: indexing bit-exact, images
    within 1e-5, gradients adjudicated by the float64 evaluation (helpers.adjudicate_gradients)."""
    F = Hh.RefFacts(f"randomised_{seed}")
    dev = cuda_device
    rng = np.random.default_rng(1000 + seed)
    P = int(rng.integers(1, 5000))
    W, H = int(rng.integers(17, 400)), int(rng.integers(17, 300))
    deg = int(rng.integers(0, 4))
    scene = S.blob_scene(P, seed=200 + seed, sh_degree=3, spread=float(rng.uniform(0.2, 3.0)),
                         scale=float(rng.uniform(0.01, 0.4)))
    cam = S.simple_camera(W, H, fov_deg=float(rng.uniform(30, 90)), distance=float(rng.uniform(3.0, 10.0)))
    kw = dict(kernel_size=float(rng.choice([0.05, 0.1, 0.3])), scale_modifier=float(rng.uniform(0.5, 2.0)), sh_degree=deg)
    bg = tuple(float(x) for x in rng.uniform(0, 1, 3))
    d, bg_t, col, ours, ref = run_pair(scene, cam, dev, bg=bg, live=F.live, **kw)
    oi = Hh.our_internals(ours, P, H, W)
    check_indexing(F, ours, ref, oi, ref_internals(ref, P, H, W), full=False)
    check_images(F, ours, ref)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=seed)]
    gb = Hh.run_ours_backward(d, cam, deg, bg_t, ours, cot, kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"])
    gbs = [gb] + [Hh.run_ours_backward(d, cam, deg, bg_t, ours, cot, kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"]) for _ in range(2)]     # this library's reductions are unordered too
    F.adjudicate(d, cam, deg, bg_t, oi, ours["alpha"], ours["radii"], cot, gbs,
                 lambda: (ref_internals(ref, P, H, W), ref["alpha"], ref["radii"],
                          [Hh.run_ref_backward(d, cam, deg, bg_t, ref, cot, kernel_size=kw["kernel_size"],
                                               scale_modifier=kw["scale_modifier"]) for _ in range(3)]),
                 f"randomised[{seed}]", kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"])


@pytest.mark.parametrize("name", CASES)
def test_against_golden_fixtures(cuda_device, name):
    path = os.path.join(GOLD, f"ref_{name}.npz")
    if not os.path.exists(path):
        pytest.skip("golden fixture not generated yet")
    g = np.load(path)
    dev = cuda_device
    scene, cam, bg, kw = build_case(name)
    d = Hh.to_torch(scene, cam, dev)
    bg_t = torch.from_numpy(bg).to(dev)
    col = torch.from_numpy(kw["colors"]).to(dev) if kw.get("colors_precomp") else None
    f = Hh.run_ours_forward(d, cam, kw["sh_degree"], bg_t, kernel_size=kw["kernel_size"],
                            scale_modifier=kw["scale_modifier"], colors=col)
    assert f["num_rendered"] == int(g["num_rendered"])
    assert np.array_equal(f["radii"].cpu().numpy(), g["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["point_list"].cpu().numpy(), g["int_point_list"])
    assert np.array_equal(it["ranges"].cpu().numpy(), g["int_ranges"])
    assert np.array_equal(it["n_contrib"].cpu().numpy(), g["int_n_contrib"])
    for k in ("color", "depth", "norm", "alpha"):
        assert np.abs(f[k].cpu().numpy() - g[k]).max() <= IMG_ATOL, k
    cot = [torch.from_numpy(c).to(dev) for c in kw["cot"]]
    gb = Hh.run_ours_backward(d, cam, kw["sh_degree"], bg_t, f, cot, kernel_size=kw["kernel_size"],
                              scale_modifier=kw["scale_modifier"], colors=col)
    gbs = [gb] + [Hh.run_ours_backward(d, cam, kw["sh_degree"], bg_t, f, cot, kernel_size=kw["kernel_size"],
                              scale_modifier=kw["scale_modifier"], colors=col) for _ in range(2)]     # this library's reductions are unordered too
    # the fixture holds one run of the reference CUDA build's gradients; whose error a deviation is, is decided by
    # the float64 adjudicator on this library's forward intermediates (asserted bit-identical on indexing above)
    ref_g = {k: torch.from_numpy(g["grad_" + k]).to(dev) for k in ("means2D", "colors", "opacity", "means3D", "cov3D",
                                                                  "norm3D", "sh", "scales", "rot")}
    # (one stored run of a non-deterministic reference: its worst element is a single draw of an extreme-value
    # statistic — on blob_sh3 this library's own worst `means3D` element ranges from 3.6e-4 to 2.1e-3 over eight runs —
    # so that factor is wider here than in the live tests, and where the reference build travels with the snapshot its
    # live gradients of the same case join the stored run: every reference statistic is the largest over the runs)
    if ref_available():
        fr = Hh.run_ref_forward(d, cam, kw["sh_degree"], bg_t, kernel_size=kw["kernel_size"],
                                scale_modifier=kw["scale_modifier"], colors=col)
        ref_g = [ref_g] + [Hh.run_ref_backward(d, cam, kw["sh_degree"], bg_t, fr, cot, kernel_size=kw["kernel_size"],
                                               scale_modifier=kw["scale_modifier"], colors=col) for _ in range(3)]
    Hh.adjudicate_gradients(d, cam, kw["sh_degree"], bg_t, it, f["alpha"], f["radii"], cot, gbs, ref_g,
                            f"golden[{name}]", kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"],
                            colors=col, factors={"mean": 1.5, "p999": 2.0, "max": 8.0})


def test_against_cpu_oracle(cuda_device):
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene, cam = S.blob_scene(2500, seed=41), S.simple_camera(190, 150)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    d = Hh.to_torch(scene, cam, dev)
    f = Hh.run_ours_forward(d, cam, 3, torch.from_numpy(bg).to(dev))
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, 3, cam.viewmatrix,
                  cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg)
    assert np.array_equal(f["radii"].cpu().numpy(), o["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    assert np.array_equal(it["tiles_touched"].cpu().numpy().astype(np.uint32), o["tiles_touched"])
    for k in ("color", "depth", "norm", "alpha"):
        assert np.abs(f[k].cpu().numpy() - o[k]).max() <= 5e-5, k   # glibc expf vs CUDA expf, borderline alpha tests
    cot = S.cotangents(cam.width, cam.height, seed=6)
    gb = Hh.run_ours_backward(d, cam, 3, torch.from_numpy(bg).to(dev), f, [torch.from_numpy(c).to(dev) for c in cot])
    og = O.backward(o, *cot)
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        a, b = gb[k].cpu().numpy().astype(np.float64), og[k].astype(np.float64)
        assert np.abs(a - b).max() <= 1e-4 + 2e-4 * np.abs(b).max(), k


@pytest.mark.parametrize("ED", [1, 34])
def test_extra_attrs_vs_cpu_oracle(cuda_device, ED):
    """extra_attrs (ED channels, 34 = SFGS_MAX_EXTRA) on an image that is not a multiple of the tile: the extras and
    their gradients against the CPU oracle, and every other forward output bit-identical to the same call without
    extras (both run one blend loop)."""
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene, cam = S.blob_scene(2500, seed=41), S.simple_camera(190, 150)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    bg_t = torch.from_numpy(bg).to(dev)
    rng = np.random.default_rng(ED)
    extras = rng.uniform(-1, 1, (scene.P, ED)).astype(np.float32)
    dL_extra = rng.uniform(-1, 1, (ED, cam.height, cam.width)).astype(np.float32)
    d = Hh.to_torch(scene, cam, dev)
    f0 = Hh.run_ours_forward(d, cam, 3, bg_t)
    f = Hh.run_ours_forward(d, cam, 3, bg_t, extras=torch.from_numpy(extras).to(dev))
    for k in ("color", "depth", "norm", "alpha"):
        assert torch.equal(bits(f[k]), bits(f0[k])), k
    n_contrib = lambda fw: Hh.our_internals(fw, scene.P, cam.height, cam.width)["n_contrib"]  # noqa: E731
    assert torch.equal(n_contrib(f), n_contrib(f0))
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, 3, cam.viewmatrix,
                  cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg, extras=extras)
    assert np.abs(f["extra"].cpu().numpy() - o["extra"]).max() <= 5e-5   # glibc expf vs CUDA expf, as above
    cot = S.cotangents(cam.width, cam.height, seed=6)
    gb = Hh.run_ours_backward(d, cam, 3, bg_t, f, [torch.from_numpy(c).to(dev) for c in cot],
                              extras=torch.from_numpy(extras).to(dev), dL_extra=torch.from_numpy(dL_extra).to(dev))
    og = O.backward(o, *cot, dL_extra=dL_extra)
    for k in ("extra", "means2D", "opacity", "means3D"):
        a, b = gb[k].cpu().numpy().astype(np.float64), og[k].astype(np.float64)
        assert np.abs(a - b).max() <= 1e-4 + 2e-4 * np.abs(b).max(), k


def test_edge_cases(cuda_device):
    dev = cuda_device
    from sfgs import rasterizer as R
    e = torch.empty(0, device=dev)
    bg = torch.tensor([0.5, 0.25, 0.125], device=dev)
    # --- everything behind the camera: background only, zero gradients
    scene, cam = S.blob_scene(500, seed=1), S.simple_camera(70, 50)
    scene.means3D[:, 2] -= 100.0
    d = Hh.to_torch(scene, cam, dev)
    f = Hh.run_ours_forward(d, cam, 3, bg)
    assert f["num_rendered"] == 0 and int((f["radii"] > 0).sum()) == 0
    assert torch.allclose(f["color"], bg[:, None, None].expand_as(f["color"]))
    assert f["alpha"].abs().max().item() == 0 and f["depth"].abs().max().item() == 0
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height)]
    gb = Hh.run_ours_backward(d, cam, 3, bg, f, cot)
    assert all(v.abs().max().item() == 0 for k, v in gb.items() if v.numel())
    # --- P == 0 short-circuits like the reference (zero images, no background)
    out = R.rasterize_gaussians(bg, torch.zeros((0, 3), device=dev), e, e, e, e, 1.0, e, e, e, 0, d["viewmatrix"],
                                d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cam.height, cam.width, e, 3,
                                d["campos"], False, False)
    assert out[0] == 0 and out[1].abs().max().item() == 0
    # --- a single huge splat covering the whole image, image size 1 px off a tile multiple
    one = S.blob_scene(1, seed=2)
    one.means3D[:] = 0; one.scales[:] = 3.0; one.opacities[:] = 0.9
    cam1 = S.simple_camera(33, 17)
    d1 = Hh.to_torch(one, cam1, dev)
    f1 = Hh.run_ours_forward(d1, cam1, 3, bg)
    tiles = ((33 + 15) // 16) * ((17 + 15) // 16)
    assert f1["num_rendered"] == tiles and f1["alpha"].max().item() > 0.5 and f1["alpha"].min().item() > 0
    # --- capacity overflow: a hint of 1 instance forces the re-run path and must give the same result
    scene2, cam2 = S.blob_scene(3000, seed=5), S.simple_camera(128, 128)
    d2 = Hh.to_torch(scene2, cam2, dev)
    a = Hh.run_ours_forward(d2, cam2, 3, bg)
    b = R.rasterize_gaussians(bg, d2["means3D"], e, d2["opacities"], d2["scales"], d2["rotations"], 1.0, e, e, e, 0,
                              d2["viewmatrix"], d2["projmatrix"], cam2.tanfovx, cam2.tanfovy, 0.1, cam2.height,
                              cam2.width, d2["shs"], 3, d2["campos"], False, False, capacity_hint=1)
    assert b[0] == a["num_rendered"] and torch.equal(b[1], a["color"]) and torch.equal(b[5], a["radii"])


def test_long_tile_lists_use_both_sort_paths(cuda_device):
    """> 1024 and > 4096 instances in one tile exercise the heavy sort window and the global radix fallback."""
    F = Hh.RefFacts("long_tile_lists")
    dev = cuda_device
    scene, cam = S.blob_scene(9000, seed=77, spread=0.25, scale=0.05), S.simple_camera(64, 64, distance=10.0)
    d, bg_t, col, ours, ref = run_pair(scene, cam, dev, bg=(0, 0, 0), live=F.live)
    oi, ri = Hh.our_internals(ours, scene.P, 64, 64), ref_internals(ref, scene.P, 64, 64)
    check_indexing(F, ours, ref, oi, ri, full=False)
    longest = int((oi["ranges"][:, 1] - oi["ranges"][:, 0]).max())
    assert longest > 4096, longest
    F.close("color", ours["color"], lambda: ref["color"], IMG_ATOL)
    # the oversized-tile path (single-CTA radix sort through global memory) must stay in the same league as the
    # reference's global radix sort on the same frame, not fall off a cliff (the reference's time is the one recorded
    # on an H100 where its build is absent)
    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize(dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            fn()
        b.record()
        torch.cuda.synchronize(dev)
        return a.elapsed_time(b) / 10
    t_ours = timed(lambda: Hh.run_ours_forward(d, cam, 3, bg_t))
    t_ref = F.value("forward_ms", lambda: timed(lambda: Hh.run_ref_forward(d, cam, 3, bg_t)))
    print(f"\n[long tile lists] longest {longest}: forward {t_ours:.3f} ms (reference {t_ref:.3f} ms)")
    assert t_ours <= 1.5 * t_ref + 0.2, (t_ours, t_ref)


@pytest.mark.parametrize("n", [1, 2, 31, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 4095, 4096, 4097])
def test_sort_class_boundaries_and_depth_ties(cuda_device, n):
    """ONE tile (a 16x16 image) whose list has exactly `n` instances, at every size-class boundary of the per-tile sort:
    warp class with 4 / 8 / 16 keys per lane (<= 128 / 256 / 512), CTA class with 4 / 16 keys per thread (<= 1024 / 4096),
    global radix beyond.  A third of the Gaussians are exact duplicates of others (what densification's clone step
    produces): equal depths, so the order inside the tile is decided by the Gaussian id exactly like the reference's stable
    radix sort decides it."""
    F = Hh.RefFacts(f"sort_boundaries_{n}")
    dev = cuda_device
    scene = S.blob_scene(n, seed=1000 + n, spread=0.05, scale=0.08)
    dup = np.arange(n) % 3 == 2
    scene.means3D[dup] = scene.means3D[np.maximum(np.flatnonzero(dup) - 1, 0)]      # exact copies: depth ties
    cam = S.simple_camera(16, 16, distance=6.0)
    d, bg_t, col, ours, ref = run_pair(scene, cam, dev, bg=(0, 0, 0), live=F.live)
    oi, ri = Hh.our_internals(ours, scene.P, 16, 16), ref_internals(ref, scene.P, 16, 16)
    assert n == F.value("num_rendered", lambda: int(ref["num_rendered"])) == int(ours["num_rendered"])
    F.same("ranges", oi["ranges"], lambda: ri["ranges"])
    assert int(oi["ranges"][0, 1] - oi["ranges"][0, 0]) == n
    F.same("point_list", oi["point_list"][:n], lambda: ri["point_list"][:n])
    F.same("n_contrib", oi["n_contrib"], lambda: ri["n_contrib"])
    F.same("depth", ours["depth"], lambda: ref["depth"])
    F.same("alpha", ours["alpha"], lambda: ref["alpha"])
    F.close("color", ours["color"], lambda: ref["color"], IMG_ATOL)


def test_unpacked_key_path_for_more_than_2p24_gaussians(cuda_device):
    """With P > 2^24 a Gaussian id no longer fits beside the reach mask in the sort key: the scatter then writes
    depth_bits << 32 | id and the sort kernels form the masks from the blend records at emit time.  The switch is read
    once per process, so the indexing / size-class / long-list / needle tests are re-run in a child process with
    SFGS_KEYS_PACKED=0 (small scenes through exactly that path)."""
    import subprocess
    import sys
    env = dict(os.environ, SFGS_KEYS_PACKED="0")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-k",
                        "indexing or boundaries or long_tile or needles"], env=env, capture_output=True, text=True,
                       timeout=900, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_full_size_properties(cuda_device):
    """BASELINE configs[1] size (1M Gaussians, 1080p): size-independent invariants."""
    dev = cuda_device
    scene, cam = S.city_scene(1_000_000, seed=0), S.jax004_camera(1920, 1080)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.zeros(3, device=dev)
    f = Hh.run_ours_forward(d, cam, 3, bg)
    g = Hh.run_ours_forward(d, cam, 3, bg)
    for k in ("color", "depth", "norm", "alpha", "radii"):
        assert torch.equal(f[k], g[k]), f"forward not deterministic: {k}"
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    R = f["num_rendered"]
    assert R == int(it["tiles_touched"].long().sum()) == int((it["ranges"][:, 1] - it["ranges"][:, 0]).sum())
    keys = Hh.ref_style_keys(it["ranges"], it["keys"])
    assert bool((keys[1:] >= keys[:-1]).all())                          # sorted by (tile, depth)
    same = keys[1:] == keys[:-1]
    assert bool((it["point_list"][1:][same] > it["point_list"][:-1][same]).all())   # ties by Gaussian id
    assert bool(((f["alpha"] >= 0) & (f["alpha"] <= 1)).all())
    assert int(it["n_contrib"].max()) <= int((it["ranges"][:, 1] - it["ranges"][:, 0]).max())
    # backward is linear in the cotangents
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=1)]
    g1 = Hh.run_ours_backward(d, cam, 3, bg, f, cot)
    g2 = Hh.run_ours_backward(d, cam, 3, bg, f, [2.0 * c for c in cot])
    for k in ("means3D", "opacity", "sh", "scales", "rot", "colors"):
        a, b = g1[k].double(), g2[k].double()
        assert (2 * a - b).abs().max().item() <= 1e-3 * (1 + b.abs().max().item()), k   # reductions are order-free
    # abs-gradient channel dominates the signed ones
    m2 = g1["means2D"]
    assert bool((m2[:, 2] + 1e-3 >= m2[:, 0].abs() * 0).all()) and bool((m2[:, 2] >= 0).all())


def test_autograd_api_matches_native_calls(cuda_device):
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam = S.blob_scene(2000, seed=51), S.simple_camera(160, 96)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.2, 0.3, 0.4], device=dev)
    leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    m2d = torch.zeros((scene.P, 3), device=dev, requires_grad=True)
    rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, 0.1, torch.zeros(1, device=dev),
                                       bg, 1.0, d["viewmatrix"], d["projmatrix"], 3, d["campos"], False, False)
    rast = GaussianRasterizer(rs)
    color, depth, norm, alpha, radii, extra = rast(leaves["means3D"], m2d, leaves["opacities"], shs=leaves["shs"],
                                                   scales=leaves["scales"], rotations=leaves["rotations"])
    assert color.shape == (3, cam.height, cam.width) and depth.shape == (1, cam.height, cam.width)
    assert radii.dtype == torch.int32 and extra.numel() == 0
    nrm = norm.norm(dim=0)
    assert bool(((nrm - 1).abs() < 1e-4)[alpha[0] > 0.05].all())      # normals come back unit length
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=8)]
    (color * cot[0]).sum().add((depth * cot[1]).sum()).add((alpha * cot[3]).sum()).backward()
    f = Hh.run_ours_forward(d, cam, 3, bg)
    zero_n = torch.zeros_like(cot[2])
    gb = Hh.run_ours_backward(d, cam, 3, bg, f, [cot[0], cot[1], zero_n, cot[3]])
    assert torch.equal(color.detach(), f["color"]) and torch.equal(radii, f["radii"])
    assert m2d.grad.shape == (scene.P, 3)
    for leaf, key in (("means3D", "means3D"), ("opacities", "opacity"), ("shs", "sh"), ("scales", "scales"),
                      ("rotations", "rot")):
        a, b = leaves[leaf].grad, gb[key]
        assert (a - b).abs().max().item() <= 1e-5 + 1e-5 * b.abs().max().item(), leaf
    vis = rast.markVisible(d["means3D"])
    assert vis.dtype == torch.bool and int(vis.sum()) >= int((radii > 0).sum())


def test_fused_normalize_matches_torch_post_op(cuda_device, monkeypatch):
    """SURVEY 8f rank 1: the F.normalize post-op of diff_gauss/__init__.py:48 fused into the blend kernels gives the
    unit normal map and the gradients of the torch formulation (fp32 rounding apart)."""
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam = S.blob_scene(3000, seed=77), S.simple_camera(200, 120)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.1, 0.0, 0.3], device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=9)]
    results = {}
    for fused in (True, False):
        monkeypatch.setattr(diff_gauss, "FUSE_NORMALIZE", fused)
        leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
        m2d = torch.zeros((scene.P, 3), device=dev, requires_grad=True)
        rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, 0.1,
                                           torch.zeros(1, device=dev), bg, 1.0, d["viewmatrix"], d["projmatrix"], 3,
                                           d["campos"], False, False)
        color, depth, norm, alpha, radii, _ = GaussianRasterizer(rs)(
            leaves["means3D"], m2d, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
            rotations=leaves["rotations"])
        # only pixels some Gaussian reached: elsewhere the raw normal is exactly 0 and the adjoint multiplies by 1/eps
        w = (alpha.detach() > 0.02).float()
        ((norm * cot[2] * w).sum() + 0.1 * (color * cot[0]).sum() + 0.1 * (depth * cot[1]).sum()).backward()
        results[fused] = (norm.detach(), {k: v.grad.clone() for k, v in leaves.items()}, m2d.grad.clone())
    n_f, g_f, m_f = results[True]
    n_t, g_t, m_t = results[False]
    assert (n_f - n_t).abs().max().item() <= 2e-6
    covered = n_t.norm(dim=0) > 0.5
    assert bool(covered.any()) and bool(((n_f.norm(dim=0) - 1).abs() < 1e-5)[covered].all())
    for k in g_t:
        tol = 1e-5 + 2e-4 * g_t[k].abs().max().item()
        assert (g_f[k] - g_t[k]).abs().max().item() <= tol, k
    assert (m_f - m_t).abs().max().item() <= 1e-5 + 2e-4 * m_t.abs().max().item()


def test_two_phase_backward_equals_single_call(cuda_device):
    """Multi-GPU building block on one GPU: blend adjoint (phase 1) -> [P,16] sums -> per-Gaussian adjoint of two
    Gaussian slices (phase 2, each fed only its slice of the sums) reproduces the one-call backward."""
    dev = cuda_device
    scene, cam = S.blob_scene(5000, seed=91), S.simple_camera(256, 144)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.3, 0.2, 0.1], device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=4)]
    f = Hh.run_ours_forward(d, cam, 3, bg)
    ref = Hh.run_ours_backward(d, cam, 3, bg, f, cot)
    acc = Hh.run_ours_backward(d, cam, 3, bg, f, cot, phase=1)
    assert acc.shape == (scene.P, 16)
    # the fused reduce-scatter variant with a single "peer" (this GPU): same sums through the system-scope path
    acc_p = torch.zeros((scene.P, 16), device=dev)
    assert Hh.run_ours_backward(d, cam, 3, bg, f, cot, phase=1, acc_peers=[acc_p.data_ptr()], peer_slice=scene.P) is None
    assert (acc_p - acc).abs().max().item() <= 1e-5 + 2e-4 * acc.abs().max().item()
    # ... and with two "peers" that are the two halves of one buffer
    half = (scene.P + 1) // 2
    acc_q = torch.zeros((2 * half, 16), device=dev)
    Hh.run_ours_backward(d, cam, 3, bg, f, cot, phase=1, acc_peers=[acc_q.data_ptr(), acc_q[half:].data_ptr()],
                         peer_slice=half)
    assert (acc_q[:scene.P] - acc).abs().max().item() <= 1e-5 + 2e-4 * acc.abs().max().item()
    cut = 2173                                                   # deliberately not a multiple of the block span
    parts = [Hh.run_ours_backward(d, cam, 3, bg, f, cot, phase=2, acc=acc[a:b].clone(), gauss_range=(a, b))
             for a, b in ((0, cut), (cut, scene.P))]
    for k in ref:
        if ref[k].numel() == 0:
            continue
        got = torch.cat([parts[0][k][:cut], parts[1][k][cut:]], 0)
        assert got.shape == ref[k].shape
        tol = 1e-5 + 2e-4 * ref[k].abs().max().item()         # the sums themselves carry the reductions' order noise
        assert (got - ref[k]).abs().max().item() <= tol, k


def test_4k_frame_many_tiles_and_debug_mode(cuda_device):
    """3840x2160 = 32400 tiles: more than one pass of the single-CTA tile scan (8192 tiles per pass), ragged right
    and bottom edges; checked against the CPU oracle.  Also runs the per-stage synchronising debug mode."""
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene = S.blob_scene(20_000, seed=17, spread=3.0, scale=0.05)
    cam = S.simple_camera(3840, 2160, fov_deg=70.0, distance=6.0)
    bg = np.array([0.2, 0.1, 0.0], np.float32)
    d = Hh.to_torch(scene, cam, dev)
    f = Hh.run_ours_forward(d, cam, 3, torch.from_numpy(bg).to(dev))
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, 3, cam.viewmatrix,
                  cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg)
    assert f["num_rendered"] == o["num_rendered"] > 0 and np.array_equal(f["radii"].cpu().numpy(), o["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["ranges"].cpu().numpy().astype(np.uint32), o["ranges"])
    assert np.array_equal(it["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    for k in ("color", "depth", "alpha"):   # CPU libm expf vs CUDA expf: isolated 1/255-threshold flips are possible
        dlt = np.abs(f[k].cpu().numpy() - o[k])
        assert np.quantile(dlt, 0.9999) <= 1e-5 * max(1.0, float(np.abs(o[k]).max())), k
    # debug mode: every stage is followed by a synchronise + error check; results must not change
    from sfgs import rasterizer as R
    e = torch.empty(0, device=dev)
    g = R.rasterize_gaussians(torch.from_numpy(bg).to(dev), d["means3D"], e, d["opacities"], d["scales"], d["rotations"],
                              1.0, e, e, e, 0, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1,
                              cam.height, cam.width, d["shs"], 3, d["campos"], False, True)
    assert g[0] == f["num_rendered"] and torch.equal(g[1], f["color"]) and torch.equal(g[4], f["alpha"])
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=3)]
    b0 = Hh.run_ours_backward(d, cam, 3, torch.from_numpy(bg).to(dev), f, cot)
    b1 = Hh.run_ours_backward(d, cam, 3, torch.from_numpy(bg).to(dev), f, cot, debug=True)
    for k in b0:
        if b0[k].numel():
            assert (b0[k] - b1[k]).abs().max().item() <= 1e-5 + 2e-4 * b0[k].abs().max().item(), k


def test_mark_visible_matches_oracle(cuda_device):
    from oracle import cpu_oracle as O
    from sfgs import rasterizer as R
    dev = cuda_device
    scene, cam = S.blob_scene(5000, seed=61, spread=6.0), S.simple_camera(64, 64, distance=3.0)
    d = Hh.to_torch(scene, cam, dev)
    got = R.mark_visible(d["means3D"], d["viewmatrix"], d["projmatrix"]).cpu().numpy()
    want = O.mark_visible(scene.means3D, cam.viewmatrix)
    assert 0 < want.sum() < scene.P and np.array_equal(got, want)


def test_tile_row_bands_reassemble_the_frame(cuda_device):
    """Screen-space sharding on one GPU: bands rendered separately equal the full frame bit for bit, and the
    per-band partial gradients add up to the full gradient."""
    from sfgs import multigpu as MG
    from sfgs import rasterizer as R
    dev = cuda_device
    scene, cam = S.city_scene(120_000, seed=9, extent=120.0), S.jax004_camera(640, 360)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.1, 0.0, 0.2], device=dev)
    e = torch.empty(0, device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=2)]

    def fwd(band):
        return R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                     d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cam.height,
                                     cam.width, d["shs"], 3, d["campos"], False, False, tile_rows=band)

    def bwd(f, band):
        return R.rasterize_gaussians_backward(bg, d["means3D"], f[5], e, d["scales"], d["rotations"], e, 1.0, e, e,
                                              d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cot[0],
                                              cot[1], cot[2], cot[3], e, d["shs"], 3, d["campos"], f[7], f[0], f[8],
                                              f[9], f[4], False, tile_rows=band)

    full = fwd(None)
    gfull = bwd(full, None)
    it = Hh.our_internals(dict(zip(("num_rendered", "color", "depth", "norm", "alpha", "radii", "extra", "geom",
                                    "binning", "img"), full)), scene.P, cam.height, cam.width)
    rows, tiles_x = MG.tile_rows(cam.height), (cam.width + 15) // 16
    cuts = MG.partition_rows(MG.row_histogram(it["ranges"], tiles_x), 3)
    assert cuts[0] == 0 and cuts[-1] == rows
    total_R, acc = 0, None
    for g in range(3):
        band = (cuts[g], cuts[g + 1])
        f = fwd(band)
        y0, y1 = MG.band_pixel_rows(cuts, g, cam.height)
        for k in (1, 2, 3, 4):
            assert torch.equal(f[k][:, y0:y1], full[k][:, y0:y1]), (g, k)
        assert torch.equal(f[5], full[5])                 # radii report full-image visibility on every rank
        total_R += f[0]
        gb = bwd(f, band)
        acc = [x.clone() for x in gb] if acc is None else [a + x for a, x in zip(acc, gb)]
    assert total_R == full[0]
    for a, b, name in zip(acc, gfull, ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")):
        assert (a - b).abs().max().item() <= 1e-5 + 2e-4 * b.abs().max().item(), name


def test_config0_100k_gaussians_512_forward_vs_cpu_oracle(cuda_device):
    """BASELINE.json configs[0]: 100k synthetic Gaussians, one 512x512 pinhole camera, forward only, against the
    CPU restatement (the reference has no CPU path; the oracle is its plain-C port)."""
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene = S.blob_scene(100_000, seed=100, spread=3.0, scale=0.03)
    cam = S.simple_camera(512, 512, fov_deg=60.0, distance=9.0)
    bg = np.zeros(3, np.float32)
    d = Hh.to_torch(scene, cam, dev)
    f = Hh.run_ours_forward(d, cam, 3, torch.from_numpy(bg).to(dev))
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, 3, cam.viewmatrix,
                  cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg)
    assert f["num_rendered"] == o["num_rendered"] and np.array_equal(f["radii"].cpu().numpy(), o["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    assert np.array_equal(it["ranges"].cpu().numpy().astype(np.uint32), o["ranges"])
    for k in ("color", "depth", "norm", "alpha"):
        dlt = np.abs(f[k].cpu().numpy() - o[k])
        assert np.quantile(dlt, 0.9999) <= 1e-5 * max(1.0, float(np.abs(o[k]).max())), k


def test_training_loop_with_all_three_ops(cuda_device):
    """BASELINE.json configs[2] in miniature: distCUDA2 scale initialisation, then render -> L1 + fused-SSIM loss ->
    backward -> Adam for a few dozen iterations against images of a hidden synthetic scene; the loss must fall."""
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from fused_ssim import fused_ssim
    from simple_knn._C import distCUDA2
    dev = cuda_device
    target_scene = S.blob_scene(4000, seed=7, spread=1.5, scale=0.12)
    cams = [S.orbit_camera(target=(0, 0, 0), elevation_deg=30.0, azimuth_deg=a, radius=7.0, fov_deg=50.0, width=160,
                           height=128) for a in (0.0, 90.0, 180.0, 270.0)]
    bg = torch.zeros(3, device=dev)

    def render(params, cam):
        means, logs, rots, logit_o, shs = params
        rs = GaussianRasterizationSettings(cam.height, cam.width, cam.tanfovx, cam.tanfovy, 0.1,
                                           torch.zeros(1, device=dev), bg, 1.0,
                                           torch.from_numpy(cam.viewmatrix).to(dev), torch.from_numpy(cam.projmatrix).to(dev),
                                           3, torch.from_numpy(cam.campos).to(dev), False, False)
        m2d = torch.zeros_like(means, requires_grad=True)
        out = GaussianRasterizer(rs)(means, m2d, torch.sigmoid(logit_o), shs=shs, scales=torch.exp(logs),
                                     rotations=torch.nn.functional.normalize(rots))
        return out[0], m2d

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    with torch.no_grad():
        tp = (t(target_scene.means3D), torch.log(t(target_scene.scales)), t(target_scene.rotations),
              torch.logit(t(target_scene.opacities).clamp(1e-4, 1 - 1e-4)), t(target_scene.shs))
        targets = [render(tp, c)[0].clone() for c in cams]
    rng = np.random.default_rng(0)
    init_xyz = t((target_scene.means3D + rng.normal(0, 0.05, target_scene.means3D.shape)).astype(np.float32))
    d2 = distCUDA2(init_xyz).clamp_min(1e-7)
    params = [init_xyz.clone().requires_grad_(True),
              torch.log(torch.sqrt(d2))[:, None].repeat(1, 3).contiguous().requires_grad_(True),
              t(np.tile(np.array([1, 0, 0, 0], np.float32), (target_scene.P, 1))).requires_grad_(True),
              torch.full((target_scene.P, 1), -2.0, device=dev).requires_grad_(True),
              torch.zeros((target_scene.P, 16, 3), device=dev).requires_grad_(True)]
    opt = torch.optim.Adam([{"params": [params[0]], "lr": 2e-3}, {"params": [params[1]], "lr": 5e-3},
                            {"params": [params[2]], "lr": 1e-3}, {"params": [params[3]], "lr": 5e-2},
                            {"params": [params[4]], "lr": 2e-2}])
    losses = []
    for it in range(60):
        cam, gt = cams[it % 4], targets[it % 4]
        img, m2d = render(params, cam)
        loss = 0.8 * (img - gt).abs().mean() + 0.2 * (1.0 - fused_ssim(img[None], gt[None]))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        assert m2d.grad is not None and torch.isfinite(m2d.grad).all()
        assert all(torch.isfinite(p.grad).all() for p in params)
        opt.step()
        losses.append(loss.item())
    assert np.mean(losses[-8:]) < 0.7 * np.mean(losses[:4]), (losses[:4], losses[-8:])


# ----------------------------------------------------------------------------- the configurations that are benched
def _benched_config(name):
    """(scene, camera) of every frame bench.py reports a number on (BASELINE.json configs[1] and configs[3], plus the
    SURVEY 8d whole-scene orbit stress frame and the dense 5M variant the round-1 numbers were quoted on)."""
    if name == "configs1_1M_jax004":       # bench.py's headline frame, exactly
        return S.city_scene(1_000_000, seed=0), S.jax004_camera(1920, 1080)
    if name == "configs1_1M_orbit":        # SURVEY 8d second camera: fov 60, radius 300, elevation 85
        return S.city_scene(1_000_000, seed=0), S.orbit_camera(width=1920, height=1080)
    if name == "configs3_5M_jax004":       # SURVEY 8d config 4: same generator, extent x sqrt(5)
        return S.city_scene(5_000_000, seed=0, extent=256.0 * 5 ** 0.5), S.jax004_camera(1920, 1080)
    if name == "dense_5M_jax004":          # 5x the density of configs[1] in the same extent (long tile lists)
        return S.city_scene(5_000_000, seed=0), S.jax004_camera(1920, 1080)
    raise KeyError(name)


@pytest.mark.parametrize("name", ["configs1_1M_jax004", "configs1_1M_orbit", "configs3_5M_jax004", "dense_5M_jax004"])
def test_benched_configurations_vs_reference(cuda_device, name):
    """The frames bench.py times, diffed against the unmodified reference CUDA build at full size: every indexing
    quantity bit for bit (radii, tiles_touched, depth bits / means2D / conic, ranges, point_list, keys, n_contrib),
    the four images within 1e-5, all nine gradient tensors adjudicated by the float64 evaluation."""
    F = Hh.RefFacts(f"benched_{name}")
    dev = cuda_device
    scene, cam = _benched_config(name)
    d, bg_t, col, ours, ref = run_pair(scene, cam, dev, bg=(0.0, 0.0, 0.0), live=F.live)
    P, H, W = scene.P, cam.height, cam.width
    oi, ri = Hh.our_internals(ours, P, H, W), ref_internals(ref, P, H, W)
    check_indexing(F, ours, ref, oi, ri)
    vis = ours["radii"] > 0
    F.same("rgb", bits(oi["rgb"][vis]), lambda: bits(ri["rgb"][vis]))         # colours, hence clamp flags, bit for bit
    ours_clamped = torch.stack([(oi["clamped"] >> k) & 1 for k in range(3)], 1).bool()
    F.same("clamped", ours_clamped[vis], lambda: ri["clamped"][vis].bool())
    check_images(F, ours, ref)
    if F.live:
        oi = None          # the reference's intermediates feed the adjudicator; keep one set resident at 5M Gaussians
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=1)]      # bench.py's cotangents
    gb = Hh.run_ours_backward(d, cam, scene.sh_degree, bg_t, ours, cot)
    gbs = [gb] + [Hh.run_ours_backward(d, cam, scene.sh_degree, bg_t, ours, cot) for _ in range(2)]     # this library's reductions are unordered too
    F.adjudicate(d, cam, scene.sh_degree, bg_t, oi, ours["alpha"], ours["radii"], cot, gbs,
                 lambda: (ri, ref["alpha"], ref["radii"],
                          [Hh.run_ref_backward(d, cam, scene.sh_degree, bg_t, ref, cot) for _ in range(3)]), name)
    inv = ours["radii"] == 0
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        assert gb[k][inv].abs().max().item() == 0.0, k       # culled Gaussians get exact zeros


def test_long_thin_splats_crossing_many_tiles(cuda_device):
    """Needle-shaped splats (axis ratio up to 1:1000) hundreds of pixels long: the quadratic form of the conic
    cancels heavily far from the centre, which is where a block-level reach test could disagree with the reference's
    per-pixel `alpha < 1/255` test.  Indexing incl. n_contrib bit for bit, images 1e-5, gradients adjudicated."""
    dev = cuda_device
    rng = np.random.default_rng(7)
    scene = S.blob_scene(4000, seed=91, spread=2.0, scale=0.02)
    scene.scales[:, 0] = np.exp(rng.uniform(np.log(0.5), np.log(8.0), scene.P)).astype(np.float32)    # long axis
    scene.scales[:, 1] = np.exp(rng.uniform(np.log(0.002), np.log(0.02), scene.P)).astype(np.float32)  # needle
    scene.scales[:, 2] = scene.scales[:, 1]
    scene.opacities[:] = rng.uniform(0.004, 1.0, (scene.P, 1)).astype(np.float32)   # includes values near 1/255
    scene.opacities[::97] = np.float32(1.0) / np.float32(255.0)                      # exactly the threshold
    cam = S.simple_camera(640, 400, fov_deg=50.0, distance=9.0)
    for ks in (0.1, 0.0005):      # the second filter size leaves the conic nearly singular
        F = Hh.RefFacts(f"needles_k{ks}")
        d, bg_t, col, ours, ref = run_pair(scene, cam, dev, bg=(0.2, 0.1, 0.0), kernel_size=ks, live=F.live)
        P, H, W = scene.P, cam.height, cam.width
        oi, ri = Hh.our_internals(ours, P, H, W), ref_internals(ref, P, H, W)
        check_indexing(F, ours, ref, oi, ri, full=False)
        check_images(F, ours, ref)
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=12)]
        gb = Hh.run_ours_backward(d, cam, 3, bg_t, ours, cot, kernel_size=ks)
        gbs = [gb] + [Hh.run_ours_backward(d, cam, 3, bg_t, ours, cot, kernel_size=ks) for _ in range(2)]     # this library's reductions are unordered too
        F.adjudicate(d, cam, 3, bg_t, oi, ours["alpha"], ours["radii"], cot, gbs,
                     lambda: (ri, ref["alpha"], ref["radii"],
                              [Hh.run_ref_backward(d, cam, 3, bg_t, ref, cot, kernel_size=ks) for _ in range(3)]),
                     f"needles[k={ks}]", kernel_size=ks)


def test_alternating_frame_sizes_do_not_rerun_the_forward(cuda_device):
    """A training loop alternates 1080p train views, 1024^2 pseudo-views and small evaluation renders of one scene.  The
    binning-capacity estimate is kept per (device, P, width, height, band): after one frame of each size nothing
    overflows any more, whichever order the sizes come in (a single process-wide estimate re-ran the whole forward
    on every switch to a larger frame)."""
    from sfgs import native as N
    dev = cuda_device
    scene = S.city_scene(200_000, seed=5)
    cams = [S.jax004_camera(1920, 1080), S.orbit_camera(width=1024, height=1024), S.orbit_camera(width=512, height=512),
            S.jax004_camera(640, 360)]
    ds = [Hh.to_torch(scene, c, dev) for c in cams]
    bg = torch.zeros(3, device=dev)
    ref_R = []
    for d, c in zip(ds, cams):                                   # warm-up: one frame of each size
        ref_R.append(Hh.run_ours_forward(d, c, 3, bg)["num_rendered"])
    before = N.lib().sfgs_overflow_reruns()
    order = [0, 1, 2, 3, 2, 0, 3, 1, 0, 2, 1, 3, 0, 0, 1, 1]
    for i in order:
        f = Hh.run_ours_forward(ds[i], cams[i], 3, bg)
        assert f["num_rendered"] == ref_R[i]
    assert N.lib().sfgs_overflow_reruns() == before, "a frame size that had been seen before overflowed its binning estimate"


def test_prefiltered_and_empty_band_semantics(cuda_device):
    """`prefiltered=True` promises that no Gaussian fails the frustum test; the reference traps the kernel when one does
    (CR/auxiliary.h:157-161) — here the call reports an argument error.  A tile-row band with begin == end != 0 is EMPTY
    (more ranks than tile rows): nothing is binned or blended, unlike (0, 0), which means the whole image."""
    from sfgs import native as N
    from sfgs import rasterizer as R
    dev = cuda_device
    e = torch.empty(0, device=dev)
    bg = torch.zeros(3, device=dev)
    scene, cam = S.blob_scene(800, seed=3, spread=1.0), S.simple_camera(96, 64)     # camera 8 units away: all in front
    d = Hh.to_torch(scene, cam, dev)
    vz = d["means3D"] @ d["viewmatrix"][:3, 2] + d["viewmatrix"][3, 2]
    assert float(vz.min()) > 0.2

    def fwd(means, prefiltered=False, tile_rows=None):
        return R.rasterize_gaussians(bg, means, e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                     d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cam.height, cam.width,
                                     d["shs"], 3, d["campos"], prefiltered, False, tile_rows=tile_rows)
    full = fwd(d["means3D"])
    # every Gaussian of this scene is in front of the camera: prefiltered=True is legal and changes nothing
    ok = fwd(d["means3D"], prefiltered=True)
    assert ok[0] == full[0] and torch.equal(ok[1], full[1])
    behind = d["means3D"].clone()
    behind[::7, 2] -= 100.0
    with pytest.raises(N.SfgsError, match="prefiltered"):
        fwd(behind, prefiltered=True)
    assert fwd(behind)[0] > 0                                   # without the promise the same input simply culls them
    # empty band
    rows = (cam.height + 15) // 16
    empty = fwd(d["means3D"], tile_rows=(2, 2))
    assert empty[0] == 0 and torch.equal(empty[5], full[5])     # nothing binned; radii still report full-image visibility
    whole = fwd(d["means3D"], tile_rows=(0, rows + 5))          # end beyond the grid is clamped
    assert whole[0] == full[0] and torch.equal(whole[1], full[1])
