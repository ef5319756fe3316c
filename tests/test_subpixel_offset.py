"""Subpixel offsets (GaussianRasterizationSettings.subpixel_offset, Mip-Splatting's ray jitter): pixel (x, y) samples
the splats at (x + off[y,x,0], y + off[y,x,1]).  CPU: the dilated reach mask restated in numpy, the C ABI's and the
Python layers' argument checks, and the reference's own render() on the opt-in switch.  GPU: zero offsets against the
default call, integer offsets against shifted default renders, fractional offsets against the CPU oracle and the
float64 adjudicator, the deterministic and two-phase backwards, the unpacked key path, non-finite offsets and the
autograd layer."""
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import helpers as Hh
import subpixel_oracle as SO
from sfgs import synthetic as S
from test_reach_mask_cpu import blended_blocks, random_conic, reach_mask_np

f32 = np.float32
SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")


# ----------------------------------------------------------------------------- CPU: the dilated reach mask
def reach_mask_dilated_np(mx, my, A, B, C_, opac, tile_px, tile_py, ex, ey):
    """csrc/sfgs_common.cuh reach_mask_t<true> in float32: the block rectangles grow by (ex, ey), and so do Xm, Ym."""
    mx, my, A, B, C_, opac, ex, ey = map(f32, (mx, my, A, B, C_, opac, ex, ey))
    if not (opac >= f32(1.0 / 255.0)):
        return 0
    det = A * C_ - B * B
    if not (A > 0 and C_ > 0 and det > 0):
        return 0xFF
    xr, yr = mx - f32(tile_px), my - f32(tile_py)
    Xm = max(abs(xr), abs(xr - f32(15))) + ex
    Ym = max(abs(yr), abs(yr - f32(15))) + ey
    thr = f32(2.004) * np.log(opac * f32(255.0), dtype=f32) + f32(0.05) + f32(1e-5) * (A * Xm * Xm + f32(2) * abs(B) * Xm * Ym + C_ * Ym * Ym)
    invA, invC = f32(1) / A, f32(1) / C_
    cols = [xr - f32((k >> 1) * 8 + (k & 1) * 7) for k in range(4)]
    cols = [X - ex if k & 1 else X + ex for k, X in enumerate(cols)]
    rows = [yr - f32((j >> 1) * 4 + (j & 1) * 3) for j in range(8)]
    rows = [Y - ey if j & 1 else Y + ey for j, Y in enumerate(rows)]
    AX2 = [A * X * X for X in cols]; BX2 = [f32(2) * B * X for X in cols]; yc = [-B * X * invC for X in cols]
    CY2 = [C_ * Y * Y for Y in rows]; BY2 = [f32(2) * B * Y for Y in rows]; xc = [-B * Y * invA for Y in rows]
    mask = 0
    for by in range(4):
        yhi = yr - f32(4 * by); ylo = yhi - f32(3)
        yhi, ylo = yhi + ey, ylo - ey
        for bx in range(2):
            xhi = xr - f32(8 * bx); xlo = xhi - f32(7)
            xhi, xlo = xhi + ex, xlo - ex
            inside = ylo <= 0 <= yhi and xlo <= 0 <= xhi
            y0 = min(max(yc[2 * bx], ylo), yhi); y1 = min(max(yc[2 * bx + 1], ylo), yhi)
            q0 = (C_ * y0 + BX2[2 * bx]) * y0 + AX2[2 * bx]
            q1 = (C_ * y1 + BX2[2 * bx + 1]) * y1 + AX2[2 * bx + 1]
            x0 = min(max(xc[2 * by], xlo), xhi); x1 = min(max(xc[2 * by + 1], xlo), xhi)
            q2 = (A * x0 + BY2[2 * by]) * x0 + CY2[2 * by]
            q3 = (A * x1 + BY2[2 * by + 1]) * x1 + CY2[2 * by + 1]
            if inside or not (min(q0, q1, q2, q3) > thr):
                mask |= 1 << (by * 2 + bx)
    return mask


def jittered_blocks(mx, my, A, B, C_, opac, tile_px, tile_py, e, rng, n=6):
    """Bit per block that holds a pixel which blends the splat at some sample within +-e of its centre: the corners
    and edge midpoints of the square and n random points, each through the reference's float32 expression."""
    pts = [(sx * e, sy * e) for sx in (-1, 0, 1) for sy in (-1, 0, 1)] + [tuple(rng.uniform(-e, e, 2)) for _ in range(n)]
    need = 0
    for ox, oy in pts:
        px = (np.arange(16, dtype=f32) + f32(tile_px))[None, :] + f32(ox)
        py = (np.arange(16, dtype=f32) + f32(tile_py))[:, None] + f32(oy)
        dx, dy = f32(mx) - px, f32(my) - py
        power = f32(-0.5) * (f32(A) * dx * dx + f32(C_) * dy * dy) - f32(B) * dx * dy
        alpha = np.minimum(f32(0.99), f32(opac) * np.exp(power, dtype=f32))
        hit = (power <= 0) & (alpha >= f32(1.0 / 255.0))
        for by in range(4):
            for bx in range(2):
                if hit[4 * by:4 * by + 4, 8 * bx:8 * bx + 8].any():
                    need |= 1 << (by * 2 + bx)
    return need


@pytest.mark.parametrize("e", [0.0, 0.25, 0.5, 1.0, 3.0])
@pytest.mark.parametrize("kind", ["round", "elongated", "needle"])
def test_dilated_reach_mask_never_drops_a_jittered_sample(kind, e):
    rng = np.random.default_rng({"round": 1, "elongated": 2, "needle": 3}[kind] * 100 + int(4 * e))
    dropped = 0
    for _ in range(200):
        A, B, C_ = random_conic(rng, kind)
        opac = float(rng.choice([rng.uniform(0.004, 0.02), rng.uniform(0.02, 1.0)]))
        tile_px, tile_py = 16 * int(rng.integers(0, 120)), 16 * int(rng.integers(0, 68))
        reach = 40.0 if kind != "needle" else 700.0
        mx, my = tile_px + 8 + rng.uniform(-reach, reach), tile_py + 8 + rng.uniform(-reach, reach)
        m = reach_mask_dilated_np(mx, my, A, B, C_, opac, tile_px, tile_py, e, e)
        if e == 0.0:
            assert m == reach_mask_np(mx, my, A, B, C_, opac, tile_px, tile_py)
            need = blended_blocks(mx, my, A, B, C_, opac, tile_px, tile_py)
        else:
            need = jittered_blocks(mx, my, A, B, C_, opac, tile_px, tile_py, e, rng)
        assert need & ~m == 0, (kind, e, mx, my, A, B, C_, opac, tile_px, tile_py, bin(m), bin(need))
        dropped += bin(0xFF & ~m).count("1")
    assert dropped > 0


# ----------------------------------------------------------------------------- CPU: argument checks
def test_abi_rejects_unsupported_combinations_before_cuda_work():
    from sfgs import native as N
    L = N.lib()
    dummy = (C.c_float * 64)()
    ptr = C.cast(dummy, C.c_void_p)
    off = ptr
    a = N.ForwardArgs()
    a.P, a.width, a.height, a.ED = 8, 32, 32, 2
    assert L.sfgs_rasterize_forward_subpixel(C.byref(a), off) == SFGS_E_UNSUPPORTED and "extra_attrs" in N.last_error()
    a.ED = 0
    peers = (C.c_void_p * 1)(ptr)
    a.out_peers, a.n_out_peers = C.cast(peers, C.POINTER(C.c_void_p)), 1
    assert L.sfgs_rasterize_forward_subpixel(C.byref(a), off) == SFGS_E_UNSUPPORTED and "out_peers" in N.last_error()
    assert L.sfgs_rasterize_forward_subpixel(None, off) == SFGS_E_BADARG
    for fn in (L.sfgs_rasterize_backward_subpixel, L.sfgs_rasterize_backward_deterministic_subpixel):
        b = N.BackwardArgs()
        b.P, b.width, b.height, b.ED = 8, 32, 32, 2
        assert fn(C.byref(b), off) == SFGS_E_UNSUPPORTED and "extra_attrs" in N.last_error()
        b.ED, b.phase, b.acc = 0, 1, ptr
        b.acc_peers, b.n_peers, b.peer_slice = C.cast(peers, C.POINTER(C.c_void_p)), 1, 8
        assert fn(C.byref(b), off) == SFGS_E_UNSUPPORTED and "acc_peers" in N.last_error()
        assert fn(None, off) == SFGS_E_BADARG


@pytest.mark.parametrize("bad", ["cpu", "dtype", "shape"])
def test_python_layer_rejects_bad_offsets(bad):
    from sfgs import rasterizer as R
    H, W = 6, 5
    t = {"cpu": torch.zeros(H, W, 2), "dtype": torch.zeros(H, W, 2, dtype=torch.float64),
         "shape": torch.zeros(W, H, 2)}[bad]
    if bad != "cpu" and torch.cuda.is_available():
        t = t.cuda()
    z = torch.zeros
    with pytest.raises(ValueError, match="subpixel_offset"):
        R.rasterize_gaussians(z(3), z(4, 3), z(0), z(4, 1), z(4, 3), z(4, 4), 1.0, z(0), z(0), z(0), 0, z(4, 4), z(4, 4),
                              1.0, 1.0, 0.1, H, W, z(4, 16, 3), 3, z(3), False, False, subpixel_offset=t)
    img = z(3, H, W)
    with pytest.raises(ValueError, match="subpixel_offset"):
        R.rasterize_gaussians_backward(z(3), z(4, 3), z(4, dtype=torch.int32), z(0), z(4, 3), z(4, 4), z(0), 1.0, z(0),
                                       z(0), z(4, 4), z(4, 4), 1.0, 1.0, 0.1, img, z(1, H, W), img, z(1, H, W), z(0),
                                       z(4, 16, 3), 3, z(3), z(1), 1, z(1), z(1), z(1, H, W), False,
                                       subpixel_offset=t)


# ----------------------------------------------------------------------------- CPU: the offset oracle itself
def _oracle_pair(off_fn):
    from oracle import cpu_oracle as O
    scene, cam = S.blob_scene(800, seed=7), S.simple_camera(70, 45)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    args = (scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, 3, cam.viewmatrix, cam.projmatrix,
            cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg)
    off = np.zeros((cam.height, cam.width, 2), np.float32)
    off_fn(off)
    return O, O.forward(*args), SO.cpu_forward(*args, subpixel_offset=off), cam


def test_offset_oracle_with_zero_offsets_is_the_oracle():
    O, o0, o1, cam = _oracle_pair(lambda off: None)
    for k in ("color", "depth", "norm", "alpha", "n_contrib"):
        assert np.array_equal(o0[k].view(np.uint32), o1[k].view(np.uint32)), k
    cot = S.cotangents(cam.width, cam.height, seed=3)
    g0, g1 = O.backward(o0, *cot), SO.cpu_backward(o1, *cot)
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        # the same sums; only the order of the OpenMP atomics differs (the scale chain amplifies it to a few 1e-6)
        assert np.abs(g0[k] - g1[k]).max() <= 1e-5 * (1 + np.abs(g0[k]).max()), k


def test_offset_oracle_with_an_integer_offset_is_the_shifted_oracle():
    O, o0, o1, cam = _oracle_pair(lambda off: off.__setitem__((Ellipsis, 0), 1.0))
    H, W = cam.height, cam.width
    x = np.arange(W)
    ok = (x + 1 < W) & ((x + 1) // 16 == x // 16)           # the sample pixel lies in the image and in the same tile
    for k in ("color", "depth", "norm", "alpha"):
        assert np.array_equal(o1[k][:, :, ok], o0[k][:, :, np.flatnonzero(ok) + 1]), k


# ----------------------------------------------------------------------------- CPU: the reference's render()
from test_reference_caller import _camera, _fill, needs_reference, reference_stack  # noqa: E402,F401


@needs_reference
@pytest.mark.parametrize("on", [True, False])
def test_reference_render_forwards_offsets_only_when_opted_in(reference_stack, monkeypatch, on):
    import diff_gauss
    from diff_gauss import _C
    render, GaussianModel, rec = reference_stack
    seen = {"fwd": [], "bwd": []}

    def recording(fn, key):
        def call(*a, subpixel_offset=None, **kw):
            seen[key].append(subpixel_offset)
            return fn(*a, **kw)
        return call
    for name, key in (("rasterize_gaussians", "fwd"), ("rasterize_gaussians_fused", "fwd"),
                      ("rasterize_gaussians_backward", "bwd"), ("rasterize_gaussians_backward_fused", "bwd")):
        monkeypatch.setattr(_C, name, recording(getattr(_C, name), key))
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", on)
    pc = GaussianModel(3, False, 4, 32)
    _fill(pc, 200, False)
    cam = _camera()
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False, convert_SHs_python=False)
    off = torch.rand((48, 80, 2)) - 0.5
    out = render(cam, pc, pipe, torch.zeros(3), kernel_size=0.1, subpixel_offset=off)
    out["render"].mean().backward()
    assert len(seen["fwd"]) == 1 and len(seen["bwd"]) == 1
    if on:
        assert seen["fwd"][0] is not None and torch.equal(seen["fwd"][0], off) and seen["bwd"][0] is seen["fwd"][0]
    else:
        assert seen["fwd"] == [None] and seen["bwd"] == [None]


# ----------------------------------------------------------------------------- GPU helpers
def inst_masks(f, W, H):
    """The reach mask of every sorted instance (BinningLayout: point_list, then inst_mask)."""
    hdr = f["img"][:32].view(torch.int32).cpu().numpy().astype(np.uint32)
    cap = int(hdr[2]) | (int(hdr[3]) << 32)
    base = (f["binning"].data_ptr() + 255) & ~255
    off = base - f["binning"].data_ptr() + ((cap * 4 + 255) & ~255)
    return f["binning"][off:off + f["num_rendered"]].clone()


def _close(a, b, k, extra=0.0):
    a, b = a.double(), b.double()
    err, tol = (a - b).abs().max().item(), 1e-4 + 2e-4 * b.abs().max().item() + extra
    assert err <= tol, (k, err, tol)


def _scene(name, dev):
    if name == "blob":
        scene, cam = S.blob_scene(2500, seed=41), S.simple_camera(190, 150)
    elif name == "city":
        scene, cam = S.city_scene(300_000, seed=3), S.jax004_camera(1920, 1080)
    else:
        scene, cam = S.city_scene(60_000, seed=9, extent=120.0), S.jax004_camera(640, 360)
    return scene, cam, Hh.to_torch(scene, cam, dev)


# ----------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["blob", "city"])
def test_zero_offsets_equal_the_default_call(cuda_device, name):
    dev = cuda_device
    scene, cam, d = _scene(name, dev)
    bg = torch.tensor([0.3, 0.1, 0.2], device=dev)
    H, W = cam.height, cam.width
    zero = torch.zeros((H, W, 2), device=dev)
    f0, f1 = Hh.run_ours_forward(d, cam, 3, bg), Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=zero)
    for k in ("color", "depth", "norm", "alpha", "radii"):
        assert torch.equal(Hh.bits(f0[k]), Hh.bits(f1[k])), k
    i0, i1 = Hh.our_internals(f0, scene.P, H, W), Hh.our_internals(f1, scene.P, H, W)
    for k in ("n_contrib", "point_list", "ranges", "keys"):
        assert torch.equal(i0[k], i1[k]), k
    assert torch.equal(inst_masks(f0, W, H), inst_masks(f1, W, H))
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=6)]
    # the ill-conditioned covariance / rotation gradients of the 1080p frame differ between two calls of the default
    # backward itself (unordered reductions) by about the bound: that spread is allowed on top of it
    ga, gb = Hh.run_ours_backward(d, cam, 3, bg, f0, cot), Hh.run_ours_backward(d, cam, 3, bg, f0, cot)
    spread = {k: (ga[k].double() - gb[k].double()).abs().max().item() for k in GRAD_KEYS}
    for det in (False, True):
        g0 = Hh.run_ours_backward(d, cam, 3, bg, f0, cot, det=det)
        g1 = Hh.run_ours_backward(d, cam, 3, bg, f1, cot, subpixel_offset=zero, det=det)
        for k in GRAD_KEYS:
            _close(g1[k], g0[k], (k, det), extra=2.0 * spread[k])


def _shift_case(dev, name, ox, oy, det_grads=True):
    scene, cam, d = _scene(name, dev)
    bg = torch.tensor([0.3, 0.1, 0.2], device=dev)
    H, W = cam.height, cam.width
    off = torch.empty((H, W, 2), device=dev)
    off[..., 0], off[..., 1] = float(ox), float(oy)
    f0, f1 = Hh.run_ours_forward(d, cam, 3, bg), Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
    assert torch.equal(f0["radii"], f1["radii"])
    y, x = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    sx, sy = x + ox, y + oy
    ok = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H) & (sx // 16 == x // 16) & (sy // 16 == y // 16)
    assert ok.sum() > 0.5 * H * W * (1 - abs(ox) / 16) * (1 - abs(oy) / 16)
    src = (sy.clamp(0, H - 1) * W + sx.clamp(0, W - 1))[ok]
    for k in ("color", "depth", "norm", "alpha"):
        a = f1[k].reshape(f1[k].shape[0], -1)[:, ok.flatten()]
        b = f0[k].reshape(f0[k].shape[0], -1)[:, src]
        assert torch.equal(Hh.bits(a), Hh.bits(b)), (k, ox, oy)
    n0 = Hh.our_internals(f0, scene.P, H, W)["n_contrib"]
    n1 = Hh.our_internals(f1, scene.P, H, W)["n_contrib"]
    assert torch.equal(n1[ok.flatten()], n0[src]), (ox, oy)
    if not det_grads:
        return
    # cotangent zero outside the compared pixels; the default call sees it at the sample pixels
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=8)]
    cot1 = [c * ok for c in cot]
    cot0 = [torch.zeros_like(c) for c in cot]
    for c0, c1 in zip(cot0, cot1):
        c0.view(c0.shape[0], -1)[:, src] = c1.view(c1.shape[0], -1)[:, ok.flatten()]
    g1 = Hh.run_ours_backward(d, cam, 3, bg, f1, cot1, subpixel_offset=off, det=True)
    g0 = Hh.run_ours_backward(d, cam, 3, bg, f0, cot0, det=True)
    for k in GRAD_KEYS:
        _close(g1[k], g0[k], (k, ox, oy))


@pytest.mark.gpu
@pytest.mark.parametrize("ox,oy", [(1, 0), (-1, 0), (0, 1), (0, -1), (2, -3)])
@pytest.mark.parametrize("name", ["blob", "banded"])
def test_integer_offsets_reproduce_shifted_renders(cuda_device, name, ox, oy):
    _shift_case(cuda_device, name, ox, oy)


@pytest.mark.gpu
def test_unpacked_key_path_with_offsets(cuda_device):
    """The masks of the unpacked key layout (P >= 2^24, forced here with SFGS_KEYS_PACKED=0, read once per process)
    come from the dilated sort kernels: the shifted-render test in a child process."""
    env = dict(os.environ, SFGS_KEYS_PACKED="0")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-k",
                        "integer_offsets and blob"], env=env, capture_output=True, text=True, timeout=900,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


def _oracle_cases():
    yield "blob", S.blob_scene(2500, seed=41), S.simple_camera(190, 150), 3
    for seed in range(5):
        rng = np.random.default_rng(5000 + seed)
        P = int(rng.integers(200, 4000))
        W, H = int(rng.integers(17, 300)) | 1, int(rng.integers(17, 200)) | 1
        scene = S.blob_scene(P, seed=300 + seed, sh_degree=3, spread=float(rng.uniform(0.3, 2.0)),
                             scale=float(rng.uniform(0.02, 0.3)))
        yield f"rand{seed}", scene, S.simple_camera(W, H, fov_deg=float(rng.uniform(40, 80))), seed % 4


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["blob"] + [f"rand{s}" for s in range(5)])
def test_fractional_offsets_against_cpu_oracle(cuda_device, case):
    dev = cuda_device
    _, scene, cam, deg = next(c for c in _oracle_cases() if c[0] == case)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    bg_t = torch.from_numpy(bg).to(dev)
    d = Hh.to_torch(scene, cam, dev)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, 17)
    f = Hh.run_ours_forward(d, cam, deg, bg_t, subpixel_offset=off)
    o = SO.cpu_forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, deg, cam.viewmatrix,
                       cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg,
                       subpixel_offset=off.cpu().numpy())
    assert np.array_equal(f["radii"].cpu().numpy(), o["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    assert np.array_equal(it["ranges"].cpu().numpy().astype(np.uint32), o["ranges"])
    for k in ("color", "depth", "norm", "alpha"):
        assert np.abs(f[k].cpu().numpy() - o[k]).max() <= 5e-5, k
    cot = S.cotangents(cam.width, cam.height, seed=6)
    gb = Hh.run_ours_backward(d, cam, deg, bg_t, f, [torch.from_numpy(c).to(dev) for c in cot], subpixel_offset=off)
    og = SO.cpu_backward(o, *cot)
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        a, b = gb[k].cpu().numpy().astype(np.float64), og[k].astype(np.float64)
        assert np.abs(a - b).max() <= 1e-4 + 2e-4 * np.abs(b).max(), k


@pytest.mark.gpu
def test_fractional_offsets_adjudicated_in_float64(cuda_device):
    """1080p, 300k Gaussians, U(-0.5, 0.5): the error of this library's gradients against the float64 adjudicator with
    the same offsets stays within {mean 1.5, p99.9 2, max 8} times its own error without offsets on the same frame."""
    from oracle import adjudicator as A
    dev = cuda_device
    scene, cam, d = _scene("city", dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    H, W = cam.height, cam.width
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=4)]
    rep = {}
    for tag, off in (("plain", None), ("jitter", Hh.uniform_offsets(H, W, dev, 23))):
        f = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
        runs = [Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off) for _ in range(3)]
        I = Hh.our_internals(f, scene.P, H, W)
        args = (I, d["means3D"], f["radii"], d["shs"], d["scales"], d["rotations"], 1.0, d["viewmatrix"],
                d["projmatrix"], d["campos"], cam.tanfovx, cam.tanfovy, 0.1, 3, bg, f["alpha"], cot)
        g64 = A.backward_f64(*args) if off is None else SO.backward_f64(*args, subpixel_offset=off)
        rep[tag] = A.error_report(runs, None, g64, keys=A.GRAD_KEYS)
    factors = {"mean": 1.5, "p999": 2.0, "max": 8.0}
    for k in A.GRAD_KEYS:
        for m, fac in factors.items():
            got, base = rep["jitter"][k]["ours"][m], rep["plain"][k]["ours"][m]
            assert got <= fac * base + 1e-7, (k, m, got, base)


@pytest.mark.gpu
def test_deterministic_backward_with_offsets(cuda_device):
    dev = cuda_device
    scene, cam, d = _scene("banded", dev)
    bg = torch.tensor([0.3, 0.1, 0.2], device=dev)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, 5)
    f = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=3)]
    a, b = (Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, det=True) for _ in range(2))
    g = Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off)
    for k in GRAD_KEYS:
        assert torch.equal(Hh.bits(a[k]), Hh.bits(b[k])), k
        _close(a[k], g[k], k)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
def test_two_phase_backward_with_offsets(cuda_device, det):
    dev = cuda_device
    scene, cam = S.blob_scene(5000, seed=91), S.simple_camera(256, 144)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.3, 0.2, 0.1], device=dev)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, 9)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=4)]
    f = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
    one = Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, det=det)
    acc = Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, det=det, phase=1)
    cut = 2173
    parts = [Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, det=det, phase=2, acc=acc[a:b].clone(),
                                  gauss_range=(a, b)) for a, b in ((0, cut), (cut, scene.P))]
    for k in GRAD_KEYS:
        got = torch.cat([parts[0][k][:cut], parts[1][k][cut:]], 0)
        if det:
            assert torch.equal(Hh.bits(got), Hh.bits(one[k])), k
        else:
            _close(got, one[k], k)


@pytest.mark.gpu
def test_non_finite_offset_is_rejected(cuda_device):
    from sfgs.native import SfgsError
    dev = cuda_device
    scene, cam, d = _scene("blob", dev)
    bg = torch.zeros(3, device=dev)
    f0 = Hh.run_ours_forward(d, cam, 3, bg)
    for bad in (float("nan"), float("inf")):
        off = torch.zeros((cam.height, cam.width, 2), device=dev)
        off[17, 33, 1] = bad
        with pytest.raises(SfgsError, match="NaN or Inf"):
            Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
    f1 = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=torch.zeros((cam.height, cam.width, 2), device=dev))
    assert torch.equal(Hh.bits(f0["color"]), Hh.bits(f1["color"]))


@pytest.mark.gpu
def test_autograd_layer(cuda_device, monkeypatch):
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    dev = cuda_device
    scene, cam, d = _scene("blob", dev)
    H, W = cam.height, cam.width
    bg = torch.tensor([0.3, 0.1, 0.2], device=dev)
    off = Hh.uniform_offsets(H, W, dev, 31)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=2)]

    def run(o):
        rs = GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, 0.1, o, bg, 1.0, d["viewmatrix"],
                                           d["projmatrix"], 3, d["campos"], False, False)
        leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        m2d = torch.zeros((scene.P, 3), device=dev, requires_grad=True)
        out = GaussianRasterizer(rs)(leaves["means3D"], m2d, leaves["opacities"], shs=leaves["shs"],
                                     scales=leaves["scales"], rotations=leaves["rotations"])
        loss = sum((o_ * c).sum() for o_, c in zip((out[0], out[1], out[2], out[3]), cot))
        loss.backward()
        return out, dict({k: v.grad for k, v in leaves.items()}, means2D=m2d.grad)

    monkeypatch.setattr(diff_gauss, "FUSE_NORMALIZE", True)
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", True)
    out_j, g_j = run(off)
    # the same through the native calls
    from sfgs import rasterizer as R
    e = torch.empty(0, device=dev)
    nat = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"], 3,
                                d["campos"], False, False, fuse_normalize=True, subpixel_offset=off)
    for a, b in zip(out_j[:4], nat[1:5]):
        assert torch.equal(Hh.bits(a), Hh.bits(b))
    out_p, g_p = run(torch.zeros(1, device=dev))      # a placeholder: the default result
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", False)
    out_d, g_d = run(off)                             # switch off: offsets ignored
    out_0, g_0 = run(torch.zeros((H, W, 2), device=dev))
    for a, b, c in zip(out_p[:4], out_d[:4], out_0[:4]):
        assert torch.equal(Hh.bits(a), Hh.bits(c)) and torch.equal(Hh.bits(b), Hh.bits(c))
    assert not torch.equal(Hh.bits(out_j[0]), Hh.bits(out_d[0]))
    for k in g_0:
        _close(g_p[k], g_0[k], k)
        _close(g_d[k], g_0[k], k)
    # the jittered gradients equal the native _subpixel backward's
    f = dict(zip(Hh.FWD_KEYS, nat[:10]))
    gn = Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, norm_raw=nat[10])
    for k, kn in (("means3D", "means3D"), ("shs", "sh"), ("opacities", "opacity"), ("scales", "scales"),
                  ("rotations", "rot"), ("means2D", "means2D")):
        _close(g_j[k], gn[kn], k)
