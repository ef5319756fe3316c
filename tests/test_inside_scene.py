"""The rasterizer with the camera inside the scene: Gaussians at the 0.2 near plane, beside the camera beyond the
guard band of the projection's Jacobian, splats that fill the screen, and centres far off screen whose rectangles
still reach the image.  Skyfall-GS's later stages render low-altitude views from among the Gaussians, so training
reaches all of these; a view from outside the scene reaches almost none of them.

  - CPU: the preprocess's conservative pre-cull (csrc/sfgs_preprocess.cu, radius_bound and phase A) restated in numpy
    float32 next to the exact projection it stands in front of (cov2d_project, lambda_1, ceil, tile_rect).  The cull
    may only drop a Gaussian whose exact tile rectangle is empty.
  - GPU: street-level views of the city, a camera inside a blob, a crafted frame at the near plane and the guard band,
    and the same frame with precomputed (also indefinite) covariances, against the reference CUDA build
    (helpers.RefFacts: live where its build is present, else the recorded facts) and the CPU oracle; the sort size
    classes the street view reaches, the deterministic and two-phase backward, and the binning capacity growing from a
    far view to a near one.
"""
import math

import numpy as np
import pytest
import torch

import helpers as Hh
from helpers import bits, release_cached_frames  # noqa: F401
from sfgs import synthetic as S
from test_gpu_parity import check_images, check_indexing, ref_internals

f32 = np.float32
TILE = 16


# ============================================================================ float32 restatement of the preprocess
def _to_int(x):
    """C's float -> int conversion on the GPU (cvt.rzi.s32.f32): truncate, saturate, NaN -> 0."""
    x = np.asarray(x, np.float64)
    return np.where(np.isnan(x), 0, np.clip(np.trunc(np.nan_to_num(x, nan=0.0)), -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def tile_rect_np(px, py, radius, gx, gy):
    """sfgs_common.cuh::tile_rect: (int)((p -/+ r (+ 15)) / 16) clamped to the grid, in float32."""
    r = np.asarray(radius).astype(f32)
    x0 = np.clip(_to_int((px - r) / f32(TILE)), 0, gx)
    y0 = np.clip(_to_int((py - r) / f32(TILE)), 0, gy)
    x1 = np.clip(_to_int((px + r + f32(TILE) - f32(1)) / f32(TILE)), 0, gx)
    y1 = np.clip(_to_int((py + r + f32(TILE) - f32(1)) / f32(TILE)), 0, gy)
    return x0, y0, x1, y1


def _ndc_to_pix(v, S_):
    return (((v.astype(np.float64) + 1.0) * S_ - 1.0) * 0.5).astype(f32)


def _project(means, vm, pm, W, H):
    px, py, pz = (means[:, i].astype(f32) for i in range(3))
    view_z = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14]
    hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12]
    hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13]
    hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15]
    p_w = f32(1) / (hw + f32(1e-7))
    return view_z, _ndc_to_pix(hx * p_w, W), _ndc_to_pix(hy * p_w, H)


def _rot(q):
    """rot_from_quat: R[:, c, k] (column c, row k) of the un-normalised quaternion (r, x, y, z)."""
    r, x, y, z = (q[:, i].astype(f32) for i in range(4))
    R = np.empty((q.shape[0], 3, 3), f32)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - r * z); R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y); R[:, 2, 1] = 2 * (y * z + r * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def cov3d_np(scales, rots, mod):
    """cov3d_from_scale_rot: Sigma = M M^T with M[c, k] = mod s_k R[c, k]; upper triangle c0..c5."""
    M = _rot(rots) * (f32(mod) * scales.astype(f32))[:, None, :]
    Sg = np.einsum("nrk,nck->nrc", M, M).astype(f32)
    return np.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1)


def _camera_consts(cam):
    tanx, tany = f32(cam.tanfovx), f32(cam.tanfovy)
    fy = f32(cam.height) / (f32(2) * tany)
    fx = f32(cam.width) / (f32(2) * tanx)
    return tanx, tany, fx, fy


def exact_rect(means, cov6, cam, kernel_size):
    """The exact path (phase B): view_z > 0.2, cov2d_project with the guard-band clamp, det != 0, lambda_1,
    radius = ceil(3 sqrt(lambda_max)), tile_rect.  Returns (radius, non-empty rectangle, pixel centre)."""
    vm, pm = cam.viewmatrix.reshape(-1).astype(f32), cam.projmatrix.reshape(-1).astype(f32)
    tanx, tany, fx, fy = _camera_consts(cam)
    k = f32(kernel_size)
    gx, gy = (cam.width + TILE - 1) // TILE, (cam.height + TILE - 1) // TILE
    view_z, pix_x, pix_y = _project(means, vm, pm, cam.width, cam.height)
    px, py, pz = (means[:, i].astype(f32) for i in range(3))
    with np.errstate(all="ignore"):
        tx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12]
        ty = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13]
        tz = view_z
        limx, limy = f32(1.3) * tanx, f32(1.3) * tany
        tx = np.minimum(limx, np.maximum(-limx, tx / tz)) * tz
        ty = np.minimum(limy, np.maximum(-limy, ty / tz)) * tz
        a0, a2 = fx / tz, -(fx * tx) / (tz * tz)
        b1, b2 = fy / tz, -(fy * ty) / (tz * tz)
        T0 = [vm[4 * i] * a0 + vm[4 * i + 2] * a2 for i in range(3)]
        T1 = [vm[4 * i + 1] * b1 + vm[4 * i + 2] * b2 for i in range(3)]
        c = [cov6[:, i].astype(f32) for i in range(6)]
        V = [(c[0], c[1], c[2]), (c[1], c[3], c[4]), (c[2], c[4], c[5])]
        X0 = [T0[0] * V[0][j] + T0[1] * V[1][j] + T0[2] * V[2][j] for j in range(3)]
        X1 = [T1[0] * V[0][j] + T1[1] * V[1][j] + T1[2] * V[2][j] for j in range(3)]
        c00 = X0[0] * T0[0] + X0[1] * T0[1] + X0[2] * T0[2] + k
        c01 = X1[0] * T0[0] + X1[1] * T0[1] + X1[2] * T0[2]
        c11 = X1[0] * T1[0] + X1[1] * T1[1] + X1[2] * T1[2] + k
        det = c00 * c11 - c01 * c01
        mid = f32(0.5) * (c00 + c11)
        disc = np.sqrt(np.fmax(f32(0.1), mid * mid - det))
        radius = _to_int(np.ceil(f32(3) * np.sqrt(np.fmax(mid + disc, mid - disc))))
        x0, y0, x1, y1 = tile_rect_np(pix_x, pix_y, radius, gx, gy)
    visible = (view_z > f32(0.2)) & (det != 0) & ((x1 - x0) * (y1 - y0) != 0)
    return np.where(visible, radius, 0), visible, pix_x, pix_y


def cull_candidate(means, cam, kernel_size, cov6=None, scales=None, rots=None, mod=1.0, precomp_bound="frobenius",
                   tighten=1.0):
    """Phase A: view_z > 0.199, radius_bound of |lambda|(Sigma) (scale / rotation: trace; precomputed: Frobenius
    norm, or `precomp_bound="trace"` as the cull had it before), tile_rect of (centre, (int)rb + 1).  `tighten`
    scales the bound (1: as the kernel has it)."""
    vm, pm = cam.viewmatrix.reshape(-1).astype(f32), cam.projmatrix.reshape(-1).astype(f32)
    tanx, tany, fx, fy = _camera_consts(cam)
    k = f32(kernel_size)
    gx, gy = (cam.width + TILE - 1) // TILE, (cam.height + TILE - 1) // TILE
    limx, limy = f32(1.3) * tanx, f32(1.3) * tany
    wf2 = f32(sum(float(vm[i]) ** 2 for i in (0, 1, 2, 4, 5, 6, 8, 9, 10)))
    jw2 = (fx * fx * (f32(1) + limx * limx) + fy * fy * (f32(1) + limy * limy)) * wf2
    view_z, pix_x, pix_y = _project(means, vm, pm, cam.width, cam.height)
    with np.errstate(all="ignore"):
        if cov6 is not None:
            c = cov6.astype(f32)
            if precomp_bound == "trace":
                sig = c[:, 0] + c[:, 3] + c[:, 5]
            else:
                sig = np.sqrt(c[:, 0] ** 2 + c[:, 3] ** 2 + c[:, 5] ** 2 + f32(2) * (c[:, 1] ** 2 + c[:, 2] ** 2 + c[:, 4] ** 2))
        else:
            n = (_rot(rots) ** 2).sum(1)                       # n_r = sum_c R[c][r]^2
            s = scales.astype(f32)
            sig = f32(mod) * f32(mod) * (s[:, 0] ** 2 * n[:, 0] + s[:, 1] ** 2 * n[:, 1] + s[:, 2] ** 2 * n[:, 2])
        tr2d = jw2 * np.abs(sig) / (view_z * view_z) * f32(1.01) + f32(2) * k + f32(0.32)
        rb = (f32(3) * np.sqrt(tr2d) + f32(3)) * f32(tighten)
        x0, y0, x1, y1 = tile_rect_np(pix_x, pix_y, _to_int(rb) + 1, gx, gy)
    wild = ~(rb < f32(1e9)) | ~(np.abs(pix_x) < f32(1e9)) | ~(np.abs(pix_y) < f32(1e9))
    return (view_z > f32(0.199)) & (wild | ((x1 - x0) * (y1 - y0) != 0))


# ----------------------------------------------------------------------------- the sampler
def _nb(x, n):
    """The float32 n ulps above (n > 0) or below x."""
    x = f32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, f32(np.inf if n > 0 else -np.inf))
    return x


def _view_camera(rng, W, H, fov_deg, rotate):
    """A pinhole camera at the origin; `rotate`: a random orientation, else the identity (view space = world)."""
    focal = (H / 2.0) / math.tan(math.radians(fov_deg) / 2.0)
    Rw = np.eye(3)
    if rotate:
        Rw, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        Rw *= np.sign(np.linalg.det(Rw))
    return S.camera_from_w2c(Rw, np.zeros(3), 2 * math.atan(W / (2 * focal)), 2 * math.atan(H / (2 * focal)), W, H), Rw


def _sample_view_points(rng, n, cam):
    """View-space points: depths at and beside the near plane (0.2f and 0.199f with their float neighbours), |tx/tz|
    from 0 to 20 limx (limx and its neighbours included), i.e. centres up to ~10^4 px off screen."""
    limx, limy = f32(1.3) * f32(cam.tanfovx), f32(1.3) * f32(cam.tanfovy)
    special_z = np.array([_nb(0.2, d) for d in (-2, -1, 0, 1, 2)] + [_nb(0.199, d) for d in (-1, 0, 1)], f32)
    z = np.where(rng.random(n) < 0.5, rng.uniform(0.2, 0.3, n), np.exp(rng.uniform(np.log(0.3), np.log(60.0), n)))
    z = np.where(rng.random(n) < 0.2, rng.choice(special_z, n), z).astype(f32)
    def ratio(lim):
        special = np.array([_nb(lim, d) for d in (-1, 0, 1)], f32)
        r = np.where(rng.random(n) < 0.5, rng.uniform(0, 20 * lim, n), rng.uniform(0, 1.5 * lim, n)).astype(f32)
        r = np.where(rng.random(n) < 0.15, rng.choice(special, n), r)
        return (r * rng.choice([-1, 1], n)).astype(f32)
    return np.stack([ratio(limx) * z, ratio(limy) * z, z], 1).astype(f32)


def _sample_scales(rng, n, kind):
    if kind == "round":
        s = np.exp(rng.uniform(np.log(1e-3), np.log(3.0), n))[:, None] * np.exp(rng.normal(0, 0.1, (n, 3)))
    elif kind == "elongated":
        s = np.exp(rng.uniform(np.log(1e-3), np.log(0.3), (n, 3)))
        s[:, 0] *= np.exp(rng.uniform(np.log(5.0), np.log(50.0), n))
    else:   # needle
        s = np.exp(rng.uniform(np.log(1e-4), np.log(1e-2), (n, 3)))
        s[:, 0] = np.exp(rng.uniform(np.log(0.3), np.log(10.0), n))
    return s.astype(f32)


def _rand_quat(rng, n):
    q = rng.normal(size=(n, 4))
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(f32)


def _sample_precomp(rng, n, indefinite):
    """Symmetric 3x3 covariances: PSD (random M M^T) or indefinite (eigenvalues of both signs)."""
    Q = np.linalg.qr(rng.normal(size=(n, 3, 3)))[0]
    lam = np.exp(rng.uniform(np.log(1e-4), np.log(4.0), (n, 3)))
    if indefinite:
        lam *= np.where(rng.random((n, 3)) < 0.5, -1.0, 1.0)
        lam[:, 0] = np.abs(lam[:, 0]); lam[:, 1] = -np.abs(lam[:, 1])   # at least one of each sign
    Sg = np.einsum("nij,nj,nkj->nik", Q, lam, Q)
    return np.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1).astype(f32)


CULL_CAMERAS = [(640, 480, 60.0), (1920, 1080, 50.0), (333, 217, 90.0), (1000, 1000, 20.0)]


def _cull_cases(seed, n=4000):
    """Every (camera, covariance kind, scale_modifier, kernel_size) case of the property test: yields the camera, the
    world-space means, the covariance inputs and the exact path's verdict."""
    rng = np.random.default_rng(seed)
    for ci, (W, H, fov) in enumerate(CULL_CAMERAS):
        for rotate in (False, True):
            cam, Rw = _view_camera(rng, W, H, fov, rotate)
            for kind in ("round", "elongated", "needle", "psd", "indefinite"):
                for mod in (0.5, 1.0, 2.0):
                    for ks in (0.0, 0.1, 0.3):
                        t = _sample_view_points(rng, n, cam)
                        means = (t.astype(np.float64) @ Rw).astype(f32)     # view = R_w2c world
                        if kind in ("psd", "indefinite"):
                            cov6 = _sample_precomp(rng, n, kind == "indefinite") * f32(mod)
                            yield cam, means, ks, dict(cov6=cov6), cov6
                        else:
                            sc, q = _sample_scales(rng, n, kind), _rand_quat(rng, n)
                            yield cam, means, ks, dict(scales=sc, rots=q, mod=mod), cov3d_np(sc, q, mod)


def test_pre_cull_never_drops_a_drawn_gaussian():
    """One-sided: a Gaussian whose exact tile rectangle is non-empty is always a candidate of the pre-cull.  The
    sampler must reach both sides of the bound: Gaussians the cull drops, and Gaussians it keeps whose centre lies
    off screen (where only the bound decides)."""
    culled = kept_off_screen = drawn = 0
    tightest = 0.0          # the largest factor < 1 by which a scaled-down bound drops a drawn Gaussian of the samples
    for cam, means, ks, cov_in, cov6 in _cull_cases(seed=7):
        rad, vis, pix_x, pix_y = exact_rect(means, cov6, cam, ks)
        cand = cull_candidate(means, cam, ks, **cov_in)
        bad = vis & ~cand
        assert not bad.any(), (cam.width, cam.height, ks, means[bad][:3], cov6[bad][:3], rad[bad][:3])
        off = (pix_x < 0) | (pix_x >= cam.width) | (pix_y < 0) | (pix_y >= cam.height)
        culled += int((~cand).sum())
        kept_off_screen += int((cand & off & vis).sum())
        drawn += int(vis.sum())
        for t in (0.9, 0.8, 0.7, 0.6, 0.5):
            if t <= tightest:
                break
            if (vis & ~cull_candidate(means, cam, ks, tighten=t, **cov_in)).any():
                tightest = t
                break
    print(f"\n[pre-cull] drawn {drawn}, culled {culled}, kept with the centre off screen {kept_off_screen}, "
          f"a bound scaled by {tightest} drops a drawn Gaussian")
    assert culled > 1000 and kept_off_screen > 1000 and drawn > 10000
    # the samples come within 2x of the bound.  Not closer: |W|_F^2 = 3 in the bound where |W|_2^2 = 1 would do, so
    # the radius bound holds a factor of sqrt(3) by construction, and a bound 20 % tighter is still safe
    assert tightest >= 0.5


def test_pre_cull_edges():
    """The cull's edges, one Gaussian each: the depth margin (0.199 < z <= 0.2 is a candidate the exact path then
    rejects), and a precomputed indefinite covariance whose trace is 0 but whose projection covers
    hundreds of pixels."""
    cam, _ = _view_camera(np.random.default_rng(0), 640, 480, 60.0, rotate=False)
    tanx = f32(cam.tanfovx)
    fx = f32(cam.width) / (f32(2) * tanx)
    one = lambda x, y, z: np.array([[x, y, z]], f32)  # noqa: E731
    sc, q = np.full((1, 3), 0.01, f32), np.array([[1, 0, 0, 0]], f32)
    cov = cov3d_np(sc, q, 1.0)
    for z, cand, vis in ((_nb(0.199, -1), False, False), (_nb(0.199, 1), True, False), (f32(0.2), True, False),
                         (_nb(0.2, 1), True, True)):
        assert bool(cull_candidate(one(0, 0, z), cam, 0.1, scales=sc, rots=q)[0]) == cand, z
        assert bool(exact_rect(one(0, 0, z), cov, cam, 0.1)[1][0]) == vis, z
    # a counterexample to a trace bound: Sigma = diag(4, -4, 0) at z = 5, centre ~330 px left of the image
    z = f32(5.0)
    x = -(tanx + f32(330.0) / fx) * z
    ind = np.array([[4, 0, 0, -4, 0, 0]], f32)
    rad, vis, pix_x, _ = exact_rect(one(x, 0, z), ind, cam, 0.1)
    assert vis[0] and rad[0] > 400 and pix_x[0] < -300, (rad, pix_x)
    assert not cull_candidate(one(x, 0, z), cam, 0.1, cov6=ind, precomp_bound="trace")[0]   # a trace bound drops it
    assert cull_candidate(one(x, 0, z), cam, 0.1, cov6=ind)[0]


# ============================================================================ GPU frames
def street_camera(width, height, eye=(3.0, -5.0, 2.5), yaw_deg=20.0, pitch_deg=-5.0, fov_deg=60.0):
    """A camera a few units above the ground of the city, looking near horizontally through the cloud (COLMAP axes;
    `fov_deg` is the vertical field of view)."""
    yaw, pitch = math.radians(yaw_deg), math.radians(pitch_deg)
    fwd = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), math.sin(pitch)])
    right = np.cross(fwd, [0.0, 0.0, 1.0]); right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, eye
    w2c = np.linalg.inv(c2w)
    focal = (height / 2.0) / math.tan(math.radians(fov_deg) / 2.0)
    return S.camera_from_w2c(w2c[:3, :3].T, w2c[:3, 3], 2 * math.atan(width / (2 * focal)),
                             2 * math.atan(height / (2 * focal)), width, height)


STREET_P = 2_000_000      # dense enough that the tiles along the horizon hold > 4096 splats


def street_scene():
    return S.city_scene(STREET_P, seed=12)


def crafted_scene():
    """The crafted near frame (identity view rotation: view space = world, so view_z is exact): Gaussians at 0.2f and
    0.199f and their float neighbours, straddling the guard band in x and y, one splat filling the screen at z = 0.21,
    off-screen centres whose rectangles reach the image, exact duplicates (depth ties) and a cloud behind them."""
    cam = S.simple_camera(647, 483, fov_deg=60.0, distance=0.0)
    rng = np.random.default_rng(3)
    limx, limy = f32(1.3) * f32(cam.tanfovx), f32(1.3) * f32(cam.tanfovy)
    tanx, tany = float(cam.tanfovx), float(cam.tanfovy)
    pts, scl = [], []
    for z in [_nb(0.2, d) for d in (-2, -1, 0, 1, 2)] + [_nb(0.199, d) for d in (-1, 0, 1)]:   # the near plane
        for _ in range(12):
            pts.append((rng.uniform(-0.9, 0.9) * tanx * z, rng.uniform(-0.9, 0.9) * tany * z, z))
            scl.append(np.exp(rng.uniform(np.log(2e-3), np.log(2e-2), 3)))
    for axis, lim in ((0, limx), (1, limy)):                                                 # the guard band
        for r in [_nb(lim, d) for d in (-1, 0, 1)] + [lim * f32(f) for f in (0.999, 1.001, 1.5, 3.0)]:
            for sgn in (-1.0, 1.0):
                for z in (0.25, 0.5, 2.0):
                    p = [rng.uniform(-0.5, 0.5) * tanx * z, rng.uniform(-0.5, 0.5) * tany * z, z]
                    p[axis] = float(sgn * r * f32(z))
                    pts.append(tuple(p))
                    scl.append(np.array([0.12, 0.2, 0.05]) * z * rng.uniform(0.7, 1.5))
    pts.append((0.0, 0.0, 0.21)); scl.append(np.array([0.5, 0.4, 0.3]))                    # fills the screen
    for _ in range(300):                                                                     # centres off screen
        z = float(np.exp(rng.uniform(np.log(0.3), np.log(20.0))))
        ang = rng.uniform(0, 2 * np.pi)
        k = float(np.exp(rng.uniform(np.log(1.1), np.log(25.0))))
        pts.append((k * tanx * math.cos(ang) * z, k * tany * math.sin(ang) * z, z))
        scl.append(np.full(3, 0.25 * k * z * rng.uniform(0.2, 1.5)) * np.exp(rng.normal(0, 0.3, 3)))
    n_special = len(pts)
    dup = rng.choice(n_special, n_special // 3, replace=False)                               # exact duplicates
    cloud = rng.normal(0, 1.0, (4000, 3)) * [1.2, 0.9, 1.0] + [0, 0, 3.5]                      # behind them
    means = np.concatenate([np.array(pts), np.array(pts)[dup], cloud]).astype(f32)
    scales = np.concatenate([np.array(scl), np.array(scl)[dup], np.exp(rng.normal(np.log(0.05), 0.5, (4000, 3)))])
    scene = S.blob_scene(means.shape[0], seed=4)
    scene.means3D, scene.scales = means, scales.astype(f32)
    scene.rotations[n_special:n_special + len(dup)] = scene.rotations[dup]
    scene.opacities[n_special:n_special + len(dup)] = scene.opacities[dup]
    scene.shs[n_special:n_special + len(dup)] = scene.shs[dup]
    scene.opacities[n_special - 301] = 0.35                                                   # the screen filler
    return scene, cam, n_special


FRAMES = {
    "street_1920x1080": lambda: (street_scene(), street_camera(1920, 1080)),
    "street_999x541": lambda: (street_scene(), street_camera(999, 541)),
    "blob": lambda: (S.blob_scene(30_000, seed=61, spread=2.5, scale=0.12), S.simple_camera(640, 400, 70.0, 0.0)),
    "crafted": lambda: crafted_scene()[:2],
}


def frame(name):
    return Hh.cached("inside_frame", name, FRAMES[name])


# ----------------------------------------------------------------------------- C. against the reference build
def _parity(dev, name, gradients=True):
    F = Hh.RefFacts(f"inside_{name}")
    scene, cam = frame(name)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    ours = Hh.run_ours_forward(d, cam, 3, bg)
    ref = Hh.run_ref_forward(d, cam, 3, bg) if F.live else None
    P, H, W = scene.P, cam.height, cam.width
    oi, ri = Hh.our_internals(ours, P, H, W), ref_internals(ref, P, H, W)
    lens = oi["ranges"][:, 1] - oi["ranges"][:, 0]
    print(f"\n[{name}] P {P}, visible {int((ours['radii'] > 0).sum())}, num_rendered {ours['num_rendered']}, "
          f"longest tile list {int(lens.max())}")
    check_indexing(F, ours, ref, oi, ri)
    vis = ours["radii"] > 0
    F.same("rgb", bits(oi["rgb"][vis]), lambda: bits(ri["rgb"][vis]))
    check_images(F, ours, ref)
    if gradients:
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=5)]
        gbs = [Hh.run_ours_backward(d, cam, 3, bg, ours, cot) for _ in range(3)]
        F.adjudicate(d, cam, 3, bg, oi, ours["alpha"], ours["radii"], cot, gbs,
                     lambda: (ri, ref["alpha"], ref["radii"],
                              [Hh.run_ref_backward(d, cam, 3, bg, ref, cot) for _ in range(3)]), f"inside[{name}]")
        inv = ~vis
        for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
            assert gbs[0][k][inv].abs().max().item() == 0.0, k
    return ours, oi


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["street_1920x1080", "street_999x541", "blob", "crafted"])
def test_inside_scene_vs_reference(cuda_device, name):
    """Indexing bit for bit (radii, tiles_touched, depth / means2D / cov3D / conic bits, keys, ranges, point_list,
    n_contrib), colours bit for bit, images within 1e-5 and gradients adjudicated by float64."""
    ours, oi = _parity(cuda_device, name)
    if name == "crafted":
        scene, cam, n_special = crafted_scene()
        radii = ours["radii"].cpu().numpy()
        z = scene.means3D[:, 2]
        assert not radii[z <= f32(0.2)].any() and radii[(z > f32(0.2)) & (z < f32(0.2001))].all()
        assert radii[n_special - 301] > max(cam.width, cam.height)          # the screen filler
        pix = np.abs(scene.means3D[:, 0] / z) > 1.3 * cam.tanfovx
        assert (radii[pix] > 0).sum() > 20                                 # drawn from beyond the guard band


@pytest.mark.gpu
def test_precomputed_covariances_vs_reference(cuda_device):
    """The crafted frame with precomputed covariances, PSD and indefinite (the reference projects any Sigma whose 2D
    determinant is non-zero): indexing bit for bit and images within 1e-5 against the reference build, called with
    cov3D_precomp directly.  Includes Sigma = diag(4, -4, 0) ~330 px left of the image, which a trace bound culls."""
    from sfgs import rasterizer as R
    dev = cuda_device
    F = Hh.RefFacts("inside_precomp")
    scene, cam, n_special = crafted_scene()
    rng = np.random.default_rng(17)
    cov6 = cov3d_np(scene.scales, scene.rotations, 1.0)
    ind = rng.choice(scene.P, scene.P // 5, replace=False)
    cov6[ind] = _sample_precomp(rng, len(ind), True) * f32(0.05)
    means = scene.means3D.copy()
    tanx = f32(cam.tanfovx)
    fx = f32(cam.width) / (f32(2) * tanx)
    means[-1] = (-(tanx + f32(330.0) / fx) * f32(5.0), 0.0, 5.0)
    cov6[-1] = (4, 0, 0, -4, 0, 0)
    # A Sigma that projects to a negative definite 2D covariance gets radius (int)NaN = 0 and a non-empty rectangle;
    # the reference then counts its tiles but writes no keys for them (it duplicates only radii > 0), so its binning
    # holds unwritten slots and its indexing is undefined.  Those keep their PSD covariance here.
    rad, vis, _, _ = exact_rect(means, cov6, cam, 0.1)
    neg = vis & (rad == 0)
    cov6[neg] = cov3d_np(scene.scales[neg], scene.rotations[neg], 1.0)
    rad, vis, _, _ = exact_rect(means, cov6, cam, 0.1)
    assert not (vis & (rad == 0)).any() and int(neg.sum()) < len(ind) // 2
    scene.means3D = means
    d = Hh.to_torch(scene, cam, dev)
    cov_t = torch.from_numpy(cov6).to(dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    e = torch.empty(0, device=dev)
    args = (bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, cov_t, e)
    out = R.rasterize_gaussians(*args, e, 0, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1,
                                cam.height, cam.width, d["shs"], 3, d["campos"], False, False)
    ours = dict(zip(Hh.FWD_KEYS, out))
    ref = None
    if F.live:
        from oracle import ref_cuda
        ref = ref_cuda.forward(*args, e, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1,
                               cam.height, cam.width, d["shs"], 3, d["campos"])
    oi, ri = Hh.our_internals(ours, scene.P, cam.height, cam.width), ref_internals(ref, scene.P, cam.height, cam.width)
    print(f"\n[precomp] num_rendered {ours['num_rendered']}, indefinite drawn "
          f"{int((ours['radii'][torch.from_numpy(ind).to(dev)] > 0).sum())}, diag(4,-4,0) radius {int(ours['radii'][-1])}")
    want_rad, want_vis, _, _ = exact_rect(means, cov6, cam, 0.1)
    assert int(ours["radii"][-1]) == want_rad[-1] > 400
    check_indexing(F, ours, ref, oi, ri, full=False)
    # check_indexing(full=True) without cov3D: neither rasterizer writes its cov3D buffer when Sigma is given
    vis = ours["radii"] > 0
    F.same("tiles_touched", oi["tiles_touched"], lambda: ri["tiles_touched"])
    for k in ("depths", "means2D", "conic_opacity"):
        F.same(k, bits(oi[k][vis]), lambda: bits(ri[k][vis]))
    F.same("keys", Hh.ref_style_keys(oi["ranges"], oi["keys"]), lambda: ri["keys"])
    check_images(F, ours, ref)


# ----------------------------------------------------------------------------- D. against the CPU oracle
@pytest.mark.gpu
def test_inside_blob_vs_cpu_oracle(cuda_device):
    """A small frame from inside a blob against the plain-C restatement of the reference, with the tolerances of
    test_gpu_parity.test_against_cpu_oracle: independent of the reference build."""
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene, cam = S.blob_scene(2500, seed=43, spread=1.5), S.simple_camera(190, 150, fov_deg=70.0, distance=0.0)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    d = Hh.to_torch(scene, cam, dev)
    f = Hh.run_ours_forward(d, cam, 3, torch.from_numpy(bg).to(dev))
    o = O.forward(scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs, 3, cam.viewmatrix,
                  cam.projmatrix, cam.campos, cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg)
    print(f"\n[blob vs oracle] num_rendered {f['num_rendered']}")
    assert f["num_rendered"] == o["num_rendered"] and np.array_equal(f["radii"].cpu().numpy(), o["radii"])
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    assert np.array_equal(it["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    assert np.array_equal(it["tiles_touched"].cpu().numpy().astype(np.uint32), o["tiles_touched"])
    for k in ("color", "depth", "norm", "alpha"):
        assert np.abs(f[k].cpu().numpy() - o[k]).max() <= 5e-5, k
    cot = S.cotangents(cam.width, cam.height, seed=6)
    gb = Hh.run_ours_backward(d, cam, 3, torch.from_numpy(bg).to(dev), f, [torch.from_numpy(c).to(dev) for c in cot])
    og = O.backward(o, *cot)
    for k in ("means2D", "opacity", "means3D", "sh", "scales", "rot"):
        a, b = gb[k].cpu().numpy().astype(np.float64), og[k].astype(np.float64)
        assert np.abs(a - b).max() <= 1e-4 + 2e-4 * np.abs(b).max(), k


# ----------------------------------------------------------------------------- E, F. the street view's tile lists, backward variants
@pytest.mark.gpu
def test_street_view_sort_classes_and_backward_variants(cuda_device):
    """The street view's tile lists fall in every size class of the per-tile sort (warp class <= 128 / 256 / 512, CTA
    class <= 1024 / 4096, global radix beyond), several beyond 4096.  On it the deterministic backward is
    bit-reproducible and passes the same float64 adjudication, and the two-phase backward equals the single call."""
    dev = cuda_device
    F = Hh.RefFacts("inside_street_det")
    scene, cam = frame("street_1920x1080")
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    ours = Hh.run_ours_forward(d, cam, 3, bg)
    oi = Hh.our_internals(ours, scene.P, cam.height, cam.width)
    lens = (oi["ranges"][:, 1] - oi["ranges"][:, 0]).cpu().numpy()
    edges = [0, 128, 256, 512, 1024, 4096, np.inf]
    counts = [int(((lens > a) & (lens <= b)).sum()) for a, b in zip(edges[:-1], edges[1:])]
    print(f"\n[street sort classes] tiles per class (<=128, <=256, <=512, <=1024, <=4096, >4096): {counts}")
    assert all(c > 0 for c in counts) and counts[-1] >= 8, counts
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=5)]
    g1 = Hh.run_ours_backward(d, cam, 3, bg, ours, cot, det=True)
    g2 = Hh.run_ours_backward(d, cam, 3, bg, ours, cot, det=True)
    for k in g1:
        assert torch.equal(bits(g1[k]), bits(g2[k])), k
    ref = Hh.run_ref_forward(d, cam, 3, bg) if F.live else None
    ri = ref_internals(ref, scene.P, cam.height, cam.width)
    check_indexing(F, ours, ref, oi, ri, full=False)
    F.adjudicate(d, cam, 3, bg, oi, ours["alpha"], ours["radii"], cot, [g1],
                 lambda: (ri, ref["alpha"], ref["radii"], [Hh.run_ref_backward(d, cam, 3, bg, ref, cot) for _ in range(3)]),
                 "inside[street, deterministic]")
    single = Hh.run_ours_backward(d, cam, 3, bg, ours, cot)
    acc = Hh.run_ours_backward(d, cam, 3, bg, ours, cot, phase=1)
    cut = 400_003
    parts = [Hh.run_ours_backward(d, cam, 3, bg, ours, cot, phase=2, acc=acc[a:b].clone(), gauss_range=(a, b))
             for a, b in ((0, cut), (cut, scene.P))]
    for k in single:
        if single[k].numel() == 0:
            continue
        got = torch.cat([parts[0][k][:cut], parts[1][k][cut:]], 0)
        tol = 1e-5 + 2e-4 * single[k].abs().max().item()
        assert (got - single[k]).abs().max().item() <= tol, k


# ----------------------------------------------------------------------------- G. capacity growth
@pytest.mark.gpu
def test_capacity_grows_from_far_to_near_view(cuda_device):
    """Far (JAX_004) -> near (street) -> far in one process with one capacity estimate: the near frame overflows the
    far frame's binning capacity and re-runs; every result equals a fresh call of the same frame bit for bit, and so
    does a capacity_hint=1 call of the near frame."""
    from sfgs import native as N
    from sfgs import rasterizer as R
    dev = cuda_device
    scene, near_cam = frame("street_1920x1080")
    scene = S.Scene(scene.means3D[:-1], scene.scales[:-1], scene.rotations[:-1], scene.opacities[:-1],
                    scene.shs[:-1], 3)       # one Gaussian fewer: a capacity estimate no other test has grown
    far_cam = S.jax004_camera(1920, 1080)
    bg = torch.tensor([0.0, 0.1, 0.2], device=dev)
    ds = {"far": Hh.to_torch(scene, far_cam, dev), "near": Hh.to_torch(scene, near_cam, dev)}
    cams = {"far": far_cam, "near": near_cam}
    L = N.lib()

    def same(a, b, what):
        assert a["num_rendered"] == b["num_rendered"], what
        for k in ("color", "depth", "norm", "alpha", "radii"):
            assert torch.equal(bits(a[k]), bits(b[k])), (what, k)
        ia = Hh.our_internals(a, scene.P, 1080, 1920)
        ib = Hh.our_internals(b, scene.P, 1080, 1920)
        for k in ("ranges", "point_list", "n_contrib"):
            assert torch.equal(ia[k], ib[k]), (what, k)

    seq = []
    for name in ("far", "near", "far"):
        before = L.sfgs_overflow_reruns()
        seq.append((name, Hh.run_ours_forward(ds[name], cams[name], 3, bg), L.sfgs_overflow_reruns() - before))
    print("\n[capacity] " + ", ".join(f"{n}: num_rendered {f['num_rendered']}, re-runs {r}" for n, f, r in seq))
    assert seq[1][2] >= 1 and seq[2][2] == 0, [r for _, _, r in seq]
    for name, f, _ in seq:
        same(f, Hh.run_ours_forward(ds[name], cams[name], 3, bg), name)
    d = ds["near"]
    e = torch.empty(0, device=dev)
    out = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                d["viewmatrix"], d["projmatrix"], near_cam.tanfovx, near_cam.tanfovy, 0.1, 1080, 1920,
                                d["shs"], 3, d["campos"], False, False, capacity_hint=1)
    same(dict(zip(Hh.FWD_KEYS, out)), seq[1][1], "near, capacity_hint=1")
