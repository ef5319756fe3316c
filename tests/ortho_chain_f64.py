"""Float64 torch restatement of the rasterizer's orthographic camera — test infrastructure for test_ortho.py.

The reference rasterizer has no orthographic camera, so this restatement is the oracle.  It states, in float64 (or any
dtype), what sfgs_rasterize_forward_ortho's preprocess computes per Gaussian (include/sfgs.h, DESIGN.md):
  - t = [m, 1]·viewmatrix, depth t_z, visible when t_z > 0.2;
  - ndc = ([m, 1]·projmatrix).xy with no divide, pixel position ((ndc + 1) S - 1) / 2;
  - the 2D covariance T Sigma T^T with T = J W, J = diag(h_x, h_y), h = S / (2 s) in float32 as the library forms it,
    then the Mip filter, the conic, radius = ceil(3 sqrt(lambda_max)) and the tile rectangle;
  - the SH colour along the view's +z axis normalize(viewmatrix[0:3, 2]) (+0.5, clamped at 0), one direction per frame;
  - the normal: the shortest scale axis of the rotation, flipped so that it does not point along the view axis.
`render` blends the restated records with the CPU oracle's blend (tests/subpixel_oracle.c, which includes the
unchanged oracle), with or without subpixel offsets.  The per-Gaussian adjoint's chain is chain_f64.chain(ortho=True).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from chain_f64 import axis_index, cov3d, eval_sh, quat_to_rot, sym6_to_mat, view_axis  # noqa: F401

TILE = 16


def pixel_scales(W, H, s_x, s_y):
    """The library's float32 h_x = W / (2 s_x), h_y = H / (2 s_y)."""
    f32 = np.float32
    return float(f32(W) / (f32(2.0) * f32(s_x))), float(f32(H) / (f32(2.0) * f32(s_y)))


def project(means3D, scales, rotations, viewmatrix, projmatrix, W, H, s_x, s_y, kernel_size, scale_modifier=1.0,
            cov3D=None):
    """Differentiable geometry of every Gaussian (no culling): dict of t [P,3], ndc [P,2], pix [P,2], cov3D [P,6],
    c00, c01, c11 (the EWA covariance before the filter), R [P,3,3]."""
    dt = means3D.dtype
    V = torch.as_tensor(viewmatrix).reshape(4, 4).to(dt)
    Pm = torch.as_tensor(projmatrix).reshape(4, 4).to(dt)
    t = means3D @ V[:3, :3] + V[3, :3]
    hom = means3D @ Pm[:3, :] + Pm[3, :]
    ndc = hom[:, 0:2]
    pix = torch.stack([((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5], 1)
    Rm = quat_to_rot(rotations)
    if cov3D is None:
        cov3D = cov3d(scale_modifier * scales, Rm)
    h_x, h_y = pixel_scales(W, H, s_x, s_y)
    T0, T1 = h_x * V[:3, 0], h_y * V[:3, 1]        # rows of T = J W, W[r][k] = viewmatrix[k][r]
    S = sym6_to_mat(cov3D)
    c00 = torch.einsum("i,gij,j->g", T0, S, T0)
    c01 = torch.einsum("i,gij,j->g", T0, S, T1)
    c11 = torch.einsum("i,gij,j->g", T1, S, T1)
    return dict(t=t, ndc=ndc, pix=pix, cov3D=cov3D, c00=c00, c01=c01, c11=c11, R=Rm)


def preprocess(means3D, scales, rotations, opacities, viewmatrix, projmatrix, W, H, s_x, s_y, kernel_size, D=0,
               shs=None, colors=None, scale_modifier=1.0):
    """The preprocess of an orthographic frame, in float64.  Inputs are arrays or tensors (CPU or CUDA).  Returns a
    dict of CPU float64 tensors: radii, tiles_touched (int64), lam3 (3 sqrt(lambda_max), before the ceil), pix [P,2],
    conic [P,3], opacity (combined: opacity times the Mip coefficient), depth, rgb [P,3], clamped [P,3] (bool), norm3D
    [P,3], cov3D [P,6]; culled Gaussians have radius 0 and no tiles."""
    f = lambda a: torch.as_tensor(a).detach().cpu().to(torch.float64)  # noqa: E731
    m, sc, q, op = f(means3D), f(scales), f(rotations), f(opacities).reshape(-1)
    g = project(m, sc, q, viewmatrix, projmatrix, W, H, s_x, s_y, kernel_size, scale_modifier)
    ks = float(np.float32(kernel_size))
    c00, c01, c11 = g["c00"], g["c01"], g["c11"]
    det0 = (c00 * c11 - c01 * c01).clamp_min(1e-6)
    det1 = ((c00 + ks) * (c11 + ks) - c01 * c01).clamp_min(1e-6)
    coef = torch.sqrt(det0 / (det1 + 1e-6) + 1e-6)
    coef = torch.where((det0 <= 1e-6) | (det1 <= 1e-6), torch.zeros_like(coef), coef)
    a, b, c = c00 + ks, c01, c11 + ks
    det = a * c - b * b
    conic = torch.stack([c / det, -b / det, a / det], 1)
    mid = 0.5 * (a + c)
    lam = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    lam3 = 3.0 * torch.sqrt(lam)
    radius = torch.ceil(lam3)
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    pix32 = g["pix"].to(torch.float32)
    r32 = radius.to(torch.float32)
    cl = lambda v, n: torch.clamp(v.to(torch.int64), 0, n)  # noqa: E731   (int) truncates toward zero, as the kernel
    x0, y0 = cl(torch.trunc((pix32[:, 0] - r32) / TILE), gx), cl(torch.trunc((pix32[:, 1] - r32) / TILE), gy)
    x1 = cl(torch.trunc((pix32[:, 0] + r32 + (TILE - 1)) / TILE), gx)
    y1 = cl(torch.trunc((pix32[:, 1] + r32 + (TILE - 1)) / TILE), gy)
    ntiles = (x1 - x0) * (y1 - y0)
    vis = (g["t"][:, 2] > 0.2) & (det != 0) & (ntiles > 0)
    d = view_axis(viewmatrix)
    if colors is not None:
        rgb, clamped = f(colors).reshape(-1, 3), torch.zeros((m.shape[0], 3), dtype=torch.bool)
    else:
        v = eval_sh(int(D), f(shs), d.expand(m.shape[0], 3)) + 0.5
        clamped = v < 0
        rgb = torch.where(clamped, torch.zeros_like(v), v)
    ax = axis_index(sc)
    n = g["R"][torch.arange(m.shape[0]), :, ax]              # R e_axis
    n = torch.where(((n @ d) > 0)[:, None], -n, n)
    z = lambda x: torch.where(vis.reshape(-1, *([1] * (x.ndim - 1))), x, torch.zeros_like(x))  # noqa: E731
    return dict(visible=vis, radii=torch.where(vis, radius, torch.zeros_like(radius)).to(torch.int64),
                tiles_touched=torch.where(vis, ntiles, torch.zeros_like(ntiles)), lam3=lam3, pix=z(g["pix"]),
                conic=z(conic), opacity=z(op * coef), depth=z(g["t"][:, 2]), rgb=z(rgb), clamped=clamped,
                norm3D=z(n), cov3D=g["cov3D"], rect=torch.stack([x0, y0, x1, y1], 1))


def render(pre, W, H, bg, subpixel_offset=None):
    """Blend the restated records with the CPU oracle's blend (float32, as the library blends them).  Returns numpy
    color [3,H,W], depth [1,H,W], norm [3,H,W] (unnormalised), alpha [1,H,W]."""
    import subpixel_oracle as SO
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    vis = np.nonzero(pre["visible"].numpy())[0]
    depth32 = pre["depth"].numpy().astype(np.float32)
    tiles, ids, depths = [], [], []
    rect = pre["rect"].numpy()
    for i in vis:
        x0, y0, x1, y1 = rect[i]
        for ty in range(y0, y1):
            for tx in range(x0, x1):
                tiles.append(ty * gx + tx)
                ids.append(i)
                depths.append(depth32[i])
    tiles, ids, depths = np.array(tiles, np.int64), np.array(ids, np.int64), np.array(depths, np.float32)
    order = np.lexsort((ids, depths, tiles))          # per tile, by depth, ties by index (the key's low word)
    tiles, plist = tiles[order], ids[order].astype(np.uint32)
    ranges = np.zeros((gx * gy, 2), np.uint32)
    if tiles.size:
        starts = np.searchsorted(tiles, np.arange(gx * gy), "left")
        ends = np.searchsorted(tiles, np.arange(gx * gy), "right")
        ranges[:, 0], ranges[:, 1] = starts, ends
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float32))  # noqa: E731
    means2D = f32(pre["pix"].numpy())
    co = f32(torch.cat([pre["conic"], pre["opacity"][:, None]], 1).numpy())
    rgb, nrm, dep = f32(pre["rgb"].numpy()), f32(pre["norm3D"].numpy()), f32(pre["depth"].numpy())
    off = np.zeros((H, W, 2), np.float32) if subpixel_offset is None else f32(subpixel_offset)
    out = dict(color=np.zeros((3, H, W), np.float32), depth=np.zeros((1, H, W), np.float32),
               norm=np.zeros((3, H, W), np.float32), alpha=np.zeros((1, H, W), np.float32))
    n_contrib = np.zeros(H * W, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    SO.cpu_lib().oracle_render_subpixel(
        C.c_int(W), C.c_int(H), C.c_int(0), p(np.ascontiguousarray(ranges)), p(np.ascontiguousarray(plist)),
        p(means2D), p(rgb), p(nrm), p(dep), None, p(co), p(f32(bg)), p(out["color"]), p(out["depth"]), p(out["norm"]),
        p(out["alpha"]), None, p(n_contrib), p(off))
    return out


def scalar_outputs(means3D, scales, rotations, opacities, viewmatrix, projmatrix, W, H, s_x, s_y, kernel_size, D,
                   shs, weights):
    """sum_g <weights_g, (ndc, depth, c00, c01, c11, rgb)>: a smooth function of the restated forward, for the
    central-difference check of `project` and the SH path."""
    g = project(means3D, scales, rotations, viewmatrix, projmatrix, W, H, s_x, s_y, kernel_size)
    d = view_axis(viewmatrix, means3D.dtype).expand(means3D.shape[0], 3)
    rgb = eval_sh(int(D), shs, d)
    cols = torch.cat([g["ndc"], g["t"][:, 2:3], torch.stack([g["c00"], g["c01"], g["c11"]], 1), rgb], 1)
    return (weights * cols).sum()


def near_integer(lam3, tol=1e-4):
    """Gaussians whose float64 3 sqrt(lambda_max) lies within tol of an integer: float32 may round them the other way."""
    return (lam3 - torch.round(lam3)).abs() < tol

