"""Float64 (or float32) torch restatement of the chain the per-Gaussian adjoint differentiates, for the camera
gradients (sfgs_rasterize_backward_camera).

The per-Gaussian adjoint is linear in the blend-adjoint sums `acc` (the [P,16] rows the blend adjoint forms).  For given
sums, the camera gradient is the autograd gradient of  sum_g <acc_g, outputs_g(camera, means)>,  where outputs_g are
the preprocess quantities the chain differentiates:
  - the projected centre [m, 1]·projmatrix with its 1/(w + 1e-7) divide (paired with dL/dmean2D);
  - the depth t_z of the view-space point t = [m, 1]·viewmatrix (paired with dL/ddepth);
  - the 2D covariance (J(t)·W) Σ (J(t)·W)^T of the EWA splat, with the limx/limy clamps: a clamped t_x / t_y enters J
    as a constant, as in the kernel;
  - the SH colour along normalize(m - campos), with the clamped channels masked (paired with dL/dcolor).
The conic inverse and the Mip coefficient enter through the kernel's own local derivatives with respect to the 2D
covariance (their 1e-7 / 1e-6 guards make those differ from the exact derivatives by up to ~1e-3 on small splats); from
the 2D covariance back to the camera and the means everything is autograd.  The same restatement's gradient with
respect to means3D reproduces the library's dL_dmean3D: that is the check that it mirrors the chain."""
from __future__ import annotations

import numpy as np
import torch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def eval_sh(D, sh, d):
    """The degree-D SH colour (without the +0.5) of coefficients sh [V,M,3] along unit directions d [V,3]."""
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    r = SH_C0 * sh[:, 0]
    if D > 0:
        r = r - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
    if D > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        r = (r + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * sh[:, 6]
             + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
    if D > 2:
        r = (r + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10]
             + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
             + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + SH_C3[5] * z * (xx - yy) * sh[:, 14]
             + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return r


def acc_from_screen_grads(means2D, colors, depths, norm3D, conic, opacity):
    """[P,16] blend-adjoint sums in the layout of the library's acc rows, from the screen-space gradients of a blend
    adjoint (e.g. the oracle's render backward): colour 3, depth, normal 3, mean2D 3, conic xx, xy, yy, opacity, 0, 0."""
    P = means2D.shape[0]
    z = np.zeros((P, 2), np.float32)
    return np.concatenate([colors, depths.reshape(P, 1), norm3D, means2D, conic[:, 0:2], conic[:, 3:4],
                           opacity.reshape(P, 1), z], 1).astype(np.float32)


def camera_chain(acc, radii, means3D, cov3D, combined_opacity, clamped, shs, D, viewmatrix, projmatrix, campos, W,
                 H, tan_fovx, tan_fovy, kernel_size, dtype=torch.float64):
    """Gradients of sum_g <acc_g, outputs_g> for the Gaussians with radii > 0, evaluated in `dtype`.

    acc [P,16]; cov3D [P,6] and combined_opacity [P] (opacity times the Mip coefficient) of the forward; clamped [P,3]
    bool (the forward's clamped colour channels); shs [P,M,3] or None (colors_precomp).  Returns a dict: means3D [P,3],
    view [4,4], proj [4,4], campos [3] (each in its input's layout), and abs [35], the sum over Gaussians of the
    magnitude of each camera term (view 16, proj 16, campos 3)."""
    t = lambda a: torch.as_tensor(a).to(dtype)  # noqa: E731
    vis = torch.as_tensor(radii) > 0
    idx = torch.nonzero(vis).flatten()
    V = int(idx.numel())
    dev = idx.device
    m = t(means3D)[idx].clone().requires_grad_(True)
    Vw = t(viewmatrix).reshape(4, 4).expand(V, 4, 4).clone().requires_grad_(True)
    Pj = t(projmatrix).reshape(4, 4).expand(V, 4, 4).clone().requires_grad_(True)
    cp = t(campos).reshape(3).expand(V, 3).clone().requires_grad_(True)
    A = t(acc)[idx]
    # the kernel's float32 constants
    f32 = np.float32
    h_x = t(float(f32(W) / (f32(2.0) * f32(tan_fovx))))
    h_y = t(float(f32(H) / (f32(2.0) * f32(tan_fovy))))
    limx, limy = float(f32(1.3) * f32(tan_fovx)), float(f32(1.3) * f32(tan_fovy))
    ks = float(f32(kernel_size))

    # projected centre
    hom = torch.einsum("gk,gkr->gr", m, Pj[:, :3, :]) + Pj[:, 3, :]
    mw = 1.0 / (hom[:, 3] + 1e-7)
    L = A[:, 7] * (hom[:, 0] * mw) + A[:, 8] * (hom[:, 1] * mw)

    # view-space point: depth and the EWA covariance
    tv = torch.einsum("gk,gkr->gr", m, Vw[:, :3, :3]) + Vw[:, 3, :3]
    tx, ty, tz = tv[:, 0], tv[:, 1], tv[:, 2]
    L = L + A[:, 3] * tz
    txtz, tytz = tx / tz, ty / tz
    tx_c = torch.where((txtz < -limx) | (txtz > limx), (txtz.clamp(-limx, limx) * tz).detach(), tx)
    ty_c = torch.where((tytz < -limy) | (tytz > limy), (tytz.clamp(-limy, limy) * tz).detach(), ty)
    a0, a2 = h_x / tz, -(h_x * tx_c) / (tz * tz)
    b1, b2 = h_y / tz, -(h_y * ty_c) / (tz * tz)
    Wm = Vw[:, :3, :3].transpose(1, 2)            # Wm[r][c] = viewmatrix[4c + r]
    T0 = a0[:, None] * Wm[:, 0, :] + a2[:, None] * Wm[:, 2, :]
    T1 = b1[:, None] * Wm[:, 1, :] + b2[:, None] * Wm[:, 2, :]
    cv = t(cov3D)[idx]
    S = torch.stack([cv[:, [0, 1, 2]], cv[:, [1, 3, 4]], cv[:, [2, 4, 5]]], 1)
    c00 = torch.einsum("gi,gij,gj->g", T0, S, T0)
    c01 = torch.einsum("gi,gij,gj->g", T0, S, T1)
    c11 = torch.einsum("gi,gij,gj->g", T1, S, T1)
    with torch.no_grad():
        # the kernel's dL/d(c00, c01, c11): the conic inverse with its 1e-7 guard, plus the Mip coefficient's share
        dLcx, dLcy, dLcz, o_opac = A[:, 10], A[:, 11], A[:, 12], A[:, 13]
        a, b, c = c00 + ks, c01, c11 + ks
        denom = a * c - b * b
        d2i = 1.0 / (denom * denom + 1e-7)
        dL_da = d2i * (-c * c * dLcx + 2 * b * c * dLcy + (denom - a * c) * dLcz)
        dL_dc = d2i * (-a * a * dLcz + 2 * a * b * dLcy + (denom - a * c) * dLcx)
        dL_db = d2i * 2 * (b * c * dLcx - (denom + 2 * b * b) * dLcy + a * b * dLcz)
        det0 = (c00 * c11 - c01 * c01).clamp_min(1e-6)
        det1 = (a * c - b * b).clamp_min(1e-6)
        coef = torch.sqrt(det0 / (det1 + 1e-6) + 1e-6)
        opacity = t(combined_opacity)[idx] / (coef + 1e-6)
        dsq = o_opac * opacity * 0.5 / (coef + 1e-6)
        dd0, dd1 = dsq / (det1 + 1e-6), dsq * det0 * (-1.0 / (det1 * det1 + 1e-6))
        ok = ((det0 > 1e-6) & (det1 > 1e-6)).to(dtype)
        dL_da = dL_da + ok * (dd0 * c11 + dd1 * (c11 + ks))
        dL_db = dL_db + ok * (dd0 * (-2 * c01) + dd1 * (-2 * c01))
        dL_dc = dL_dc + ok * (dd0 * c00 + dd1 * (c00 + ks))
    L = L + dL_da * c00 + dL_db * c01 + dL_dc * c11

    # SH colour along the view direction
    if shs is not None:
        d = m - cp
        d = d / torch.sqrt((d * d).sum(1, keepdim=True))
        rgb = eval_sh(int(D), t(shs)[idx], d)
        keep = (~torch.as_tensor(clamped).to(device=dev, dtype=torch.bool)[idx]).to(dtype)
        L = L + (keep * A[:, 0:3] * rgb).sum(1)

    L.sum().backward()
    g_mean = torch.zeros((int(vis.numel()), 3), dtype=dtype, device=dev)
    g_mean[idx] = m.grad
    g_cp = cp.grad if cp.grad is not None else torch.zeros_like(cp)     # colors_precomp: no view direction
    terms = torch.cat([Vw.grad.reshape(V, 16), Pj.grad.reshape(V, 16), g_cp], 1)
    return dict(means3D=g_mean, view=Vw.grad.sum(0), proj=Pj.grad.sum(0), campos=g_cp.sum(0), abs=terms.abs().sum(0))


def translation_residual(g, viewmatrix, projmatrix):
    """sum_g dL/dmeans3D[g,i] + dL/dcampos[i] - sum_k V[i][k] G_V[3][k] - sum_k Pm[i][k] G_P[3][k], i = 0..2: zero when
    moving the world and the camera together leaves the loss unchanged.  Also returns the sum of the terms' magnitudes."""
    Vm = torch.as_tensor(viewmatrix).reshape(4, 4).to(g["view"])
    Pm = torch.as_tensor(projmatrix).reshape(4, 4).to(g["proj"])
    gm = g["means3D"].to(g["view"])
    parts = [gm.sum(0), g["campos"].to(g["view"]), -(Vm[:3] * g["view"][3]).sum(1), -(Pm[:3] * g["proj"][3]).sum(1)]
    scale = gm.abs().sum(0) + parts[1].abs() + (Vm[:3] * g["view"][3]).abs().sum(1) + (Pm[:3] * g["proj"][3]).abs().sum(1)
    return sum(parts), scale
