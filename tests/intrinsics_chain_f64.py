"""Float64 (or float32) torch restatement of the per-Gaussian adjoint's chain with tan_fovx / tan_fovy as leaves, for
the focal-length gradients (sfgs_rasterize_backward_camera_intrinsics).

It is tests/camera_chain_f64.py's restatement, sum_g <acc_g, outputs_g(camera, means)>, with the two places the
focal lengths enter made functions of tan_fov:
  - h_x = W / (2 tan_fovx) and h_y = H / (2 tan_fovy) in the EWA Jacobian J;
  - the frustum clamp bounds limx = 1.3 tan_fovx, limy = 1.3 tan_fovy, written as torch.clamp on tensor bounds: a
    clamped t_x / t_y is a constant with respect to t (as in the kernel) but moves with its bound.
By default h and lim take the kernel's float32 values (W / (2 tan) and 1.3 tan rounded to float), so every other
gradient is the camera restatement's, bit for bit; `exact=True` evaluates them in `dtype` from tan_fov, the function
whose finite differences the gradient must match.  The kernel's local derivatives with respect to the 2D covariance
(the conic inverse and the Mip coefficient, evaluated without autograd) can be passed in as `coef`, so that the loss
is a fixed function of tan_fov for finite differences."""
from __future__ import annotations

import numpy as np
import torch

from camera_chain_f64 import eval_sh


def intrinsics_chain(acc, radii, means3D, cov3D, combined_opacity, clamped, shs, D, viewmatrix, projmatrix, campos,
                     W, H, tan_fovx, tan_fovy, kernel_size, dtype=torch.float64, exact=False, coef=None,
                     hold_bound=False):
    """camera_chain_f64.camera_chain's gradients plus tanx, tany: dL/dtan_fovx, dL/dtan_fovy.  abs [37] is the sum
    over Gaussians of each camera term's magnitude (view 16, proj 16, campos 3, tan_fovx, tan_fovy); Lg [V] the
    per-Gaussian loss; coef the conic / Mip derivatives used (pass them back in to hold them fixed); txtz_lim [V] the
    ratio |t_x / t_z| / limx, and tytz_lim likewise (1 at the clamp's kink).  hold_bound: the clamp bounds do not
    move with tan_fov (the focal gradient without its clamp term)."""
    t = lambda a: torch.as_tensor(a).to(dtype)  # noqa: E731
    vis = torch.as_tensor(radii) > 0
    idx = torch.nonzero(vis).flatten()
    V = int(idx.numel())
    dev = idx.device
    m = t(means3D)[idx].clone().requires_grad_(True)
    Vw = t(viewmatrix).reshape(4, 4).expand(V, 4, 4).clone().requires_grad_(True)
    Pj = t(projmatrix).reshape(4, 4).expand(V, 4, 4).clone().requires_grad_(True)
    cp = t(campos).reshape(3).expand(V, 3).clone().requires_grad_(True)
    tnx = torch.full((V,), float(tan_fovx), dtype=dtype, device=dev, requires_grad=True)
    tny = torch.full((V,), float(tan_fovy), dtype=dtype, device=dev, requires_grad=True)
    A = t(acc)[idx]
    f32 = np.float32
    if exact:
        h_x, h_y = W / (2.0 * tnx), H / (2.0 * tny)
        limx, limy = 1.3 * tnx, 1.3 * tny
    else:
        # the kernel's float32 constants as values, their derivatives with respect to tan_fov as gradients
        def pinned(value, x):
            return value + (x - x.detach())
        h_x = pinned(float(f32(W) / (f32(2.0) * f32(tan_fovx))), W / (2.0 * tnx))
        h_y = pinned(float(f32(H) / (f32(2.0) * f32(tan_fovy))), H / (2.0 * tny))
        limx = pinned(float(f32(1.3) * f32(tan_fovx)), 1.3 * tnx)
        limy = pinned(float(f32(1.3) * f32(tan_fovy)), 1.3 * tny)
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
    with torch.no_grad():
        clx, cly = (txtz < -limx) | (txtz > limx), (tytz < -limy) | (tytz > limy)
    bx, by = (limx.detach(), limy.detach()) if hold_bound else (limx, limy)
    tx_c = torch.where(clx, txtz.detach().clamp(-bx, bx) * tz.detach(), tx)
    ty_c = torch.where(cly, tytz.detach().clamp(-by, by) * tz.detach(), ty)
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
    if coef is None:
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
            cf = torch.sqrt(det0 / (det1 + 1e-6) + 1e-6)
            opacity = t(combined_opacity)[idx] / (cf + 1e-6)
            dsq = o_opac * opacity * 0.5 / (cf + 1e-6)
            dd0, dd1 = dsq / (det1 + 1e-6), dsq * det0 * (-1.0 / (det1 * det1 + 1e-6))
            ok = ((det0 > 1e-6) & (det1 > 1e-6)).to(dtype)
            dL_da = dL_da + ok * (dd0 * c11 + dd1 * (c11 + ks))
            dL_db = dL_db + ok * (dd0 * (-2 * c01) + dd1 * (-2 * c01))
            dL_dc = dL_dc + ok * (dd0 * c00 + dd1 * (c00 + ks))
            coef = (dL_da, dL_db, dL_dc)
    dL_da, dL_db, dL_dc = coef
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
    terms = torch.cat([Vw.grad.reshape(V, 16), Pj.grad.reshape(V, 16), g_cp, tnx.grad[:, None], tny.grad[:, None]], 1)
    with torch.no_grad():
        txtz_lim, tytz_lim = txtz.abs() / limx, tytz.abs() / limy
    return dict(means3D=g_mean, view=Vw.grad.sum(0), proj=Pj.grad.sum(0), campos=g_cp.sum(0), tanx=tnx.grad.sum(0),
                tany=tny.grad.sum(0), abs=terms.abs().sum(0), Lg=L.detach(), coef=coef, txtz_lim=txtz_lim.detach(),
                tytz_lim=tytz_lim.detach(), n_clamped=int(clx.sum()) + int(cly.sum()))
