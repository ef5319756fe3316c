"""Float64 (or float32) restatement of the per-Gaussian adjoint with the ray-depth terms, for tests/test_ray_depth.py.

`chain` below is tests/chain_f64.py's `chain` with one more keyword, `ray_depth`.  With it on, the restatement also has:
  - each splat's depth slope g = C s, paired with acc words 14-15.  Here C is the conic (cov2D + k I)^-1, held at its
    value, and s = (w3^T Sigma T0^T, w3^T Sigma T1^T), with w3 the view's depth row;
  - the depth's moving centre: dL/dmean2D gains -g dL/ddepth, as the kernel adds it;
  - dL/dC of g in the conic words, which reach the 2D covariance through the kernel's local conic derivative, as in
    the kernel.
With it off, the function is chain_f64.chain; test_ray_depth.py holds the two equal bit for bit.  Everything else
(the helpers, the conic / Mip derivatives) is imported from chain_f64."""
from __future__ import annotations

import numpy as np
import torch

from chain_f64 import axis_index, conic_mip_grads, cov3d, eval_sh, quat_to_rot, sym6_to_mat, view_axis


def chain(acc, radii, means3D, combined_opacity, clamped, shs, D, viewmatrix, projmatrix, campos, W, H, tan_fovx,
          tan_fovy, kernel_size, cov3D=None, scales=None, rotations=None, norm_rec=None, ortho=False, focal=False,
          exact=False, coef=None, hold_bound=False, dtype=torch.float64, ray_depth=False):
    """Gradients of sum_g <acc_g, outputs_g> for the Gaussians with radii > 0, evaluated in `dtype` on the device of
    `radii`.

    acc [P,16]; combined_opacity [P] (opacity times the Mip coefficient) and clamped [P,3] bool (the forward's clamped
    colour channels) of the forward; shs [P,M,3] or None (colors_precomp).  tan_fovx / tan_fovy are the orthographic
    half-extents s_x / s_y with ortho=True, as the library takes them.  The 3D covariance is either the fixed cov3D
    [P,6], or formed from scales [P,3] and rotations [P,4] as leaves (then norm_rec [P,3], the forward's blended
    normals, fixes the normal's adjoint sign).

    Always returns means3D [P,3] (rows of culled Gaussians are 0), Lg [V] (the per-Gaussian loss) and coef (the conic /
    Mip derivatives used; pass them back in to hold them fixed, so that the loss is a fixed function of the camera for
    finite differences).
    A pinhole camera's view, proj and campos are leaves: view [4,4], proj [4,4], campos [3] (each in its input's
    layout), abs [35] (the sum over Gaussians of the magnitude of each camera term: view 16, proj 16, campos 3),
    txtz_lim [V] (|t_x / t_z| / limx, 1 at the clamp's kink), tytz_lim and n_clamped.  focal=True makes tan_fovx and
    tan_fovy leaves too: tanx, tany, and abs [37].  h = W / (2 tan) and lim = 1.3 tan then take the kernel's float32
    values, their derivatives with respect to tan_fov as gradients, so that every other gradient is the focal=False one
    bit for bit; exact=True evaluates them in `dtype` from tan_fov, the function whose finite differences the gradient
    must match; hold_bound=True keeps the clamp bounds from moving with tan_fov (the focal gradient without its clamp
    term).
    ray_depth=True: the ray-depth chain (see the module's note); with it off every result is the one without it.
    With scales / rotations as leaves, also the rest of the per-Gaussian adjoint's rows: means2D, colors, opacity [P,1],
    cov3D, norm3D, sh (with shs), scales and rot."""
    t = lambda a: torch.as_tensor(a).to(dtype)  # noqa: E731
    vis = torch.as_tensor(radii) > 0
    idx = torch.nonzero(vis).flatten()
    P, V = int(vis.numel()), int(idx.numel())
    dev = idx.device
    leaves = scales is not None
    m = t(means3D)[idx].clone().requires_grad_(True)
    Vw = t(viewmatrix).reshape(4, 4).expand(V, 4, 4)
    Pj = t(projmatrix).reshape(4, 4).expand(V, 4, 4)
    if not ortho:
        Vw, Pj = Vw.clone().requires_grad_(True), Pj.clone().requires_grad_(True)
        cp = t(campos).reshape(3).expand(V, 3).clone().requires_grad_(True)
    A = t(acc)[idx]
    f32 = np.float32
    if focal:
        tnx = torch.full((V,), float(tan_fovx), dtype=dtype, device=dev, requires_grad=True)
        tny = torch.full((V,), float(tan_fovy), dtype=dtype, device=dev, requires_grad=True)
    if focal and exact:
        h_x, h_y = W / (2.0 * tnx), H / (2.0 * tny)
        limx, limy = 1.3 * tnx, 1.3 * tny
    elif focal:
        # the kernel's float32 constants as values, their derivatives with respect to tan_fov as gradients
        def pinned(value, x):
            return value + (x - x.detach())
        h_x = pinned(float(f32(W) / (f32(2.0) * f32(tan_fovx))), W / (2.0 * tnx))
        h_y = pinned(float(f32(H) / (f32(2.0) * f32(tan_fovy))), H / (2.0 * tny))
        limx = pinned(float(f32(1.3) * f32(tan_fovx)), 1.3 * tnx)
        limy = pinned(float(f32(1.3) * f32(tan_fovy)), 1.3 * tny)
    else:
        # the kernel's float32 constants
        h_x = t(float(f32(W) / (f32(2.0) * f32(tan_fovx))))
        h_y = t(float(f32(H) / (f32(2.0) * f32(tan_fovy))))
        limx, limy = float(f32(1.3) * f32(tan_fovx)), float(f32(1.3) * f32(tan_fovy))
    ks = float(f32(kernel_size))

    # projected centre
    hom = torch.einsum("gk,gkr->gr", m, Pj[:, :3, :]) + Pj[:, 3, :]
    if ortho:
        L = A[:, 7] * hom[:, 0] + A[:, 8] * hom[:, 1]
    else:
        mw = 1.0 / (hom[:, 3] + 1e-7)
        L = A[:, 7] * (hom[:, 0] * mw) + A[:, 8] * (hom[:, 1] * mw)

    # view-space point: depth and the EWA covariance
    tv = torch.einsum("gk,gkr->gr", m, Vw[:, :3, :3]) + Vw[:, 3, :3]
    tx, ty, tz = tv[:, 0], tv[:, 1], tv[:, 2]
    L = L + A[:, 3] * tz
    Wm = Vw[:, :3, :3].transpose(1, 2)            # Wm[r][c] = viewmatrix[4c + r]
    if ortho:
        T0, T1 = h_x * Wm[:, 0, :], h_y * Wm[:, 1, :]
    else:
        txtz, tytz = tx / tz, ty / tz
        with torch.no_grad():
            clx, cly = (txtz < -limx) | (txtz > limx), (tytz < -limy) | (tytz > limy)
        bx, by = (limx.detach(), limy.detach()) if hold_bound else (limx, limy)
        tx_c = torch.where(clx, txtz.detach().clamp(-bx, bx) * tz.detach(), tx)
        ty_c = torch.where(cly, tytz.detach().clamp(-by, by) * tz.detach(), ty)
        a0, a2 = h_x / tz, -(h_x * tx_c) / (tz * tz)
        b1, b2 = h_y / tz, -(h_y * ty_c) / (tz * tz)
        T0 = a0[:, None] * Wm[:, 0, :] + a2[:, None] * Wm[:, 2, :]
        T1 = b1[:, None] * Wm[:, 1, :] + b2[:, None] * Wm[:, 2, :]
    if leaves:
        sc = t(scales)[idx].clone().requires_grad_(True)
        q = t(rotations)[idx].clone().requires_grad_(True)
        Rm = quat_to_rot(q)
        cv = cov3d(sc, Rm)
        cv.retain_grad()
    else:
        cv = t(cov3D)[idx]
    S = sym6_to_mat(cv)
    c00 = torch.einsum("gi,gij,gj->g", T0, S, T0)
    c01 = torch.einsum("gi,gij,gj->g", T0, S, T1)
    c11 = torch.einsum("gi,gij,gj->g", T1, S, T1)
    if ray_depth:
        # g = C s with the conic C held at its value (its derivative enters through the conic words and the kernel's
        # conic -> cov2D derivative, as in the kernel); s differentiable
        w3 = Wm[:, 2, :]
        s0 = torch.einsum("gi,gij,gj->g", w3, S, T0)
        s1 = torch.einsum("gi,gij,gj->g", w3, S, T1)
        with torch.no_grad():
            a_, b_, c_ = c00 + ks, c01, c11 + ks
            den = a_ * c_ - b_ * b_
            Cx, Cy, Cz = c_ / den, -b_ / den, a_ / den
            gx, gy = Cx * s0 + Cy * s1, Cy * s0 + Cz * s1
            dgx, dgy = A[:, 14], A[:, 15]
            A = A.clone()
            A[:, 10] += s0 * dgx
            A[:, 11] += 0.5 * (s1 * dgx + s0 * dgy)
            A[:, 12] += s1 * dgy
            d7, d8 = -A[:, 3] * gx * (0.5 * W), -A[:, 3] * gy * (0.5 * H)
            A[:, 7] += d7
            A[:, 8] += d8
        L = L + dgx * (Cx * s0 + Cy * s1) + dgy * (Cy * s0 + Cz * s1)
        ndc = hom[:, :2] if ortho else hom[:, :2] * mw[:, None]
        L = L + d7 * ndc[:, 0] + d8 * ndc[:, 1]
    if coef is None:
        coef, mip = conic_mip_grads(A, c00, c01, c11, ks, t(combined_opacity).reshape(-1)[idx])
    dL_da, dL_db, dL_dc = coef
    L = L + dL_da * c00 + dL_db * c01 + dL_dc * c11

    if leaves:
        # the normal R e_axis: the adjoint takes its sign from (R^T e_axis) . n_rec, the rule of computeNorm3D's backward
        ax = axis_index(sc.detach())
        ar = torch.arange(V, device=dev)
        n = Rm[ar, :, ax]
        with torch.no_grad():
            rt = Rm.transpose(1, 2)[ar, :, ax]
            sgn = torch.where((rt * t(norm_rec)[idx]).sum(1) < 0, -1.0, 1.0).to(dtype)
        L = L + (A[:, 4:7] * n * sgn[:, None]).sum(1)

    # SH colour along the view direction
    if shs is not None:
        sh = t(shs)[idx]
        if leaves:
            sh = sh.clone().requires_grad_(True)
        if ortho:
            d = view_axis(viewmatrix, dtype).to(dev).expand(V, 3)
        else:
            d = m - cp
            d = d / torch.sqrt((d * d).sum(1, keepdim=True))
        rgb = eval_sh(int(D), sh, d)
        keep = (~torch.as_tensor(clamped).to(device=dev, dtype=torch.bool)[idx]).to(dtype)
        L = L + (keep * A[:, 0:3] * rgb).sum(1)

    L.sum().backward()
    z = lambda *s: torch.zeros(s, dtype=dtype, device=dev)  # noqa: E731
    out = dict(means3D=z(P, 3), Lg=L.detach(), coef=coef)
    out["means3D"][idx] = m.grad
    if not ortho:
        g_cp = cp.grad if cp.grad is not None else torch.zeros_like(cp)     # colors_precomp: no view direction
        terms = [Vw.grad.reshape(V, 16), Pj.grad.reshape(V, 16), g_cp]
        if focal:
            terms += [tnx.grad[:, None], tny.grad[:, None]]
            out.update(tanx=tnx.grad.sum(0), tany=tny.grad.sum(0))
        with torch.no_grad():
            txtz_lim, tytz_lim = txtz.abs() / limx, tytz.abs() / limy
        out.update(view=Vw.grad.sum(0), proj=Pj.grad.sum(0), campos=g_cp.sum(0), abs=torch.cat(terms, 1).abs().sum(0),
                   txtz_lim=txtz_lim.detach(), tytz_lim=tytz_lim.detach(), n_clamped=int(clx.sum()) + int(cly.sum()))
    if leaves:
        rows = dict(means2D=A[:, 7:10], colors=A[:, 0:3], opacity=(A[:, 13] * mip)[:, None], cov3D=cv.grad,
                    norm3D=A[:, 4:7], scales=sc.grad, rot=q.grad)
        if shs is not None:
            rows["sh"] = sh.grad
        for k, v in rows.items():
            out[k] = z(P, *v.shape[1:])
            out[k][idx] = v
    return out
