"""Float64 (or float32) torch restatement of the chain the per-Gaussian adjoint differentiates, for the camera, focal
and orthographic gradient tests.

The per-Gaussian adjoint is linear in the blend-adjoint sums `acc` (the [P,16] rows the blend adjoint forms).  For given
sums, its gradients are the autograd gradients of  sum_g <acc_g, outputs_g>,  where outputs_g are the preprocess
quantities the chain differentiates:
  - the projected centre [m, 1]·projmatrix, with its 1/(w + 1e-7) divide for a pinhole camera and none for an
    orthographic one (paired with dL/dmean2D);
  - the depth t_z of the view-space point t = [m, 1]·viewmatrix (paired with dL/ddepth);
  - the 2D covariance (J·W) Σ (J·W)^T of the EWA splat: for a pinhole camera J(t) with the limx/limy clamps (a clamped
    t_x / t_y enters J as a constant, as in the kernel), for an orthographic one the constant J = diag(h_x, h_y);
  - the SH colour with the clamped channels masked (paired with dL/dcolor), along normalize(m - campos) for a pinhole
    camera and along the view's +z axis for an orthographic one;
  - with scales / rotations as leaves, the normal: the shortest scale axis of the rotation, its adjoint sign taken by
    the kernel's rule.
The conic inverse and the Mip coefficient enter through the kernel's own local derivatives with respect to the 2D
covariance (`conic_mip_grads`; their 1e-7 / 1e-6 guards make those differ from the exact derivatives by up to ~1e-3 on
small splats); from the 2D covariance back to the camera and the Gaussians everything is autograd.  The restatement's
gradient with respect to means3D reproduces the library's dL_dmean3D: that is the check that it mirrors the chain."""
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


def quat_to_rot(q):
    """The library's rotation of an un-normalised quaternion (r, x, y, z): R[a][b] with Sigma = R diag(s^2) R^T."""
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
        torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
        torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def cov3d(s, Rm):
    """The 3D covariance R diag(s^2) R^T as its six upper-triangle entries [P,6]."""
    Sig = Rm @ torch.diag_embed(s * s) @ Rm.transpose(1, 2)
    return torch.stack([Sig[:, 0, 0], Sig[:, 0, 1], Sig[:, 0, 2], Sig[:, 1, 1], Sig[:, 1, 2], Sig[:, 2, 2]], 1)


def sym6_to_mat(c):
    return torch.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], 1)


def view_axis(viewmatrix, dtype=torch.float64):
    """The world-space unit vector of the view's +z axis (the orthographic SH and normal view direction)."""
    V = torch.as_tensor(viewmatrix).reshape(4, 4).to(dtype)
    d = V[:3, 2]
    return d / torch.sqrt((d * d).sum())


def axis_index(scales):
    """Index of the shortest-axis rule of the normal: z if sx > sz and sy > sz, else y if sx > sy and sz > sy, else x."""
    sx, sy, sz = scales[:, 0], scales[:, 1], scales[:, 2]
    return torch.where((sx > sz) & (sy > sz), 2, torch.where((sx > sy) & (sz > sy), 1, 0))


def acc_from_screen_grads(means2D, colors, depths, norm3D, conic, opacity):
    """[P,16] blend-adjoint sums in the layout of the library's acc rows, from the screen-space gradients of a blend
    adjoint (e.g. the oracle's render backward): colour 3, depth, normal 3, mean2D 3, conic xx, xy, yy, opacity, 0, 0."""
    P = means2D.shape[0]
    z = np.zeros((P, 2), np.float32)
    return np.concatenate([colors, depths.reshape(P, 1), norm3D, means2D, conic[:, 0:2], conic[:, 3:4],
                           opacity.reshape(P, 1), z], 1).astype(np.float32)


def conic_mip_grads(A, c00, c01, c11, ks, combined_opacity):
    """The kernel's dL/d(c00, c01, c11) for the acc rows A [V,16] (gauss_adjoint): the conic inverse with its 1e-7
    guard, plus the Mip coefficient's share, with the opacity recovered as combined_opacity / (coef + 1e-6), as the
    kernel recovers it.  Evaluated without autograd.  Returns the three derivatives and the Mip coefficient (0 where
    either determinant is degenerate)."""
    with torch.no_grad():
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
        opacity = combined_opacity / (coef + 1e-6)
        dsq = o_opac * opacity * 0.5 / (coef + 1e-6)
        dd0, dd1 = dsq / (det1 + 1e-6), dsq * det0 * (-1.0 / (det1 * det1 + 1e-6))
        ok = ((det0 > 1e-6) & (det1 > 1e-6)).to(c00.dtype)
        dL_da = dL_da + ok * (dd0 * c11 + dd1 * (c11 + ks))
        dL_db = dL_db + ok * (dd0 * (-2 * c01) + dd1 * (-2 * c01))
        dL_dc = dL_dc + ok * (dd0 * c00 + dd1 * (c00 + ks))
    return (dL_da, dL_db, dL_dc), coef * ok


def chain(acc, radii, means3D, combined_opacity, clamped, shs, D, viewmatrix, projmatrix, campos, W, H, tan_fovx,
          tan_fovy, kernel_size, cov3D=None, scales=None, rotations=None, norm_rec=None, ortho=False, focal=False,
          exact=False, coef=None, hold_bound=False, dtype=torch.float64):
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


def translation_residual(g, viewmatrix, projmatrix):
    """sum_g dL/dmeans3D[g,i] + dL/dcampos[i] - sum_k V[i][k] G_V[3][k] - sum_k Pm[i][k] G_P[3][k], i = 0..2: zero when
    moving the world and the camera together leaves the loss unchanged.  Also returns the sum of the terms' magnitudes."""
    Vm = torch.as_tensor(viewmatrix).reshape(4, 4).to(g["view"])
    Pm = torch.as_tensor(projmatrix).reshape(4, 4).to(g["proj"])
    gm = g["means3D"].to(g["view"])
    parts = [gm.sum(0), g["campos"].to(g["view"]), -(Vm[:3] * g["view"][3]).sum(1), -(Pm[:3] * g["proj"][3]).sum(1)]
    scale = gm.abs().sum(0) + parts[1].abs() + (Vm[:3] * g["view"][3]).abs().sum(1) + (Pm[:3] * g["proj"][3]).abs().sum(1)
    return sum(parts), scale
