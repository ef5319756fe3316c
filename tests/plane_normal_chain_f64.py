"""Float64 (or float32) restatement of the per-Gaussian adjoint with the plane-normal terms, for
tests/test_plane_normals.py.

`chain` below is tests/ray_depth_chain_f64.py's `chain` with one more keyword, `plane_normals`.  With it on (it needs
ray_depth=True and scales / rotations as leaves), record i's normal is the normal of its ray-depth plane,
    u = w3 - g_x T0 - g_y T1,   n = sigma u / |u|,
with T0, T1 the rows of T = J W (the chain's J, clamp and focal handling), w3 the view's depth row, g = C s the ray-depth
slope and sigma the sign the forward chose, read off the record normals `norm_rec` as the kernel reads it.  The
restatement is split where the kernel splits it:
  - sum c . n (c = acc words 4-6) with g held at its value, differentiated by autograd with respect to means3D, the
    viewmatrix and tan_fov through T and w3 (the kernel's dL/dT and dL/dw3 routes);
  - dL/dg = -(T0 . dL/du, T1 . dL/du) added to acc words 14-15, and words 4-6 set to 0 (no shortest-axis term, and
    dL_dnorm3D is 0), then ray_depth_chain_f64.chain(ray_depth=True) on those sums (the ray-depth chain takes dL/dg to
    the conic, Sigma, T, w3, scales and rotations).
The results are the sum of the two.  `abs` (the camera terms' magnitude scale) adds the magnitudes of both parts, an
upper bound of the combined terms' magnitudes.  With plane_normals off the function is ray_depth_chain_f64.chain,
bit for bit."""
from __future__ import annotations

import numpy as np
import torch

import ray_depth_chain_f64 as RC
from chain_f64 import cov3d, quat_to_rot, sym6_to_mat


def plane_rows(m, Vw, h_x, h_y, limx, limy, Sig, ks, ortho, hold_bound=False):
    """T0, T1 [V,3], w3 [V,3] and the slope g [V,2] of Gaussians at m [V,3] under views Vw [V,4,4] (the chain's
    conventions; h / lim may be tensors carrying tan_fov's gradient).  g is formed without autograd."""
    tv = torch.einsum("gk,gkr->gr", m, Vw[:, :3, :3]) + Vw[:, 3, :3]
    tx, ty, tz = tv[:, 0], tv[:, 1], tv[:, 2]
    Wm = Vw[:, :3, :3].transpose(1, 2)
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
    w3 = Wm[:, 2, :]
    with torch.no_grad():
        S = Sig.detach()
        T0d, T1d, w3d = T0.detach(), T1.detach(), w3.detach()
        c00 = torch.einsum("gi,gij,gj->g", T0d, S, T0d) + ks
        c01 = torch.einsum("gi,gij,gj->g", T0d, S, T1d)
        c11 = torch.einsum("gi,gij,gj->g", T1d, S, T1d) + ks
        s0 = torch.einsum("gi,gij,gj->g", w3d, S, T0d)
        s1 = torch.einsum("gi,gij,gj->g", w3d, S, T1d)
        den = c00 * c11 - c01 * c01
        g = torch.stack([(c11 * s0 - c01 * s1) / den, (c00 * s1 - c01 * s0) / den], 1)
    return T0, T1, w3, g


def chain(acc, radii, means3D, combined_opacity, clamped, shs, D, viewmatrix, projmatrix, campos, W, H, tan_fovx,
          tan_fovy, kernel_size, cov3D=None, scales=None, rotations=None, norm_rec=None, ortho=False, focal=False,
          exact=False, coef=None, hold_bound=False, dtype=torch.float64, ray_depth=False, plane_normals=False):
    """ray_depth_chain_f64.chain's results (same arguments and keys); plane_normals=True: with the plane-normal terms
    (see the module's note)."""
    kw = dict(cov3D=cov3D, scales=scales, rotations=rotations, norm_rec=norm_rec, ortho=ortho, focal=focal,
              exact=exact, coef=coef, hold_bound=hold_bound, dtype=dtype, ray_depth=ray_depth)
    args = (radii, means3D, combined_opacity, clamped, shs, D, viewmatrix, projmatrix, campos, W, H, tan_fovx, tan_fovy,
            kernel_size)
    if not plane_normals:
        return RC.chain(acc, *args, **kw)
    assert ray_depth and scales is not None, "plane normals are a ray-depth option of a scales / rotations model"
    t = lambda a: torch.as_tensor(a).to(dtype)  # noqa: E731
    vis = torch.as_tensor(radii) > 0
    idx = torch.nonzero(vis).flatten()
    P, V = int(vis.numel()), int(idx.numel())
    dev = idx.device
    m = t(means3D)[idx].clone().requires_grad_(True)
    Vw = t(viewmatrix).reshape(4, 4).expand(V, 4, 4).clone().requires_grad_(not ortho)
    f32 = np.float32
    if focal:
        tnx = torch.full((V,), float(tan_fovx), dtype=dtype, device=dev, requires_grad=True)
        tny = torch.full((V,), float(tan_fovy), dtype=dtype, device=dev, requires_grad=True)
    if focal and exact:
        h_x, h_y, limx, limy = W / (2.0 * tnx), H / (2.0 * tny), 1.3 * tnx, 1.3 * tny
    elif focal:
        def pinned(value, x):
            return value + (x - x.detach())
        h_x = pinned(float(f32(W) / (f32(2.0) * f32(tan_fovx))), W / (2.0 * tnx))
        h_y = pinned(float(f32(H) / (f32(2.0) * f32(tan_fovy))), H / (2.0 * tny))
        limx = pinned(float(f32(1.3) * f32(tan_fovx)), 1.3 * tnx)
        limy = pinned(float(f32(1.3) * f32(tan_fovy)), 1.3 * tny)
    else:
        h_x = t(float(f32(W) / (f32(2.0) * f32(tan_fovx))))
        h_y = t(float(f32(H) / (f32(2.0) * f32(tan_fovy))))
        limx, limy = float(f32(1.3) * f32(tan_fovx)), float(f32(1.3) * f32(tan_fovy))
    ks = float(f32(kernel_size))
    Sig = sym6_to_mat(cov3d(t(scales)[idx], quat_to_rot(t(rotations)[idx])))
    T0, T1, w3, g = plane_rows(m, Vw, h_x, h_y, limx, limy, Sig, ks, ortho, hold_bound)
    u = w3 - g[:, 0:1] * T0 - g[:, 1:2] * T1
    if not u.requires_grad:           # orthographic: u is a constant of the camera, its gradient is dL/dg's alone
        u.requires_grad_(True)
    u.retain_grad()
    with torch.no_grad():
        sgn = torch.where((u * t(norm_rec)[idx]).sum(1) < 0, -1.0, 1.0).to(dtype)
    n = sgn[:, None] * u / torch.sqrt((u * u).sum(1, keepdim=True))
    A = t(acc)[idx]
    Ln = (A[:, 4:7] * n).sum(1)
    Ln.sum().backward()
    with torch.no_grad():
        du = u.grad
        acc2 = t(acc).clone()
        acc2[idx, 14] -= (T0 * du).sum(1)
        acc2[idx, 15] -= (T1 * du).sum(1)
        acc2[:, 4:7] = 0.0
    out = RC.chain(acc2, *args, **kw)
    with torch.no_grad():
        if m.grad is not None:
            out["means3D"][idx] += m.grad
        out["Lg"] = out["Lg"] + Ln.detach()
        if not ortho:
            terms = [Vw.grad.reshape(V, 16), torch.zeros((V, 19), dtype=dtype, device=dev)]
            out["view"] = out["view"] + Vw.grad.sum(0)
            if focal:
                terms += [tnx.grad[:, None], tny.grad[:, None]]
                out["tanx"] = out["tanx"] + tnx.grad.sum(0)
                out["tany"] = out["tany"] + tny.grad.sum(0)
            out["abs"] = out["abs"] + torch.cat(terms, 1).abs().sum(0)
        out["plane_normal"] = torch.zeros((P, 3), dtype=dtype, device=dev)
        out["plane_normal"][idx] = n.detach()
    return out
